// libmldb200 engine: weight packing, scheduler tables, transformer-stack orchestration,
// CUDA-graph capture and the C ABI declared in include/mldb.h.
#include "engine.h"

#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>

#include "gemm_tc.h"

// ----------------------------------------------------------------------------- errors
static thread_local std::string g_err;
void mldb_set_err(const std::string& s) { g_err = s; }
extern "C" const char* mldb_last_error(void) { return g_err.c_str(); }
extern "C" int mldb_abi_version(void) { return MLDB_ABI_VERSION; }

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t e__ = (call);                                                         \
    if (e__ != cudaSuccess) {                                                         \
      char buf__[512];                                                                \
      snprintf(buf__, sizeof buf__, "%s:%d: %s failed: %s", __FILE__, __LINE__, #call, \
               cudaGetErrorString(e__));                                              \
      mldb_set_err(buf__);                                                            \
      return MLDB_ERR_CUDA;                                                           \
    }                                                                                 \
  } while (0)

#define FAIL(code, ...)                         \
  do {                                          \
    char buf__[512];                            \
    snprintf(buf__, sizeof buf__, __VA_ARGS__); \
    mldb_set_err(buf__);                        \
    return (code);                              \
  } while (0)

#define TRY(expr)                 \
  do {                            \
    int rc__ = (expr);            \
    if (rc__ != MLDB_OK) return rc__; \
  } while (0)

// Every ABI call runs on the handle's device and restores the caller's current device afterwards
// (a single-process multi-GPU program must not find torch.cuda.current_device() changed under it).
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev); else prev = -1;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

static inline void count_launch(mldb_handle* h, int n = 1) {
  if (h->capturing) h->capture_nodes += n; else h->launches += n;
}

// ----------------------------------------------------------------------------- config
extern "C" void mldb_default_config(mldb_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = MLDB_ABI_VERSION;
  c->cond_kind = MLDB_COND_TEXT;
  c->arch = MLDB_ARCH_TRANS_ENC;
  c->latent_dim = 256; c->n_lat = 1; c->num_heads = 4; c->ff_size = 1024; c->num_layers = 9;
  c->text_dim = 768; c->nclasses = 12; c->nfeats = 263; c->diffusion_only = 0;
  c->flip_sin_to_cos = 1; c->freq_shift = 0.0f; c->guidance_scale = 7.5f;
  c->vae_kind = MLDB_VAE_MLD; c->vae_layers = 9; c->vae_heads = 4; c->vae_ff = 1024;
  c->vae_nfeats = 263;
  c->sched_kind = MLDB_SCHED_DDIM; c->num_train_timesteps = 1000;
  c->beta_start = 0.00085; c->beta_end = 0.012; c->steps_offset = 1; c->set_alpha_to_one = 0;
  c->eta = 0.0f; c->njoints = 22;
}

// ----------------------------------------------------------------------------- tensor spec
static void spec_add(mldb_handle* h, const std::string& key, std::vector<int64_t> shape) {
  RawTensor t; t.shape = std::move(shape);
  h->raw[key] = std::move(t);
}
static void spec_attn(mldb_handle* h, const std::string& p, int d) {
  spec_add(h, p + "in_proj_weight", {3 * d, d});
  spec_add(h, p + "in_proj_bias", {3 * d});
  spec_add(h, p + "out_proj.weight", {d, d});
  spec_add(h, p + "out_proj.bias", {d});
}
static void spec_ln(mldb_handle* h, const std::string& p, int d) {
  spec_add(h, p + "weight", {d});
  spec_add(h, p + "bias", {d});
}
static void spec_layer(mldb_handle* h, const std::string& p, int d, int ff, bool dec) {
  spec_attn(h, p + "self_attn.", d);
  if (dec) spec_attn(h, p + "multihead_attn.", d);
  spec_add(h, p + "linear1.weight", {ff, d});
  spec_add(h, p + "linear1.bias", {ff});
  spec_add(h, p + "linear2.weight", {d, ff});
  spec_add(h, p + "linear2.bias", {d});
  spec_ln(h, p + "norm1.", d);
  spec_ln(h, p + "norm2.", d);
  if (dec) spec_ln(h, p + "norm3.", d);
}
static void spec_skip_stack(mldb_handle* h, const std::string& p, int d, int ff, int layers, bool dec) {
  const int nb = (layers - 1) / 2;
  spec_ln(h, p + "norm.", d);
  for (int i = 0; i < nb; ++i) spec_layer(h, p + "input_blocks." + std::to_string(i) + ".", d, ff, dec);
  spec_layer(h, p + "middle_block.", d, ff, dec);
  for (int i = 0; i < nb; ++i) spec_layer(h, p + "output_blocks." + std::to_string(i) + ".", d, ff, dec);
  for (int i = 0; i < nb; ++i) {
    spec_add(h, p + "linear_blocks." + std::to_string(i) + ".weight", {d, 2 * d});
    spec_add(h, p + "linear_blocks." + std::to_string(i) + ".bias", {d});
  }
}

static int build_spec(mldb_handle* h) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim;
  const std::string D = "denoiser.";
  if (c.num_layers > 0) {   // num_layers == 0: VAE-only handle
  if (c.diffusion_only) {
    spec_add(h, D + "pose_embd.weight", {d, c.nfeats});
    spec_add(h, D + "pose_embd.bias", {d});
    spec_add(h, D + "pose_proj.weight", {c.nfeats, d});
    spec_add(h, D + "pose_proj.bias", {c.nfeats});
  }
  const int tdim = c.cond_kind == MLDB_COND_TEXT ? c.text_dim : d;   // mld_denoiser.py:57,70
  spec_add(h, D + "time_embedding.linear_1.weight", {d, tdim});
  spec_add(h, D + "time_embedding.linear_1.bias", {d});
  spec_add(h, D + "time_embedding.linear_2.weight", {d, d});
  spec_add(h, D + "time_embedding.linear_2.bias", {d});
  if (c.cond_kind == MLDB_COND_TEXT) {
    if (c.text_dim != d) {
      spec_add(h, D + "emb_proj.1.weight", {d, c.text_dim});
      spec_add(h, D + "emb_proj.1.bias", {d});
    }
  } else {
    spec_add(h, D + "emb_proj.action_embedding", {c.nclasses, d});
  }
  spec_add(h, D + "query_pos.pe", {500, 1, d});
  spec_add(h, D + "mem_pos.pe", {500, 1, d});
  if (c.arch == MLDB_ARCH_TRANS_ENC) {
    spec_skip_stack(h, D + "encoder.", d, c.ff_size, c.num_layers, false);
  } else {
    for (int i = 0; i < c.num_layers; ++i)
      spec_layer(h, D + "decoder.layers." + std::to_string(i) + ".", d, c.ff_size, true);
    spec_ln(h, D + "decoder.norm.", d);
  }
  }
  const std::string V = "vae.";
  if (c.vae_kind == MLDB_VAE_MLD) {
    spec_add(h, V + "global_motion_token", {2 * c.n_lat, d});
    spec_add(h, V + "query_pos_encoder.pe", {500, 1, d});
    spec_add(h, V + "query_pos_decoder.pe", {500, 1, d});
    spec_skip_stack(h, V + "encoder.", d, c.vae_ff, c.vae_layers, false);
    spec_skip_stack(h, V + "decoder.", d, c.vae_ff, c.vae_layers, true);
    spec_add(h, V + "skel_embedding.weight", {d, c.vae_nfeats});
    spec_add(h, V + "skel_embedding.bias", {d});
    spec_add(h, V + "final_layer.weight", {c.vae_nfeats, d});
    spec_add(h, V + "final_layer.bias", {c.vae_nfeats});
  } else if (c.vae_kind == MLDB_VAE_ACTOR) {
    spec_add(h, V + "decoder.sequence_pos_encoding.pe", {5000, 1, d});
    for (int i = 0; i < c.vae_layers; ++i)
      spec_layer(h, V + "decoder.seqTransDecoder.layers." + std::to_string(i) + ".", d, c.vae_ff, true);
    spec_add(h, V + "decoder.final_layer.weight", {c.vae_nfeats, d});
    spec_add(h, V + "decoder.final_layer.bias", {c.vae_nfeats});
  }
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- alloc / pack
static int dev_alloc(mldb_handle* h, void** p, size_t bytes) {
  CK(cudaMalloc(p, bytes ? bytes : 16));
  h->allocs.push_back(*p);
  return MLDB_OK;
}
static int upload_f32(mldb_handle* h, const float* src, size_t n, float** out) {
  TRY(dev_alloc(h, (void**)out, n * sizeof(float)));
  CK(cudaMemcpy(*out, src, n * sizeof(float), cudaMemcpyHostToDevice));
  return MLDB_OK;
}
static const RawTensor& rt(mldb_handle* h, const std::string& k) { return h->raw.at(k); }

// Pack a host [N, K] fp32 matrix into split fp16 planes scaled by 2^s.  Kpad > K zero-pads the rows
// (odd K such as the 263 motion features: the tensor-core GEMM wants K % 64 == 0).
static int pack_linear(mldb_handle* h, const float* W, int N, int K, const float* bias, LinW* out, int Kpad = 0) {
  if (Kpad < K) Kpad = K;
  float mx = 0.0f;
  for (int64_t i = 0; i < (int64_t)N * K; ++i) mx = std::max(mx, fabsf(W[i]));
  int s = 0;
  if (mx > 0.0f) {
    s = (int)floorf(log2f(16384.0f / mx));
    s = std::max(-14, std::min(14, s));
  }
  const float sc = ldexpf(1.0f, s);
  std::vector<__half> buf((size_t)2 * N * Kpad, __float2half_rn(0.0f));
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) {
      const float w = W[(size_t)n * K + k] * sc;
      const __half hi = __float2half_rn(w);
      buf[(size_t)n * Kpad + k] = hi;
      buf[(size_t)N * Kpad + (size_t)n * Kpad + k] = __float2half_rn(w - __half2float(hi));
    }
  TRY(dev_alloc(h, (void**)&out->w, buf.size() * sizeof(__half)));
  CK(cudaMemcpy(out->w, buf.data(), buf.size() * sizeof(__half), cudaMemcpyHostToDevice));
  out->plane_stride = (int64_t)N * Kpad;
  out->N = N; out->K = Kpad; out->inv_scale = ldexpf(1.0f, -s);
  out->bias = nullptr;
  if (bias) TRY(upload_f32(h, bias, N, &out->bias));
  static int next_id = 0;
  out->id = next_id++;
  return MLDB_OK;
}
static int pack_named(mldb_handle* h, const std::string& wkey, const std::string& bkey, LinW* out,
                      int row0 = 0, int nrows = -1, bool pad_k = false) {
  const RawTensor& w = rt(h, wkey);
  const int K = (int)w.shape.back();
  const int Nall = (int)w.shape[0];
  if (nrows < 0) nrows = Nall;
  const float* b = bkey.empty() ? nullptr : rt(h, bkey).host.data() + row0;
  return pack_linear(h, w.host.data() + (size_t)row0 * K, nrows, K, b, out, pad_k ? (K + 63) / 64 * 64 : 0);
}
static int pack_ln(mldb_handle* h, const std::string& p, int d, LnW* out) {
  TRY(upload_f32(h, rt(h, p + "weight").host.data(), d, &out->g));
  TRY(upload_f32(h, rt(h, p + "bias").host.data(), d, &out->b));
  return MLDB_OK;
}
static int pack_enc_layer(mldb_handle* h, const std::string& p, int d, EncW* w) {
  TRY(pack_named(h, p + "self_attn.in_proj_weight", p + "self_attn.in_proj_bias", &w->in_proj));
  TRY(pack_named(h, p + "self_attn.out_proj.weight", p + "self_attn.out_proj.bias", &w->out_proj));
  TRY(pack_named(h, p + "linear1.weight", p + "linear1.bias", &w->l1));
  TRY(pack_named(h, p + "linear2.weight", p + "linear2.bias", &w->l2));
  TRY(pack_ln(h, p + "norm1.", d, &w->n1));
  TRY(pack_ln(h, p + "norm2.", d, &w->n2));
  return MLDB_OK;
}
static int pack_dec_layer(mldb_handle* h, const std::string& p, int d, DecW* w) {
  TRY(pack_named(h, p + "self_attn.in_proj_weight", p + "self_attn.in_proj_bias", &w->sa_in));
  TRY(pack_named(h, p + "self_attn.out_proj.weight", p + "self_attn.out_proj.bias", &w->sa_out));
  // packed in_proj rows are [Wq; Wk; Wv] (nn.MultiheadAttention): q part and kv part
  TRY(pack_named(h, p + "multihead_attn.in_proj_weight", p + "multihead_attn.in_proj_bias", &w->ca_q, 0, d));
  TRY(pack_named(h, p + "multihead_attn.in_proj_weight", p + "multihead_attn.in_proj_bias", &w->ca_kv, d, 2 * d));
  TRY(pack_named(h, p + "multihead_attn.in_proj_weight", p + "multihead_attn.in_proj_bias", &w->ca_v, 2 * d, d));
  TRY(pack_named(h, p + "multihead_attn.out_proj.weight", p + "multihead_attn.out_proj.bias", &w->ca_out));
  TRY(pack_named(h, p + "linear1.weight", p + "linear1.bias", &w->l1));
  TRY(pack_named(h, p + "linear2.weight", p + "linear2.bias", &w->l2));
  TRY(pack_ln(h, p + "norm1.", d, &w->n1));
  TRY(pack_ln(h, p + "norm2.", d, &w->n2));
  TRY(pack_ln(h, p + "norm3.", d, &w->n3));
  return MLDB_OK;
}
static int pack_skip_stack(mldb_handle* h, const std::string& p, int d, int ff, int heads, int layers,
                           bool dec, StackW* s) {
  s->kind = dec ? STACK_SKIP_DEC : STACK_SKIP_ENC;
  s->d = d; s->ff = ff; s->heads = heads; s->layers = layers;
  const int nb = (layers - 1) / 2;
  std::vector<std::string> names;
  for (int i = 0; i < nb; ++i) names.push_back(p + "input_blocks." + std::to_string(i) + ".");
  names.push_back(p + "middle_block.");
  for (int i = 0; i < nb; ++i) names.push_back(p + "output_blocks." + std::to_string(i) + ".");
  for (auto& n : names) {
    if (dec) { s->dec.emplace_back(); TRY(pack_dec_layer(h, n, d, &s->dec.back())); }
    else     { s->enc.emplace_back(); TRY(pack_enc_layer(h, n, d, &s->enc.back())); }
  }
  if (!dec) {   // the last block only has to produce the first few tokens of every sequence
    const std::string& n = names.back();
    EncW& w = s->enc.back();
    TRY(pack_named(h, n + "self_attn.in_proj_weight", n + "self_attn.in_proj_bias", &w.q_only, 0, d));
    TRY(pack_named(h, n + "self_attn.in_proj_weight", n + "self_attn.in_proj_bias", &w.kv_only, d, 2 * d));
  }
  for (int i = 0; i < nb; ++i) {
    s->skip.emplace_back();
    const std::string lp = p + "linear_blocks." + std::to_string(i) + ".";
    TRY(pack_named(h, lp + "weight", lp + "bias", &s->skip.back()));
  }
  TRY(pack_ln(h, p + "norm.", d, &s->norm));
  return MLDB_OK;
}
static int upload_pe(mldb_handle* h, const std::string& key, float** out, int* rows = nullptr) {
  const RawTensor& t = rt(h, key);
  if (rows) *rows = (int)t.shape[0];
  return upload_f32(h, t.host.data(), t.host.size(), out);
}

// ----------------------------------------------------------------------------- scheduler
// betas = linspace(sqrt(b0), sqrt(b1), T, fp32) ** 2 ; alphas_cumprod = cumprod(1 - betas)
// (diffusers scaled_linear schedule; fp32 throughout like torch).
static void build_alphas(const mldb_config& c, std::vector<float>* out) {
  // Bit-exact with torch on CPU (checked in tests/test_scheduler.py): linspace evaluates
  // start + step*i (first half) / end - step*(T-1-i) (second half) with one rounding (FMA);
  // cumprod accumulates in double (at::acc_type<float> on CPU) and rounds each output.
  const int T = c.num_train_timesteps;
  out->resize(T);
  const float s0 = (float)sqrt(c.beta_start), s1 = (float)sqrt(c.beta_end);
  const float step = (s1 - s0) / (float)(T - 1);
  double prod = 1.0;
  for (int i = 0; i < T; ++i) {
    const float v = (i < T / 2) ? fmaf(step, (float)i, s0) : fmaf(-step, (float)(T - 1 - i), s1);
    const float beta = v * v;
    const float alpha = 1.0f - beta;
    prod *= (double)alpha;
    (*out)[i] = (float)prod;
  }
}
extern "C" int mldb_scheduler_table(const mldb_config* cfg, float* alphas_cumprod_out) {
  if (!cfg || !alphas_cumprod_out) FAIL(MLDB_ERR_INVALID, "null argument");
  std::vector<float> a;
  build_alphas(*cfg, &a);
  memcpy(alphas_cumprod_out, a.data(), a.size() * sizeof(float));
  return MLDB_OK;
}
// Integer timestep schedule, bit-exact with diffusers set_timesteps.
extern "C" int mldb_scheduler_timesteps(const mldb_config* cfg, int32_t n, int64_t* out) {
  if (!cfg || !out || n <= 0 || n > cfg->num_train_timesteps) FAIL(MLDB_ERR_INVALID, "bad n");
  const int64_t ratio = cfg->num_train_timesteps / n;
  const int64_t off = cfg->sched_kind == MLDB_SCHED_DDIM ? cfg->steps_offset : 0;
  for (int i = 0; i < n; ++i) out[i] = (int64_t)(n - 1 - i) * ratio + off;
  return MLDB_OK;
}
static StepCoef make_coef(const mldb_handle* h, int64_t t, int n_inference) {
  const mldb_config& c = h->cfg;
  const std::vector<float>& ac = h->alphas_cumprod;
  StepCoef k{};
  const int64_t prev_t = t - c.num_train_timesteps / n_inference;
  const float a_t = ac[t];
  k.c0 = sqrtf(a_t);
  k.c1 = sqrtf(1.0f - a_t);
  if (c.sched_kind == MLDB_SCHED_DDIM) {
    const float a_prev = prev_t >= 0 ? ac[prev_t] : (c.set_alpha_to_one ? 1.0f : ac[0]);
    k.kind = 0;
    k.c2 = sqrtf(a_prev);
    k.c3 = sqrtf(1.0f - a_prev - 0.0f);   // eta == 0 => std_dev_t == 0
    k.sigma = 0.0f;
  } else {
    const float a_prev = prev_t >= 0 ? ac[prev_t] : 1.0f;
    const float bpt = 1.0f - a_t, bpp = 1.0f - a_prev;
    const float cur_alpha = a_t / a_prev, cur_beta = 1.0f - cur_alpha;
    k.kind = 1;
    k.c2 = (sqrtf(a_prev) * cur_beta) / bpt;
    k.c3 = sqrtf(cur_alpha) * bpp / bpt;
    k.sigma = t > 0 ? sqrtf(std::max(bpp / bpt * cur_beta, 1e-20f)) : 0.0f;
  }
  return k;
}

static inline unsigned nblk(int64_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }

// ----------------------------------------------------------------------------- op dispatch
static inline ActBuf rows_of(ActBuf b, int64_t row0, int rows) {
  b.hi += row0 * b.cols; b.rows = rows; return b;
}
static inline void kcount(mldb_handle* h, int kind) { h->kstat[kind]++; count_launch(h); }
static void op_gemm(mldb_handle* h, const GemmArgs& g, cudaStream_t st) {
  if (h->use_tc && tc_gemm_supported(h->tc, g)) {
    if (!tc_gemm(h->tc, g, nullptr, st)) h->op_failed = true;
    kcount(h, MLDB_KSTAT_GEMM_TC);
    return;
  }
  simt_gemm(g, st);
  kcount(h, MLDB_KSTAT_GEMM_SIMT);
}
// GEMM followed by residual + LayerNorm (one fused wgmma kernel when the tile covers a row)
static void op_gemm_ln(mldb_handle* h, GemmArgs g, LnArgs l, float* cf32, cudaStream_t st) {
  if (h->use_tc && tc_gemm_ln_supported(h->tc, g, l)) {
    if (!tc_gemm(h->tc, g, &l, st)) h->op_failed = true;
    kcount(h, MLDB_KSTAT_GEMM_LN_TC);
    return;
  }
  g.out = ActBuf{}; g.out_f32 = cf32; g.ldc = g.w.N;
  op_gemm(h, g, st);
  l.c = cf32; l.ldc = g.w.N;
  simt_ln(l, st);
  kcount(h, h->use_tc ? MLDB_KSTAT_LN_UNFUSED : MLDB_KSTAT_LN_SIMT);
}
static void op_ln(mldb_handle* h, const LnArgs& l, cudaStream_t st) { simt_ln(l, st); kcount(h, MLDB_KSTAT_LN_SIMT); }
static void op_attn(mldb_handle* h, const AttnArgs& a, cudaStream_t st) {
  if (h->use_tc && h->attn_kind == 0 && tc_attention_supported(a)) {
    if (!tc_attention(a, st)) h->op_failed = true;
    kcount(h, MLDB_KSTAT_ATTN_TC);
  } else if (h->use_tc && h->attn_kind <= 1 && mma_attention_supported(a)) {
    mma_attention(a, st);
    kcount(h, MLDB_KSTAT_ATTN_MMA);
  } else {
    simt_attention(a, st);
    kcount(h, MLDB_KSTAT_ATTN_SIMT);
  }
}
// the fused FFN block when the shape allows it, else the two GEMMs
static void op_ffn(mldb_handle* h, const GemmArgs& g1, const GemmArgs& g2, const LnArgs& l2, float* cf32, cudaStream_t st) {
  if (h->use_tc && tc_ffn_supported(h->tc, g1, g2, l2)) {
    // one launch: the hidden activations stay in registers (gemm_tc.cu k_ffn_tc)
    int k = 0;                                     // which stream: its own scratch (branches run concurrently)
    for (int i = 0; i < mldb_handle::MAX_BRANCHES - 1; ++i) if (st == h->br_stream[i]) k = i + 1;
    if (!tc_ffn(h->tc, g1, g2, l2, h->ffn_scratch[k], h->ffn_flags[k], st)) h->op_failed = true;
    kcount(h, MLDB_KSTAT_FFN_TC);
    return;
  }
  op_gemm(h, g1, st);
  op_gemm_ln(h, g2, l2, cf32, st);
}

// ----------------------------------------------------------------------------- workspaces
static int alloc_act(mldb_handle* h, int rows, int cols, ActBuf* out) {
  const int64_t rp = ((int64_t)rows + 127) / 128 * 128;
  __half* p = nullptr;
  TRY(dev_alloc(h, (void**)&p, (size_t)2 * rp * cols * sizeof(__half)));
  CK(cudaMemset(p, 0, (size_t)2 * rp * cols * sizeof(__half)));
  out->hi = p; out->plane_stride = rp * cols; out->rows = rows; out->cols = cols;
  return MLDB_OK;
}
static int alloc_stack_ws(mldb_handle* h, const StackW& sw, int nseq, int L, int Lmem, StackWs* ws,
                          int n_sel = 0) {
  ws->nseq = nseq; ws->L = L; ws->M = nseq * L; ws->d = sw.d; ws->ff = sw.ff; ws->Lmem = Lmem;
  const int M = ws->M, d = sw.d;
  TRY(alloc_act(h, M, d, &ws->x0));
  TRY(alloc_act(h, M, d, &ws->cur[0]));
  TRY(alloc_act(h, M, d, &ws->cur[1]));
  TRY(alloc_act(h, M, d, &ws->x1));
  TRY(alloc_act(h, M, d, &ws->att));
  TRY(alloc_act(h, M, 3 * d, &ws->qkv));
  TRY(alloc_act(h, M, sw.ff, &ws->h));
  if (sw.kind != STACK_SKIP_ENC) {
    TRY(alloc_act(h, M, d, &ws->x2));
    TRY(alloc_act(h, M, d, &ws->qc));
    TRY(alloc_act(h, nseq * Lmem, 2 * d, &ws->kvm));
    TRY(alloc_act(h, nseq, d, &ws->vrow));
    TRY(dev_alloc(h, (void**)&ws->cvec, (size_t)nseq * d * sizeof(float)));
  }
  if (sw.kind != STACK_PLAIN_DEC) {
    TRY(alloc_act(h, M, d, &ws->cat));
    const int nb = (sw.layers - 1) / 2;
    ws->ys.resize(nb);
    for (int i = 0; i < nb; ++i) TRY(alloc_act(h, M, d, &ws->ys[i]));
  }
  TRY(dev_alloc(h, (void**)&ws->cf32, (size_t)M * d * sizeof(float)));
  if (sw.kind == STACK_SKIP_ENC && n_sel > 0) {
    ws->n_sel = n_sel;
    const int R = nseq * n_sel;
    TRY(alloc_act(h, R, d, &ws->sx));
    TRY(alloc_act(h, R, d, &ws->sq));
    TRY(alloc_act(h, R, d, &ws->satt));
    TRY(alloc_act(h, R, d, &ws->sx1));
    TRY(alloc_act(h, R, sw.ff, &ws->sh));
    TRY(alloc_act(h, R, d, &ws->sout));
  }
  return MLDB_OK;
}

struct SeqInfo {
  const int32_t* lengths = nullptr;  // key-padding: valid keys = kv_prefix + lengths[s % len_mod]
  int kv_prefix = 0;
  int len_mod = 0;
};

// the workspace rows of sequences [s0, s0 + n): a self-contained workspace for that sub-batch
static StackWs ws_slice(const StackWs& ws, int s0, int n) {
  StackWs w = ws;
  w.nseq = n; w.M = n * ws.L;
  auto tok = [&](ActBuf b) { return b.hi ? rows_of(b, (int64_t)s0 * ws.L, n * ws.L) : b; };
  auto sel = [&](ActBuf b) { return b.hi ? rows_of(b, (int64_t)s0 * ws.n_sel, n * ws.n_sel) : b; };
  w.x0 = tok(ws.x0); w.cur[0] = tok(ws.cur[0]); w.cur[1] = tok(ws.cur[1]); w.x1 = tok(ws.x1); w.x2 = tok(ws.x2);
  w.att = tok(ws.att); w.qkv = tok(ws.qkv); w.qc = tok(ws.qc); w.h = tok(ws.h); w.cat = tok(ws.cat);
  for (auto& y : w.ys) y = tok(y);
  if (ws.kvm.hi) w.kvm = rows_of(ws.kvm, (int64_t)s0 * ws.Lmem, n * ws.Lmem);
  if (ws.vrow.hi) w.vrow = rows_of(ws.vrow, s0, n);
  if (ws.cvec) w.cvec = ws.cvec + (size_t)s0 * ws.d;
  if (ws.cf32) w.cf32 = ws.cf32 + (size_t)s0 * ws.L * ws.d;
  w.sx = sel(ws.sx); w.sq = sel(ws.sq); w.satt = sel(ws.satt); w.sx1 = sel(ws.sx1); w.sh = sel(ws.sh); w.sout = sel(ws.sout);
  return w;
}
// out-projection + residual + LayerNorm (cross_attention.py:262-263)
static void out_proj_ln(mldb_handle* h, const LinW& w, const LnW& n, ActBuf att, ActBuf res, ActBuf xout, int M, int d,
                        float* cf32, cudaStream_t st) {
  GemmArgs g; g.a1 = att; g.K1 = d; g.M = M; g.w = w;
  LnArgs l; l.res = res; l.gamma = n.g; l.beta = n.b; l.M = M; l.d = d; l.out = xout;
  op_gemm_ln(h, g, l, cf32, st);
}
static void self_attn_block(mldb_handle* h, const LinW& in_proj, const LinW& out_proj, const LnW& n,
                            ActBuf xin, ActBuf xout, StackWs& ws, const SeqInfo& si, int heads,
                            cudaStream_t st) {
  const int d = ws.d;
  GemmArgs g; g.a1 = xin; g.K1 = d; g.M = ws.M; g.w = in_proj; g.out = ws.qkv;
  op_gemm(h, g, st);
  AttnArgs a; a.q = ws.qkv; a.q_col0 = 0; a.Lq = ws.L; a.kv = ws.qkv; a.k_col0 = d; a.v_col0 = 2 * d;
  a.Lk = ws.L; a.nseq = ws.nseq; a.heads = heads; a.hd = d / heads;
  a.lengths = si.lengths; a.kv_prefix = si.kv_prefix; a.len_mod = si.len_mod; a.seq0 = 0; a.out = ws.att;
  op_attn(h, a, st);
  out_proj_ln(h, out_proj, n, ws.att, xin, xout, ws.M, d, ws.cf32, st);
}
static void ffn_block(mldb_handle* h, const LinW& l1, const LinW& l2, const LnW& n, ActBuf xin,
                      ActBuf xout, StackWs& ws, int act, cudaStream_t st) {
  GemmArgs g; g.a1 = xin; g.K1 = ws.d; g.M = ws.M; g.w = l1; g.act = act; g.out = ws.h;
  GemmArgs g2; g2.a1 = ws.h; g2.K1 = ws.ff; g2.M = ws.M; g2.w = l2;
  LnArgs l; l.res = xin; l.gamma = n.g; l.beta = n.b; l.M = ws.M; l.d = ws.d; l.out = xout;
  op_ffn(h, g, g2, l, ws.cf32, st);
}
// TransformerEncoderLayer.forward_post (cross_attention.py:259-272)
static void enc_layer(mldb_handle* h, const StackW& sw, const EncW& w, ActBuf xin, ActBuf xout,
                      StackWs& ws, const SeqInfo& si, cudaStream_t st) {
  self_attn_block(h, w.in_proj, w.out_proj, w.n1, xin, ws.x1, ws, si, sw.heads, st);
  ffn_block(h, w.l1, w.l2, w.n2, ws.x1, xout, ws, ACT_GELU, st);
}
// TransformerDecoderLayer.forward_post (cross_attention.py:323-345)
static void dec_layer(mldb_handle* h, const StackW& sw, const DecW& w, ActBuf xin, ActBuf xout,
                      ActBuf mem, StackWs& ws, const SeqInfo& si, cudaStream_t st) {
  const int d = ws.d;
  self_attn_block(h, w.sa_in, w.sa_out, w.n1, xin, ws.x1, ws, si, sw.heads, st);
  if (ws.Lmem == 1) {
    // One memory token: softmax over a single key is exactly 1, so the cross-attention output of
    // every query row of sequence b is out_proj(W_v z_b + b_v) + b_o - a per-sequence vector added
    // before norm2 (no q projection, no attention kernel, no [M,d] out-projection).
    GemmArgs gv; gv.a1 = mem; gv.K1 = d; gv.M = ws.nseq; gv.w = w.ca_v; gv.out = ws.vrow;
    op_gemm(h, gv, st);
    GemmArgs gc; gc.a1 = ws.vrow; gc.K1 = d; gc.M = ws.nseq; gc.w = w.ca_out; gc.out_f32 = ws.cvec; gc.ldc = d;
    op_gemm(h, gc, st);
    LnArgs lc; lc.res = ws.x1; lc.rowvec = ws.cvec; lc.rv_group = ws.L; lc.gamma = w.n2.g; lc.beta = w.n2.b;
    lc.M = ws.M; lc.d = d; lc.out = ws.x2;
    op_ln(h, lc, st);
    ffn_block(h, w.l1, w.l2, w.n3, ws.x2, xout, ws, ACT_GELU, st);
    return;
  }
  // cross attention: query = tgt, key = value = memory, no memory mask
  GemmArgs gq; gq.a1 = ws.x1; gq.K1 = d; gq.M = ws.M; gq.w = w.ca_q; gq.out = ws.qc;
  op_gemm(h, gq, st);
  GemmArgs gk; gk.a1 = mem; gk.K1 = d; gk.M = ws.nseq * ws.Lmem; gk.w = w.ca_kv; gk.out = ws.kvm;
  op_gemm(h, gk, st);
  AttnArgs a; a.q = ws.qc; a.q_col0 = 0; a.Lq = ws.L; a.kv = ws.kvm; a.k_col0 = 0; a.v_col0 = d;
  a.Lk = ws.Lmem; a.nseq = ws.nseq; a.heads = sw.heads; a.hd = d / sw.heads; a.out = ws.att;
  op_attn(h, a, st);
  out_proj_ln(h, w.ca_out, w.n2, ws.att, ws.x1, ws.x2, ws.M, d, ws.cf32, st);
  ffn_block(h, w.l1, w.l2, w.n3, ws.x2, xout, ws, ACT_GELU, st);
}
static void any_layer(mldb_handle* h, const StackW& sw, int li, ActBuf xin, ActBuf xout, ActBuf mem,
                      StackWs& ws, const SeqInfo& si, cudaStream_t st) {
  if (sw.kind == STACK_SKIP_ENC) enc_layer(h, sw, sw.enc[li], xin, xout, ws, si, st);
  else dec_layer(h, sw, sw.dec[li], xin, xout, mem, ws, si, st);
}
// rows (s, j < n_sel) of a [nseq, L] token buffer -> compact [nseq * n_sel] rows
__global__ void k_gather_rows(ActBuf src, ActBuf dst, int L, int n_sel, int nrows_out, int d) {
  pdl_trigger();
  pdl_wait();
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)nrows_out * (d / 8)) return;
  const int c = (int)(idx % (d / 8));
  const int r = (int)(idx / (d / 8));
  const int64_t srow = (int64_t)(r / n_sel) * L + r % n_sel;
  const uint4* sh = reinterpret_cast<const uint4*>(src.hi + srow * src.cols) + c;
  const uint4* sl = reinterpret_cast<const uint4*>(src.lo() + srow * src.cols) + c;
  reinterpret_cast<uint4*>(dst.hi + (int64_t)r * dst.cols)[c] = *sh;
  reinterpret_cast<uint4*>(dst.lo() + (int64_t)r * dst.cols)[c] = *sl;
}

// Last block of a skip encoder when only the first n_sel tokens of every sequence are consumed
// downstream (the denoiser returns tokens[:n_lat], mld_denoiser.py:206; MldVae.encode keeps the
// distribution tokens, mld_vae.py:161).  Keys and values still come from every token, but queries,
// the out-projection, both LayerNorms and the whole FFN run on the selected rows only - exactly
// the rows the full layer would have produced, since everything after attention is per-token.
static ActBuf enc_layer_selected(mldb_handle* h, const StackW& sw, const EncW& w, ActBuf xin, StackWs& ws,
                                 const SeqInfo& si, cudaStream_t st) {
  const int d = ws.d, R = ws.nseq * ws.n_sel;
  GemmArgs gk; gk.a1 = xin; gk.K1 = d; gk.M = ws.M; gk.w = w.kv_only; gk.out = ws.qkv;   // K | V in cols [0, 2d)
  op_gemm(h, gk, st);
  launch_pdl(k_gather_rows, dim3(nblk((int64_t)R * (d / 8))), dim3(256), 0, st, xin, ws.sx, ws.L, ws.n_sel, R, d);
  kcount(h, MLDB_KSTAT_MISC);
  GemmArgs gq; gq.a1 = ws.sx; gq.K1 = d; gq.M = R; gq.w = w.q_only; gq.out = ws.sq;
  op_gemm(h, gq, st);
  AttnArgs a; a.q = ws.sq; a.q_col0 = 0; a.Lq = ws.n_sel; a.kv = ws.qkv; a.k_col0 = 0; a.v_col0 = d;
  a.Lk = ws.L; a.nseq = ws.nseq; a.heads = sw.heads; a.hd = d / sw.heads; a.lengths = si.lengths;
  a.kv_prefix = si.kv_prefix; a.len_mod = si.len_mod; a.out = ws.satt;
  op_attn(h, a, st);
  out_proj_ln(h, w.out_proj, w.n1, ws.satt, ws.sx, ws.sx1, R, d, ws.cf32, st);
  GemmArgs g1; g1.a1 = ws.sx1; g1.K1 = d; g1.M = R; g1.w = w.l1; g1.act = ACT_GELU; g1.out = ws.sh;
  GemmArgs g2; g2.a1 = ws.sh; g2.K1 = ws.ff; g2.M = R; g2.w = w.l2;
  LnArgs l2; l2.res = ws.sx1; l2.gamma = w.n2.g; l2.beta = w.n2.b; l2.M = R; l2.d = d; l2.out = ws.sout;
  op_ffn(h, g1, g2, l2, ws.cf32, st);
  return ws.sout;
}

// SkipTransformerEncoder/Decoder.forward (cross_attention.py:41-64, 89-125) and the plain
// decoder stacks (cross_attention.py:204-233; torch nn.TransformerDecoder for ActorVae).
// Returns the buffer holding the last layer's output (before the stack's final norm).
static ActBuf run_stack(mldb_handle* h, const StackW& sw, ActBuf x0, ActBuf mem, StackWs& ws,
                        const SeqInfo& si, cudaStream_t st) {
  if (sw.kind == STACK_PLAIN_DEC) {
    ActBuf x = x0;
    for (int i = 0; i < sw.layers; ++i) {
      any_layer(h, sw, i, x, ws.cur[i & 1], mem, ws, si, st);
      x = ws.cur[i & 1];
    }
    return x;
  }
  const int nb = (sw.layers - 1) / 2;
  ActBuf x = x0;
  for (int i = 0; i < nb; ++i) {
    any_layer(h, sw, i, x, ws.ys[i], mem, ws, si, st);
    x = ws.ys[i];
  }
  any_layer(h, sw, nb, x, ws.cur[0], mem, ws, si, st);
  x = ws.cur[0];
  for (int i = 0; i < nb; ++i) {
    GemmArgs g; g.a1 = x; g.K1 = sw.d; g.a2 = ws.ys[nb - 1 - i]; g.K2 = sw.d; g.M = ws.M;
    g.w = sw.skip[i]; g.out = ws.cat;
    op_gemm(h, g, st);
    if (i == nb - 1 && sw.kind == STACK_SKIP_ENC && ws.n_sel > 0)
      return enc_layer_selected(h, sw, sw.enc[nb + 1 + i], ws.cat, ws, si, st);   // compact rows
    any_layer(h, sw, nb + 1 + i, ws.cat, ws.cur[(i + 1) & 1], mem, ws, si, st);
    x = ws.cur[(i + 1) & 1];
  }
  return x;
}

// ----------------------------------------------------------------------------- create/destroy
extern "C" int mldb_create(const mldb_config* cfg, int device, mldb_handle** out) {
  if (!cfg || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  if (cfg->abi_version != MLDB_ABI_VERSION) FAIL(MLDB_ERR_INVALID, "abi_version mismatch");
  if (cfg->latent_dim % cfg->num_heads || cfg->latent_dim % 32) FAIL(MLDB_ERR_INVALID, "latent_dim must be a multiple of 32 and of num_heads");
  if (cfg->latent_dim > 1024) FAIL(MLDB_ERR_UNSUPPORTED, "latent_dim > 1024");
  if (cfg->arch == MLDB_ARCH_TRANS_ENC && cfg->num_layers > 0 && cfg->num_layers % 2 != 1) FAIL(MLDB_ERR_INVALID, "skip encoder needs an odd layer count");
  if (cfg->arch == MLDB_ARCH_TRANS_ENC && cfg->diffusion_only) FAIL(MLDB_ERR_UNSUPPORTED, "diffusion_only requires arch trans_dec");
  if (cfg->vae_kind == MLDB_VAE_MLD && cfg->vae_layers % 2 != 1) FAIL(MLDB_ERR_INVALID, "MldVae needs an odd layer count");
  if (cfg->sched_kind == MLDB_SCHED_DDIM && cfg->eta != 0.0f) FAIL(MLDB_ERR_UNSUPPORTED, "DDIM eta != 0");
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) FAIL(MLDB_ERR_INVALID, "no such CUDA device %d (no CPU fallback exists)", device);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9) FAIL(MLDB_ERR_UNSUPPORTED, "device %d is sm_%d%d; libmldb200 is sm_90a only", device, prop.major, prop.minor);
  DeviceGuard guard(device);
  mldb_handle* h = new mldb_handle();
  h->cfg = *cfg; h->device = device; h->sm_count = prop.multiProcessorCount;
  build_spec(h);
  build_alphas(h->cfg, &h->alphas_cumprod);
  cudaError_t e = cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete h; FAIL(MLDB_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e)); }
  simt_init();
  mma_attention_init();
  h->tc = tc_create(device);
  if (!h->tc) { delete h; return MLDB_ERR_CUDA; }
  if (!tc_attention_init(device)) { tc_destroy(h->tc); delete h; FAIL(MLDB_ERR_CUDA, "wgmma attention kernel: setup failed"); }
  const char* env = getenv("MLDB_GEMM");
  if (env && !strcmp(env, "simt")) h->use_tc = false;
  env = getenv("MLDB_GRAPH");
  if (env && !strcmp(env, "0")) h->use_graph = false;
  env = getenv("MLDB_ATTN");
  if (env) h->attn_kind = !strcmp(env, "mma") ? 1 : (!strcmp(env, "simt") ? 2 : 0);
  env = getenv("MLDB_BRANCHES");
  if (env) h->branches = std::min(std::max(atoi(env), 1), (int)mldb_handle::MAX_BRANCHES);
  e = cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming);
  for (int i = 0; i < mldb_handle::MAX_BRANCHES - 1 && e == cudaSuccess; ++i) {
    e = cudaStreamCreateWithFlags(&h->br_stream[i], cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_join[i], cudaEventDisableTiming);
  }
  if (e != cudaSuccess) { mldb_destroy(h); FAIL(MLDB_ERR_CUDA, "branch streams: %s", cudaGetErrorString(e)); }
  for (int i = 0; i < mldb_handle::MAX_BRANCHES && e == cudaSuccess; ++i) {
    e = cudaMalloc((void**)&h->ffn_scratch[i], TC_FFN_SCRATCH_BYTES);
    if (e == cudaSuccess) e = cudaMalloc((void**)&h->ffn_flags[i], TC_FFN_FLAG_BYTES);
    if (e == cudaSuccess) e = cudaMemset(h->ffn_flags[i], 0, TC_FFN_FLAG_BYTES);
  }
  if (e != cudaSuccess) { mldb_destroy(h); FAIL(MLDB_ERR_CUDA, "ffn scratch: %s", cudaGetErrorString(e)); }
  env = getenv("MLDB_FFN_SPLIT");
  if (env) tc_set_ffn_split(h->tc, atoi(env) != 0);
  env = getenv("MLDB_FFN_FUSED");
  if (env) tc_set_ffn_fused(h->tc, atoi(env) != 0);
  *out = h;
  return MLDB_OK;
}

extern "C" void mldb_destroy(mldb_handle* h) {
  if (!h) return;
  DeviceGuard guard(h->device);
  cudaDeviceSynchronize();
  for (auto& kv : h->plans) {
    if (kv.second->exec) cudaGraphExecDestroy(kv.second->exec);
    delete kv.second;
  }
  for (void* p : h->allocs) cudaFree(p);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  for (int i = 0; i < mldb_handle::MAX_BRANCHES - 1; ++i) {
    if (h->br_stream[i]) cudaStreamDestroy(h->br_stream[i]);
    if (h->ev_join[i]) cudaEventDestroy(h->ev_join[i]);
  }
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  for (int i = 0; i < mldb_handle::MAX_BRANCHES; ++i) { cudaFree(h->ffn_scratch[i]); cudaFree(h->ffn_flags[i]); }
  mldb_comm_release(h);
  tc_destroy(h->tc);
  delete h;
}

extern "C" int mldb_set_option(mldb_handle* h, const char* name, const char* value) {
  if (!h || !name || !value) FAIL(MLDB_ERR_INVALID, "null argument");
  if (!strcmp(name, "gemm")) {
    if (!strcmp(value, "tc")) h->use_tc = true;
    else if (!strcmp(value, "simt")) h->use_tc = false;
    else FAIL(MLDB_ERR_INVALID, "gemm must be tc|simt");
  } else if (!strcmp(name, "ffn_fused")) {
    tc_set_ffn_fused(h->tc, atoi(value) != 0);
  } else if (!strcmp(name, "ffn_split")) {
    tc_set_ffn_split(h->tc, atoi(value) != 0);
  } else if (!strcmp(name, "attn")) {
    if (!strcmp(value, "tc")) h->attn_kind = 0;
    else if (!strcmp(value, "mma")) h->attn_kind = 1;
    else if (!strcmp(value, "simt")) h->attn_kind = 2;
    else FAIL(MLDB_ERR_INVALID, "attn must be tc|mma|simt");
  } else if (!strcmp(name, "branches")) {
    h->branches = std::min(std::max(atoi(value), 1), (int)mldb_handle::MAX_BRANCHES);
  } else if (!strcmp(name, "graph")) {
    h->use_graph = strcmp(value, "0") != 0;
  } else {
    FAIL(MLDB_ERR_INVALID, "unknown option %s", name);
  }
  // plans hold captured graphs of the previous configuration
  for (auto& kv : h->plans) {
    if (kv.second->exec) { cudaGraphExecDestroy(kv.second->exec); kv.second->exec = nullptr; }
  }
  return MLDB_OK;
}

extern "C" int64_t mldb_launch_count(const mldb_handle* h) { return h ? h->launches : 0; }

// ----------------------------------------------------------------------------- weights
extern "C" int mldb_load_tensor(mldb_handle* h, const char* key, const void* data,
                                const int64_t* shape, int32_t ndim, int32_t dtype) {
  if (!h || !key || !data || !shape) FAIL(MLDB_ERR_INVALID, "null argument");
  if (dtype != MLDB_DTYPE_F32) FAIL(MLDB_ERR_UNSUPPORTED, "only fp32 tensors are accepted");
  if (h->finalized) FAIL(MLDB_ERR_STATE, "weights already finalized");
  auto it = h->raw.find(key);
  if (it == h->raw.end()) {
    // ActorVae's encoder half is not on the sampling path: accept and ignore
    if (h->cfg.vae_kind == MLDB_VAE_ACTOR && !strncmp(key, "vae.encoder.", 12)) return MLDB_OK;
    FAIL(MLDB_ERR_INVALID, "unexpected state-dict key '%s'", key);
  }
  RawTensor& t = it->second;
  if ((int)t.shape.size() != ndim) FAIL(MLDB_ERR_INVALID, "key '%s': rank %d, expected %d", key, ndim, (int)t.shape.size());
  size_t n = 1;
  for (int i = 0; i < ndim; ++i) {
    if (shape[i] != t.shape[i]) FAIL(MLDB_ERR_INVALID, "key '%s': dim %d is %lld, expected %lld", key, i, (long long)shape[i], (long long)t.shape[i]);
    n *= (size_t)shape[i];
  }
  t.host.resize(n);
  DeviceGuard guard(h->device);
  CK(cudaMemcpy(t.host.data(), data, n * sizeof(float), cudaMemcpyDefault));
  t.loaded = true;
  return MLDB_OK;
}

extern "C" int mldb_finalize_weights(mldb_handle* h, void* stream) {
  (void)stream;
  if (!h) FAIL(MLDB_ERR_INVALID, "null handle");
  if (h->finalized) FAIL(MLDB_ERR_STATE, "already finalized");
  for (auto& kv : h->raw)
    if (!kv.second.loaded) FAIL(MLDB_ERR_STATE, "missing state-dict key '%s' (strict load)", kv.first.c_str());
  DeviceGuard guard(h->device);
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim;
  const std::string D = "denoiser.", V = "vae.";
  if (c.num_layers > 0) {
  TRY(pack_named(h, D + "time_embedding.linear_1.weight", D + "time_embedding.linear_1.bias", &h->time_l1));
  TRY(pack_named(h, D + "time_embedding.linear_2.weight", D + "time_embedding.linear_2.bias", &h->time_l2));
  if (c.cond_kind == MLDB_COND_TEXT) {
    if (c.text_dim != d) TRY(pack_named(h, D + "emb_proj.1.weight", D + "emb_proj.1.bias", &h->emb_proj));
  } else {
    TRY(upload_f32(h, rt(h, D + "emb_proj.action_embedding").host.data(), (size_t)c.nclasses * d, &h->action_emb));
  }
  TRY(upload_pe(h, D + "query_pos.pe", &h->query_pe));
  TRY(upload_pe(h, D + "mem_pos.pe", &h->mem_pe));
  if (c.diffusion_only) {
    TRY(pack_named(h, D + "pose_embd.weight", D + "pose_embd.bias", &h->pose_embd, 0, -1, true));
    TRY(pack_named(h, D + "pose_proj.weight", D + "pose_proj.bias", &h->pose_proj));
  }
  if (c.arch == MLDB_ARCH_TRANS_ENC) {
    TRY(pack_skip_stack(h, D + "encoder.", d, c.ff_size, c.num_heads, c.num_layers, false, &h->den));
  } else {
    h->den.kind = STACK_PLAIN_DEC; h->den.d = d; h->den.ff = c.ff_size; h->den.heads = c.num_heads;
    h->den.layers = c.num_layers;
    for (int i = 0; i < c.num_layers; ++i) {
      h->den.dec.emplace_back();
      TRY(pack_dec_layer(h, D + "decoder.layers." + std::to_string(i) + ".", d, &h->den.dec.back()));
    }
    TRY(pack_ln(h, D + "decoder.norm.", d, &h->den.norm));
  }
  }
  if (c.vae_kind == MLDB_VAE_MLD) {
    TRY(pack_skip_stack(h, V + "encoder.", d, c.vae_ff, c.vae_heads, c.vae_layers, false, &h->venc));
    TRY(pack_skip_stack(h, V + "decoder.", d, c.vae_ff, c.vae_heads, c.vae_layers, true, &h->vdec));
    TRY(upload_pe(h, V + "query_pos_decoder.pe", &h->vae_dec_pe, &h->vae_dec_pe_rows));
    TRY(upload_pe(h, V + "query_pos_encoder.pe", &h->vae_enc_pe));
    TRY(upload_f32(h, rt(h, V + "global_motion_token").host.data(), (size_t)2 * c.n_lat * d, &h->global_token));
    TRY(pack_named(h, V + "skel_embedding.weight", V + "skel_embedding.bias", &h->skel_emb, 0, -1, true));
    TRY(pack_named(h, V + "final_layer.weight", V + "final_layer.bias", &h->final_layer));
  } else if (c.vae_kind == MLDB_VAE_ACTOR) {
    h->vdec.kind = STACK_PLAIN_DEC; h->vdec.d = d; h->vdec.ff = c.vae_ff; h->vdec.heads = c.vae_heads;
    h->vdec.layers = c.vae_layers;
    for (int i = 0; i < c.vae_layers; ++i) {
      h->vdec.dec.emplace_back();
      TRY(pack_dec_layer(h, V + "decoder.seqTransDecoder.layers." + std::to_string(i) + ".", d, &h->vdec.dec.back()));
    }
    TRY(upload_pe(h, V + "decoder.sequence_pos_encoding.pe", &h->vae_dec_pe, &h->vae_dec_pe_rows));
    TRY(pack_named(h, V + "decoder.final_layer.weight", V + "decoder.final_layer.bias", &h->final_layer));
  }
  for (auto& kv : h->raw) { kv.second.host.clear(); kv.second.host.shrink_to_fit(); }
  h->finalized = true;
  return MLDB_OK;
}

extern "C" int mldb_set_mean_std(mldb_handle* h, const float* mean, const float* stdv, int32_t nfeats) {
  if (!h || !mean || !stdv || nfeats <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  DeviceGuard guard(h->device);
  if (!h->mean || h->nstat != nfeats) {
    TRY(dev_alloc(h, (void**)&h->mean, nfeats * sizeof(float)));
    TRY(dev_alloc(h, (void**)&h->stdv, nfeats * sizeof(float)));
    h->nstat = nfeats;
  }
  CK(cudaMemcpy(h->mean, mean, nfeats * sizeof(float), cudaMemcpyDefault));
  CK(cudaMemcpy(h->stdv, stdv, nfeats * sizeof(float), cudaMemcpyDefault));
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- scheduler API
// Time tokens for a list of timesteps: time_embedding(time_proj(t)) (mld_denoiser.py:151-155)
// + the positional row the token will occupy.  out [n, d] fp32.
static int time_tokens(mldb_handle* h, const int64_t* d_ts, int64_t t_scalar, int n, const float* pe_row,
                       float* out, float* scratch_feats, float* scratch_h, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim;
  const int tdim = c.cond_kind == MLDB_COND_TEXT ? c.text_dim : d;
  const int half = tdim / 2;
  k_timestep_features<<<(n * half + 255) / 256, 256, 0, st>>>(d_ts, t_scalar, n, tdim, c.flip_sin_to_cos, c.freq_shift, scratch_feats);
  kcount(h, MLDB_KSTAT_MISC);
  GemmArgs g; g.a_kind = A_F32; g.a_f32 = scratch_feats; g.lda = tdim; g.M = n; g.w = h->time_l1;
  g.act = ACT_SILU; g.out_f32 = scratch_h; g.ldc = d;
  simt_gemm(g, st); kcount(h, MLDB_KSTAT_GEMM_SIMT);
  GemmArgs g2; g2.a_kind = A_F32; g2.a_f32 = scratch_h; g2.lda = d; g2.M = n; g2.w = h->time_l2;
  g2.out_f32 = out; g2.ldc = d; g2.in_group = 1; g2.out_group = 1; g2.out_off = 0;
  // addtab row index is (out_off + r % in_group) = 0 -> pe_row
  g2.addtab = pe_row;
  simt_gemm(g2, st); kcount(h, MLDB_KSTAT_GEMM_SIMT);
  return MLDB_OK;
}

extern "C" int mldb_scheduler_set_timesteps(mldb_handle* h, int32_t n, int64_t* timesteps_out) {
  if (!h) FAIL(MLDB_ERR_INVALID, "null handle");
  if (!h->finalized) FAIL(MLDB_ERR_STATE, "finalize weights first");
  if (n <= 0 || n > h->cfg.num_train_timesteps) FAIL(MLDB_ERR_INVALID, "bad number of inference steps %d", n);
  DeviceGuard guard(h->device);
  const mldb_config& c = h->cfg;
  if ((int)h->timesteps.size() == n) {          // the reference calls set_timesteps before every reverse loop
    if (timesteps_out) memcpy(timesteps_out, h->timesteps.data(), n * sizeof(int64_t));
    return MLDB_OK;
  }
  std::vector<int64_t> ts(n);
  TRY(mldb_scheduler_timesteps(&c, n, ts.data()));
  for (int i = 0; i < n; ++i)
    if (ts[i] < 0 || ts[i] >= c.num_train_timesteps)
      FAIL(MLDB_ERR_INVALID, "timestep %lld is outside the %d training timesteps (steps_offset with n == num_train_timesteps)",
           (long long)ts[i], c.num_train_timesteps);
  h->timesteps = ts;
  h->coefs_host.resize(n);
  for (int i = 0; i < n; ++i) h->coefs_host[i] = make_coef(h, h->timesteps[i], n);
  const int d = c.latent_dim;
  const int tdim = c.cond_kind == MLDB_COND_TEXT ? c.text_dim : d;
  const int cap = c.num_train_timesteps;        // n <= cap: the tables are allocated once
  if (!h->d_timesteps) {
    TRY(dev_alloc(h, (void**)&h->d_timesteps, cap * sizeof(int64_t)));
    TRY(dev_alloc(h, (void**)&h->d_coefs, cap * sizeof(StepCoef)));
    TRY(dev_alloc(h, (void**)&h->d_tt, (size_t)cap * d * sizeof(float)));
    TRY(dev_alloc(h, (void**)&h->d_tfeats, (size_t)cap * tdim * sizeof(float)));
    TRY(dev_alloc(h, (void**)&h->d_thid, (size_t)cap * d * sizeof(float)));
  }
  CK(cudaMemcpy(h->d_timesteps, h->timesteps.data(), n * sizeof(int64_t), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->d_coefs, h->coefs_host.data(), n * sizeof(StepCoef), cudaMemcpyHostToDevice));
  if (c.num_layers == 0) {   // scheduler-only use (no denoiser loaded)
    h->sched_epoch++;
    if (timesteps_out) memcpy(timesteps_out, h->timesteps.data(), n * sizeof(int64_t));
    return MLDB_OK;
  }
  float *feats = h->d_tfeats, *hid = h->d_thid;
  // the time token sits at row n_lat of the encoder sequence (mld_denoiser.py:171,187) or at
  // row 0 of the decoder memory (mld_denoiser.py:215)
  const float* pe_row = c.arch == MLDB_ARCH_TRANS_ENC ? h->query_pe + (size_t)c.n_lat * d : h->mem_pe;
  TRY(time_tokens(h, h->d_timesteps, 0, n, pe_row, h->d_tt, feats, hid, h->cap_stream));
  CK(cudaStreamSynchronize(h->cap_stream));
  h->sched_epoch++;
  if (timesteps_out) memcpy(timesteps_out, h->timesteps.data(), n * sizeof(int64_t));
  return MLDB_OK;
}

extern "C" int mldb_scheduler_step(mldb_handle* h, const float* model_output, int64_t timestep,
                                   const float* sample, const float* noise, int64_t count,
                                   float* prev_sample, void* stream) {
  if (!h || !model_output || !sample || !prev_sample) FAIL(MLDB_ERR_INVALID, "null argument");
  if (h->timesteps.empty()) FAIL(MLDB_ERR_STATE, "call mldb_scheduler_set_timesteps first");
  if (timestep < 0 || timestep >= h->cfg.num_train_timesteps) FAIL(MLDB_ERR_INVALID, "timestep out of range");
  DeviceGuard guard(h->device);
  StepCoef k = make_coef(h, timestep, (int)h->timesteps.size());
  if (k.kind == 1 && k.sigma != 0.0f && !noise) FAIL(MLDB_ERR_INVALID, "DDPM step at t > 0 needs the injected noise tensor");
  k_sched_step<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(model_output, sample, noise, prev_sample, count, k);
  kcount(h, MLDB_KSTAT_MISC);
  CK(cudaGetLastError());
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- plans
static Plan* find_plan(mldb_handle* h, int kind, int B, int S, int T) {
  char key[64];
  snprintf(key, sizeof key, "%d:%d:%d:%d", kind, B, S, T);
  auto it = h->plans.find(key);
  return it == h->plans.end() ? nullptr : it->second;
}
static Plan* add_plan(mldb_handle* h, int kind, int B, int S, int T) {
  char key[64];
  snprintf(key, sizeof key, "%d:%d:%d:%d", kind, B, S, T);
  Plan* p = new Plan();
  p->kind = kind; p->B = B; p->S = S; p->T = T;
  h->plans[key] = p;
  return p;
}

// an operator could not be enqueued (its tensor maps could not be encoded): the output is unwritten,
// so the call must not report success (mldb_last_error() holds the encoder's message)
static int check_ops(mldb_handle* h) {
  if (!h->op_failed) return MLDB_OK;
  h->op_failed = false;
  return MLDB_ERR_CUDA;
}

// Run `record` either directly on `st` or as a (cached) CUDA graph.
template <typename F>
static int run_graphed(mldb_handle* h, Plan* p, cudaStream_t st, F record) {
  if (!h->use_graph) { record(st); CK(cudaGetLastError()); return check_ops(h); }
  if (!p->exec || p->sched_epoch != h->sched_epoch) {
    if (p->exec) { cudaGraphExecDestroy(p->exec); p->exec = nullptr; }
    cudaGraph_t graph = nullptr;
    h->capturing = true; h->capture_nodes = 0;
    cudaError_t e = cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal);
    if (e == cudaSuccess) {
      record(h->cap_stream);
      e = cudaStreamEndCapture(h->cap_stream, &graph);
    }
    h->capturing = false;
    if (e != cudaSuccess) FAIL(MLDB_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
    if (h->op_failed) { cudaGraphDestroy(graph); return check_ops(h); }
    e = cudaGraphInstantiate(&p->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) FAIL(MLDB_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(e));
    p->graph_nodes = h->capture_nodes;
    p->sched_epoch = h->sched_epoch;
  }
  CK(cudaGraphLaunch(p->exec, st));
  h->launches += p->graph_nodes;
  return MLDB_OK;
}


// ----------------------------------------------------------------------------- denoiser (trans_enc)
// Gather + place the action tokens (EmbedAction.forward, mld_denoiser.py:250-262): rows of the
// first (uncond) half are zero when guidance is on.
__global__ void k_action_tokens(ActBuf X, int Ntok, int Bx, int pos, int d, const int64_t* __restrict__ ids,
                                const float* __restrict__ table, int nclasses, int cfg_on,
                                const float* __restrict__ pe_row) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)Bx * d) return;
  const int n = (int)(idx % d), s = (int)(idx / d);
  float v = 0.0f;
  if (!(cfg_on && s < Bx / 2)) {
    int64_t id = ids[s];
    id = id < 0 ? 0 : (id >= nclasses ? nclasses - 1 : id);
    v = table[id * d + n];
  }
  v += pe_row[n];
  __half hh, ll;
  split_f32(v, hh, ll);
  const int64_t o = ((int64_t)s * Ntok + pos) * X.cols + n;
  X.hi[o] = hh;
  X.lo()[o] = ll;
}

static int enc_plan(mldb_handle* h, int kind, int B, int Bx, int S, Plan** out) {
  Plan* p = find_plan(h, kind, B, S, 0);
  if (!p) {
    const mldb_config& c = h->cfg;
    p = add_plan(h, kind, B, S, 0);
    p->Bx = Bx;
    const int Sc = c.cond_kind == MLDB_COND_TEXT ? S : 1;
    p->Ntok = c.n_lat + 1 + Sc;
    if (p->Ntok > 500) FAIL(MLDB_ERR_INVALID, "sequence of %d tokens exceeds the learned PE table (500)", p->Ntok);
    TRY(alloc_stack_ws(h, h->den, Bx, p->Ntok, 0, &p->ws, h->den.layers >= 3 ? c.n_lat : 0));
    const size_t per = (size_t)c.n_lat * c.latent_dim;
    TRY(dev_alloc(h, (void**)&p->latents, (size_t)B * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->eps, (size_t)Bx * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->tt_single, (size_t)3 * std::max(c.text_dim, c.latent_dim) * sizeof(float) + 64));
    if (c.cond_kind == MLDB_COND_TEXT && c.text_dim != c.latent_dim)
      TRY(alloc_act(h, Bx * S, c.text_dim, &p->ctx_split));
  }
  *out = p;
  return MLDB_OK;
}

// condition tokens -> X0 (once per batch; step invariant, hoisted out of the loop although the
// reference recomputes emb_proj every step, mld_denoiser.py:165)
// fp32 rows -> split16 rows (+ table row, ReLU) with the (seq, pos) mapping of k_rows_to_split; the
// 128-bit path whenever the shapes allow it
static void rows_to_split(mldb_handle* h, ActBuf X, const float* src, int ld_src, int M, int d, int in_group,
                          int out_group, int out_off, int src_bcast, const float* tab, int relu, cudaStream_t st) {
  const bool vec = d % 8 == 0 && X.cols % 8 == 0 && (!src || (ld_src % 4 == 0 && ((uintptr_t)src & 15) == 0)) &&
                   (!tab || ((uintptr_t)tab & 15) == 0) && ((uintptr_t)X.hi & 15) == 0 && X.plane_stride % 8 == 0;
  if (vec)
    k_rows_to_split8<<<nblk((int64_t)M * (d / 8)), 256, 0, st>>>(X, src, ld_src, M, d, in_group, out_group, out_off,
                                                                 src_bcast, tab, relu);
  else
    k_rows_to_split<<<nblk((int64_t)M * d), 256, 0, st>>>(X, src, ld_src, M, d, in_group, out_group, out_off, src_bcast,
                                                          tab, relu);
  kcount(h, MLDB_KSTAT_MISC);
}

static int place_condition(mldb_handle* h, Plan* p, const void* cond, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim, Bx = p->Bx;
  if (c.cond_kind == MLDB_COND_TEXT) {
    const int S = p->S;
    if (c.text_dim != d) {
      // emb_proj = ReLU -> Linear (mld_denoiser.py:67-68): ReLU + hi/lo split in one pass over the
      // CLIP context, then the tensor-core GEMM writes the tokens (+ PE) straight into X0
      GemmArgs g; g.M = Bx * S; g.w = h->emb_proj; g.out = p->ws.x0;
      g.in_group = S; g.out_group = p->Ntok; g.out_off = c.n_lat + 1; g.addtab = h->query_pe;
      if (h->use_tc && p->ctx_split.hi && c.text_dim % 64 == 0) {
        rows_to_split(h, p->ctx_split, (const float*)cond, c.text_dim, Bx * S, c.text_dim, 1 << 30, 0, 0, 0, nullptr, 1, st);
        g.a1 = p->ctx_split; g.K1 = c.text_dim;
      } else {
        g.a_kind = A_F32_RELU; g.a_f32 = (const float*)cond; g.lda = c.text_dim;
      }
      op_gemm(h, g, st);
    } else {
      rows_to_split(h, p->ws.x0, (const float*)cond, d, Bx * S, d, S, p->Ntok, c.n_lat + 1, 0, h->query_pe, 0, st);
    }
  } else {
    const int cfg_on = c.guidance_scale > 1.0f;
    k_action_tokens<<<nblk((int64_t)Bx * d), 256, 0, st>>>(p->ws.x0, p->Ntok, Bx, c.n_lat + 1, d, (const int64_t*)cond,
                                                          h->action_emb, c.nclasses, cfg_on,
                                                          h->query_pe + (size_t)(c.n_lat + 1) * d);
    kcount(h, MLDB_KSTAT_MISC);
  }
  CK(cudaGetLastError());
  return MLDB_OK;
}

// the stack + final norm over the n sequences of workspace (slice) wsv: eps[n, n_lat*d]
static void denoiser_range(mldb_handle* h, Plan* p, const StackWs& wsv, int n, float* eps, cudaStream_t s) {
  const mldb_config& c = h->cfg;
  SeqInfo si;
  StackWs w = wsv;
  ActBuf x = run_stack(h, h->den, w.x0, ActBuf{}, w, si, s);
  // encoder.norm on the latent tokens only (cross_attention.py:62-63, mld_denoiser.py:206)
  LnArgs l; l.res = x; l.gamma = h->den.norm.g; l.beta = h->den.norm.b; l.M = n * c.n_lat; l.d = c.latent_dim;
  if (w.n_sel == 0) { l.sel_group = c.n_lat; l.in_group = p->Ntok; }   // else x is already compact
  l.out_f32 = eps; l.ld_out = c.latent_dim;
  op_ln(h, l, s);
}

// one denoiser pass over the assembled tokens: eps[Bx, n_lat*d] = norm(stack(X0))[:n_lat]
static void denoiser_pass(mldb_handle* h, Plan* p, const float* latents, int lat_mod, const float* tt,
                          float* eps_out, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim;
  launch_pdl(k_assemble_tokens, dim3(nblk((int64_t)p->Bx * (c.n_lat + 1) * d)), dim3(256), 0, st,
             p->ws.x0, p->Ntok, p->Bx, lat_mod, c.n_lat, d, latents, (const float*)h->query_pe, tt);
  kcount(h, MLDB_KSTAT_MISC);
  // Sequences are independent: the stack runs as `branches` contiguous sequence ranges with their own
  // workspace rows on parallel streams (parallel chains inside the captured graph).
  const int nbr = (h->branches > 1 && p->Bx * p->Ntok >= 2 * 128 * h->branches) ? h->branches : 1;
  if (nbr == 1) {
    denoiser_range(h, p, p->ws, p->Bx, eps_out, st);
    return;
  }
  // fork: every range waits for the token assembly; join: the caller's stream waits for every range
  cudaEventRecord(h->ev_fork, st);
  for (int k = 0; k < nbr; ++k) {
    cudaStream_t s = k == 0 ? st : h->br_stream[k - 1];
    if (k) cudaStreamWaitEvent(s, h->ev_fork, 0);
    const int s0 = (int)((int64_t)p->Bx * k / nbr), s1 = (int)((int64_t)p->Bx * (k + 1) / nbr);
    denoiser_range(h, p, ws_slice(p->ws, s0, s1 - s0), s1 - s0, eps_out + (size_t)s0 * c.n_lat * d, s);
    if (k) cudaEventRecord(h->ev_join[k - 1], s);
  }
  for (int k = 1; k < nbr; ++k) cudaStreamWaitEvent(st, h->ev_join[k - 1], 0);
}

// ----------------------------------------------------------------------------- denoiser (trans_dec)
// The no-VAE model (configs/modules_novae/denoiser.yaml): frames are the decoder targets, the
// memory is [time, text...] (mld_denoiser.py:208-221).  No key-padding mask is passed on either
// attention (padded frames attend and are attended, like the reference); padded output frames are
// zeroed after pose_proj (:219-221).
static int decden_plan(mldb_handle* h, int kind, int B, int Bx, int S, int T, Plan** out) {
  Plan* p = find_plan(h, kind, B, S, T);
  if (!p) {
    const mldb_config& c = h->cfg;
    if (T > 500 || 1 + S > 500) FAIL(MLDB_ERR_INVALID, "sequence exceeds the learned PE table (500)");
    p = add_plan(h, kind, B, S, T);
    p->Bx = Bx;
    p->Ntok = T;
    const int Lmem = 1 + (c.cond_kind == MLDB_COND_TEXT ? S : 1);
    TRY(alloc_stack_ws(h, h->den, Bx, T, Lmem, &p->ws));
    TRY(alloc_act(h, Bx * Lmem, c.latent_dim, &p->mem));
    const size_t per = (size_t)T * c.nfeats;
    TRY(dev_alloc(h, (void**)&p->latents, (size_t)B * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->eps, (size_t)Bx * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->stage_f32, (size_t)Bx * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->lengths, (size_t)Bx * sizeof(int32_t)));
    TRY(dev_alloc(h, (void**)&p->tt_single, (size_t)3 * std::max(c.text_dim, c.latent_dim) * sizeof(float) + 64));
    TRY(dev_alloc(h, (void**)&p->d_step, sizeof(int)));
    if (h->pose_embd.K % 64 == 0 && h->pose_embd.K >= c.nfeats) TRY(alloc_act(h, Bx * T, h->pose_embd.K, &p->in_split));
  }
  *out = p;
  return MLDB_OK;
}

static int place_condition_dec(mldb_handle* h, Plan* p, const void* cond, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim, Bx = p->Bx, Lmem = p->ws.Lmem;
  if (c.cond_kind == MLDB_COND_TEXT) {
    const int S = p->S;
    if (c.text_dim != d) {
      GemmArgs g; g.a_kind = A_F32_RELU; g.a_f32 = (const float*)cond; g.lda = c.text_dim;
      g.M = Bx * S; g.w = h->emb_proj; g.out = p->mem;
      g.in_group = S; g.out_group = Lmem; g.out_off = 1; g.addtab = h->mem_pe;
      op_gemm(h, g, st);
    } else {
      rows_to_split(h, p->mem, (const float*)cond, d, Bx * S, d, S, Lmem, 1, 0, h->mem_pe, 0, st);
    }
  } else {
    const int cfg_on = c.guidance_scale > 1.0f;
    k_action_tokens<<<nblk((int64_t)Bx * d), 256, 0, st>>>(p->mem, Lmem, Bx, 1, d, (const int64_t*)cond, h->action_emb,
                                                          c.nclasses, cfg_on, h->mem_pe + (size_t)d);
    kcount(h, MLDB_KSTAT_MISC);
  }
  CK(cudaGetLastError());
  return MLDB_OK;
}

// model_in: [rows_in, T, F] fp32 (device) fed `rep` times (rep * rows_in == Bx: torch.cat([latents] * 2),
// mld.py:325); lengths: device int32[Bx]; eps_out [Bx, T, F].  tt: time token(s); step_ptr != null selects
// row *step_ptr of tt (replayed step graph).
static void denoiser_pass_dec(mldb_handle* h, Plan* p, const float* model_in, int rep, const float* tt,
                              const int* step_ptr, float* eps_out, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim, Bx = p->Bx, T = p->T, F = c.nfeats, Lmem = p->ws.Lmem;
  // memory row 0 = time token (mem_pos.pe[0] already added)
  k_rows_to_split<<<nblk((int64_t)Bx * d), 256, 0, st>>>(p->mem, tt, d, Bx, d, 1, Lmem, 0, 1, nullptr, 0, step_ptr, (int64_t)d);
  kcount(h, MLDB_KSTAT_MISC);
  // pose_embd + query_pos (mld_denoiser.py:210,214): the 263 features zero-padded to the packed K (320)
  // so that the embedding runs on the tensor cores
  GemmArgs g; g.M = Bx * T; g.w = h->pose_embd;
  g.out = p->ws.x0; g.in_group = T; g.out_group = T; g.out_off = 0; g.addtab = h->query_pe;
  if (h->use_tc && p->in_split.hi) {
    k_f32_to_split_pad<<<nblk((int64_t)(Bx / rep) * T * p->in_split.cols), 256, 0, st>>>(p->in_split, model_in, F, (Bx / rep) * T, F, rep);
    kcount(h, MLDB_KSTAT_MISC);
    g.a1 = p->in_split; g.K1 = p->in_split.cols;
  } else {
    if (rep > 1) {   // CUDA-core reference path: materialise the duplicated input
      for (int k = 0; k < rep; ++k)
        cudaMemcpyAsync(p->stage_f32 + (size_t)k * (Bx / rep) * T * F, model_in, (size_t)(Bx / rep) * T * F * sizeof(float),
                        cudaMemcpyDeviceToDevice, st);
      model_in = p->stage_f32;
    }
    g.a_kind = A_F32; g.a_f32 = model_in; g.lda = F;
  }
  op_gemm(h, g, st);
  SeqInfo si;
  ActBuf x = run_stack(h, h->den, p->ws.x0, p->mem, p->ws, si, st);
  LnArgs l; l.res = x; l.gamma = h->den.norm.g; l.beta = h->den.norm.b; l.M = Bx * T; l.d = d; l.out = p->ws.x1;
  op_ln(h, l, st);
  GemmArgs go; go.a1 = p->ws.x1; go.K1 = d; go.M = Bx * T; go.w = h->pose_proj; go.out_f32 = eps_out; go.ldc = F;
  go.in_group = T; go.out_group = T; go.out_off = 0; go.zero_lengths = p->lengths;
  op_gemm(h, go, st);
}

__global__ void k_dup_lengths(const int32_t* __restrict__ src, int32_t* __restrict__ dst, int B, int Bx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Bx) dst[i] = src[i % B];
}

static int check_ready(mldb_handle* h, bool need_sched) {
  if (!h) FAIL(MLDB_ERR_INVALID, "null handle");
  if (!h->finalized) FAIL(MLDB_ERR_STATE, "weights not finalized");
  if (need_sched && h->timesteps.empty()) FAIL(MLDB_ERR_STATE, "call mldb_scheduler_set_timesteps first");
  return MLDB_OK;
}

extern "C" int mldb_denoise(mldb_handle* h, const float* sample, int64_t timestep, const void* cond,
                            const int32_t* lengths, int32_t Bx, int32_t S_ctx, int32_t T, float* out,
                            void* stream) {
  (void)lengths; (void)T;
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!sample || !cond || !out || Bx <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  const mldb_config& c = h->cfg;
  if (c.num_layers == 0) FAIL(MLDB_ERR_STATE, "this handle has no denoiser");
  if (c.cond_kind == MLDB_COND_TEXT && S_ctx <= 0) FAIL(MLDB_ERR_INVALID, "S_ctx must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  Plan* p = nullptr;
  if (c.arch == MLDB_ARCH_TRANS_DEC) {
    if (!c.diffusion_only) FAIL(MLDB_ERR_UNSUPPORTED, "arch trans_dec is built for the no-VAE model (diffusion_only)");
    if (!lengths || T <= 0) FAIL(MLDB_ERR_INVALID, "the no-VAE denoiser needs lengths and T");
    TRY(decden_plan(h, 4, Bx, Bx, S_ctx, T, &p));
    TRY(place_condition_dec(h, p, cond, st));
    CK(cudaMemcpyAsync(p->lengths, lengths, (size_t)Bx * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    const int d = c.latent_dim;
    const int tdim = c.cond_kind == MLDB_COND_TEXT ? c.text_dim : d;
    float* feats = p->tt_single + 16;
    float* hid = feats + tdim;
    float* tt = hid + std::max(tdim, d);
    TRY(time_tokens(h, nullptr, timestep, 1, h->mem_pe, tt, feats, hid, st));
    denoiser_pass_dec(h, p, sample, 1, tt, nullptr, out, st);
    CK(cudaGetLastError());
    return MLDB_OK;
  }
  TRY(enc_plan(h, 3, Bx, Bx, S_ctx, &p));
  TRY(place_condition(h, p, cond, st));
  // time token for this timestep
  const int d = c.latent_dim;
  const int tdim = c.cond_kind == MLDB_COND_TEXT ? c.text_dim : d;
  float* feats = p->tt_single + 16;
  float* hid = feats + tdim;
  float* tt = hid + std::max(tdim, d);
  TRY(time_tokens(h, nullptr, timestep, 1, h->query_pe + (size_t)c.n_lat * d, tt, feats, hid, st));
  denoiser_pass(h, p, sample, Bx, tt, out, st);
  CK(cudaGetLastError());
  return MLDB_OK;
}

static int run_reverse(mldb_handle* h, const void* cond, const float* init_noise, const float* step_noise,
                       const int32_t* lengths, int B, int S, int T, float* latents_out, cudaStream_t st,
                       Plan** plan_out) {
  const mldb_config& c = h->cfg;
  if (c.num_layers == 0) FAIL(MLDB_ERR_STATE, "this handle has no denoiser");
  const bool cfg_on = c.guidance_scale > 1.0f;
  const int Bx = cfg_on ? 2 * B : B;
  if (c.arch == MLDB_ARCH_TRANS_DEC) {
    // no-VAE model: latents are the motion itself, [B, T, F]; DDPM draws noise every step, which
    // the caller injects (step_noise [n_steps, B, T, F]).  Eager loop: 1000 big steps, no graph.
    if (!c.diffusion_only) FAIL(MLDB_ERR_UNSUPPORTED, "arch trans_dec is built for the no-VAE model (diffusion_only)");
    if (!lengths || T <= 0) FAIL(MLDB_ERR_INVALID, "the no-VAE model needs lengths and T");
    Plan* p = nullptr;
    TRY(decden_plan(h, 5, B, Bx, S, T, &p));
    const int64_t per = (int64_t)T * c.nfeats;
    TRY(place_condition_dec(h, p, cond, st));
    k_dup_lengths<<<nblk(Bx), 256, 0, st>>>(lengths, p->lengths, B, Bx);
    kcount(h, MLDB_KSTAT_MISC);
    CK(cudaMemcpyAsync(p->latents, init_noise, (size_t)B * per * sizeof(float), cudaMemcpyDeviceToDevice, st));
    const int nsteps = (int)h->timesteps.size();
    bool needs_noise = false;
    for (int i = 0; i < nsteps; ++i) needs_noise |= h->coefs_host[i].kind == 1 && h->coefs_host[i].sigma != 0.0f;
    if (needs_noise && !step_noise) FAIL(MLDB_ERR_INVALID, "DDPM needs step_noise [n_steps, B, T, F]");
    // ONE captured step, replayed n_steps times: the step index lives on the device (k_step_inc), the
    // kernels that depend on it (time token, scheduler coefficients, noise slice) read it through p->d_step.
    // The graph holds the caller's noise pointer: a different buffer re-captures.
    if (p->noise_ptr != step_noise && p->exec) { cudaGraphExecDestroy(p->exec); p->exec = nullptr; }
    p->noise_ptr = step_noise;
    k_step_set<<<1, 1, 0, st>>>(p->d_step, 0);
    kcount(h, MLDB_KSTAT_MISC);
    for (int i = 0; i < nsteps; ++i) {
      TRY(run_graphed(h, p, st, [&](cudaStream_t s) {
        denoiser_pass_dec(h, p, p->latents, cfg_on ? 2 : 1, h->d_tt, p->d_step, p->eps, s);
        k_cfg_sched<<<nblk(B * per), 256, 0, s>>>(p->eps, p->latents, needs_noise ? step_noise : nullptr, B * per,
                                                cfg_on ? 1 : 0, c.guidance_scale, h->d_coefs, 0, p->d_step);
        kcount(h, MLDB_KSTAT_MISC);
        k_step_inc<<<1, 1, 0, s>>>(p->d_step);
        kcount(h, MLDB_KSTAT_MISC);
      }));
    }
    if (latents_out) {                                        // [T, B, F] (mld.py:359)
      k_permute_01<<<nblk(B * per), 256, 0, st>>>(p->latents, latents_out, B, T, c.nfeats);
      kcount(h, MLDB_KSTAT_MISC);
    }
    CK(cudaGetLastError());
    if (plan_out) *plan_out = p;
    return MLDB_OK;
  }
  Plan* p = nullptr;
  TRY(enc_plan(h, 0, B, Bx, S, &p));
  const int d = c.latent_dim;
  const int64_t per = (int64_t)c.n_lat * d;
  TRY(place_condition(h, p, cond, st));
  // latents = init_noise * init_noise_sigma (== 1 for DDIM/DDPM), mld.py:310
  CK(cudaMemcpyAsync(p->latents, init_noise, (size_t)B * per * sizeof(float), cudaMemcpyDeviceToDevice, st));
  const int nsteps = (int)h->timesteps.size();
  // DDPM draws noise at every step with t > 0 (diffusers DDPMScheduler.step): the caller injects it
  const float* nz_all = nullptr;
  bool needs_noise = false;
  for (int i = 0; i < nsteps; ++i) needs_noise |= h->coefs_host[i].kind == 1 && h->coefs_host[i].sigma != 0.0f;
  if (needs_noise) {
    if (!step_noise) FAIL(MLDB_ERR_INVALID, "the DDPM scheduler needs step_noise [n_steps, B, n_lat, d] (injected N(0,1) per step)");
    if (p->noise_cap < (size_t)nsteps * B * per) {
      TRY(dev_alloc(h, (void**)&p->step_noise, (size_t)nsteps * B * per * sizeof(float)));
      p->noise_cap = (size_t)nsteps * B * per;
      if (p->exec) { cudaGraphExecDestroy(p->exec); p->exec = nullptr; }   // the graph holds the old pointer
    }
    CK(cudaMemcpyAsync(p->step_noise, step_noise, (size_t)nsteps * B * per * sizeof(float), cudaMemcpyDeviceToDevice, st));
    nz_all = p->step_noise;
  }
  TRY(run_graphed(h, p, st, [&](cudaStream_t s) {
    for (int i = 0; i < nsteps; ++i) {                                           // mld.py:323
      denoiser_pass(h, p, p->latents, B, h->d_tt + (size_t)i * d, p->eps, s);
      launch_pdl(k_cfg_sched, dim3(nblk(B * per)), dim3(256), 0, s, (const float*)p->eps, p->latents,
                 nz_all, (int64_t)(B * per), cfg_on ? 1 : 0, c.guidance_scale, (const StepCoef*)h->d_coefs, i,
                 (const int*)nullptr);
      kcount(h, MLDB_KSTAT_MISC);
    }
  }));
  if (latents_out) {                                                             // mld.py:359
    k_permute_01<<<nblk(B * per), 256, 0, st>>>(p->latents, latents_out, B, c.n_lat, d);
    kcount(h, MLDB_KSTAT_MISC);
  }
  CK(cudaGetLastError());
  if (plan_out) *plan_out = p;
  return MLDB_OK;
}

extern "C" int mldb_diffusion_reverse(mldb_handle* h, const void* cond, const float* init_noise,
                                      const float* step_noise, const int32_t* lengths, int32_t B,
                                      int32_t S_ctx, int32_t T, float* latents_out, void* stream) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!cond || !init_noise || !latents_out || B <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  return run_reverse(h, cond, init_noise, step_noise, lengths, B, S_ctx, T, latents_out, (cudaStream_t)stream, nullptr);
}

// ----------------------------------------------------------------------------- VAE decode
// z rows: [n_lat, B, d] fp32 -> memory tokens split [B * n_lat, d] (row = b * n_lat + j)
__global__ void k_mem_tokens(ActBuf mem, const float* __restrict__ z, int n_lat, int B, int d) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_lat * B * d) return;
  const int n = (int)(idx % d);
  const int b = (int)((idx / d) % B);
  const int j = (int)(idx / ((int64_t)d * B));
  __half hh, ll;
  split_f32(z[idx], hh, ll);
  const int64_t o = ((int64_t)b * n_lat + j) * mem.cols + n;
  mem.hi[o] = hh;
  mem.lo()[o] = ll;
}

static int dec_plan(mldb_handle* h, int B, int T, Plan** out) {
  Plan* p = find_plan(h, 1, B, 0, T);
  if (!p) {
    const mldb_config& c = h->cfg;
    if (T > h->vae_dec_pe_rows) FAIL(MLDB_ERR_INVALID, "T=%d exceeds the positional table (%d rows)", T, h->vae_dec_pe_rows);
    p = add_plan(h, 1, B, 0, T);
    TRY(alloc_stack_ws(h, h->vdec, B, T, c.n_lat, &p->ws));
    TRY(alloc_act(h, B * c.n_lat, c.latent_dim, &p->mem));
    TRY(dev_alloc(h, (void**)&p->lengths, (size_t)B * sizeof(int32_t)));
    TRY(dev_alloc(h, (void**)&p->feats, (size_t)B * T * c.vae_nfeats * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->joints, (size_t)B * T * c.njoints * 3 * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->latents, (size_t)B * c.n_lat * c.latent_dim * sizeof(float)));
  }
  *out = p;
  return MLDB_OK;
}

// z_is_plan_latents: z already sits in [n_lat,B,d] order in a device buffer
static int run_decode(mldb_handle* h, const float* z, const int32_t* lengths, int B, int T,
                      float* feats_out, cudaStream_t st, Plan** plan_out) {
  const mldb_config& c = h->cfg;
  if (c.vae_kind == MLDB_VAE_NONE) FAIL(MLDB_ERR_STATE, "no VAE configured");
  Plan* p = nullptr;
  TRY(dec_plan(h, B, T, &p));
  const int d = c.latent_dim, F = c.vae_nfeats;
  CK(cudaMemcpyAsync(p->lengths, lengths, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(p->latents, z, (size_t)B * c.n_lat * d * sizeof(float), cudaMemcpyDeviceToDevice, st));
  float* fout = feats_out ? feats_out : p->feats;
  TRY(run_graphed(h, p, st, [&](cudaStream_t s) {
    k_mem_tokens<<<nblk((int64_t)c.n_lat * B * d), 256, 0, s>>>(p->mem, p->latents, c.n_lat, B, d);
    kcount(h, MLDB_KSTAT_MISC);
    // queries = zeros + PE rows (mld_vae.py:190,224; actor_vae.py:219-225)
    rows_to_split(h, p->ws.x0, nullptr, 0, B * T, d, T, T, 0, 0, h->vae_dec_pe, 0, s);
    SeqInfo si; si.lengths = p->lengths; si.kv_prefix = 0;
    ActBuf x = run_stack(h, h->vdec, p->ws.x0, p->mem, p->ws, si, s);
    if (h->vdec.norm.g) {
      LnArgs l; l.res = x; l.gamma = h->vdec.norm.g; l.beta = h->vdec.norm.b; l.M = B * T; l.d = d; l.out = p->ws.x1;
      op_ln(h, l, s);
      x = p->ws.x1;
    }
    // final_layer + output[~mask.T] = 0 (mld_vae.py:243-245); rows are already [B, T]
    GemmArgs g; g.a1 = x; g.K1 = d; g.M = B * T; g.w = h->final_layer; g.out_f32 = p->feats; g.ldc = F;
    g.in_group = T; g.out_group = T; g.out_off = 0; g.zero_lengths = p->lengths;
    op_gemm(h, g, s);
  }));
  if (fout != p->feats)
    CK(cudaMemcpyAsync(fout, p->feats, (size_t)B * T * F * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (plan_out) *plan_out = p;
  return MLDB_OK;
}

extern "C" int mldb_vae_decode(mldb_handle* h, const float* z, const int32_t* lengths, int32_t B,
                               int32_t T, float* feats_out, void* stream) {
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!z || !lengths || !feats_out || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  return run_decode(h, z, lengths, B, T, feats_out, (cudaStream_t)stream, nullptr);
}

// ----------------------------------------------------------------------------- VAE encode
__global__ void k_rows_out_permuted(const float* __restrict__ src, float* __restrict__ mu, float* __restrict__ logvar,
                                    int B, int n_lat, int d) {
  // src rows (b, j) j < 2*n_lat -> mu[j, b, :] (j < n_lat) / logvar[j - n_lat, b, :]
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)B * 2 * n_lat * d) return;
  const int n = (int)(idx % d);
  const int j = (int)((idx / d) % (2 * n_lat));
  const int b = (int)(idx / ((int64_t)d * 2 * n_lat));
  if (j < n_lat) mu[((int64_t)j * B + b) * d + n] = src[idx];
  else logvar[((int64_t)(j - n_lat) * B + b) * d + n] = src[idx];
}

extern "C" int mldb_vae_encode(mldb_handle* h, const float* feats, const int32_t* lengths, int32_t B,
                               int32_t T, float* mu, float* logvar, void* stream) {
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!feats || !lengths || !mu || !logvar || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  const mldb_config& c = h->cfg;
  if (c.vae_kind != MLDB_VAE_MLD) FAIL(MLDB_ERR_UNSUPPORTED, "encode is built for MldVae only");
  cudaStream_t st = (cudaStream_t)stream;
  const int d = c.latent_dim, G = 2 * c.n_lat, L = G + T;
  if (L > 500) FAIL(MLDB_ERR_INVALID, "sequence too long for the learned PE table");
  Plan* p = find_plan(h, 2, B, 0, T);
  if (!p) {
    p = add_plan(h, 2, B, 0, T);
    TRY(alloc_stack_ws(h, h->venc, B, L, 0, &p->ws, h->venc.layers >= 3 ? G : 0));
    TRY(dev_alloc(h, (void**)&p->lengths, (size_t)B * sizeof(int32_t)));
    TRY(dev_alloc(h, (void**)&p->stage_f32, (size_t)B * G * d * sizeof(float)));
    if (h->skel_emb.K % 64 == 0) TRY(alloc_act(h, B * T, h->skel_emb.K, &p->in_split));
  }
  CK(cudaMemcpyAsync(p->lengths, lengths, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  // skel_embedding rows -> token rows (b, G + t) + PE (mld_vae.py:139-161); the 263 features are
  // zero-padded to the packed K so that the embedding runs on the tensor cores
  GemmArgs g; g.M = B * T; g.w = h->skel_emb;
  g.out = p->ws.x0; g.in_group = T; g.out_group = L; g.out_off = G; g.addtab = h->vae_enc_pe;
  if (h->use_tc && p->in_split.hi) {
    k_f32_to_split_pad<<<nblk((int64_t)B * T * p->in_split.cols), 256, 0, st>>>(p->in_split, feats, c.vae_nfeats, B * T, c.vae_nfeats, 1);
    kcount(h, MLDB_KSTAT_MISC);
    g.a1 = p->in_split; g.K1 = p->in_split.cols;
  } else {
    g.a_kind = A_F32; g.a_f32 = feats; g.lda = c.vae_nfeats;
  }
  op_gemm(h, g, st);
  // global motion tokens (b, 0..G-1) = token + PE (mld_vae.py:146,157)
  k_rows_to_split<<<nblk((int64_t)B * G * d), 256, 0, st>>>(p->ws.x0, h->global_token, d, B * G, d, G, L, 0, 1, h->vae_enc_pe);
  kcount(h, MLDB_KSTAT_MISC);
  SeqInfo si; si.lengths = p->lengths; si.kv_prefix = G;
  ActBuf x = run_stack(h, h->venc, p->ws.x0, ActBuf{}, p->ws, si, st);
  LnArgs l; l.res = x; l.gamma = h->venc.norm.g; l.beta = h->venc.norm.b; l.M = B * G; l.d = d;
  if (p->ws.n_sel == 0) { l.sel_group = G; l.in_group = L; }
  l.out_f32 = p->stage_f32; l.ld_out = d;
  op_ln(h, l, st);
  k_rows_out_permuted<<<nblk((int64_t)B * G * d), 256, 0, st>>>(p->stage_f32, mu, logvar, B, c.n_lat, d);
  kcount(h, MLDB_KSTAT_MISC);
  CK(cudaGetLastError());
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- feats2joints
static int run_f2j(mldb_handle* h, const float* feats, int B, int T, float* joints, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int F = c.vae_kind != MLDB_VAE_NONE ? c.vae_nfeats : c.nfeats;
  if (!h->mean || h->nstat != F) FAIL(MLDB_ERR_STATE, "call mldb_set_mean_std with %d features first", F);
  if (F < 4 + (c.njoints - 1) * 3) FAIL(MLDB_ERR_UNSUPPORTED, "feats2joints needs the HumanML3D/KIT layout");
  k_feats2joints<<<B, 256, (size_t)4 * T * sizeof(float), st>>>(feats, h->mean, h->stdv, T, F, c.njoints, joints);
  kcount(h, MLDB_KSTAT_MISC);
  CK(cudaGetLastError());
  return MLDB_OK;
}
extern "C" int mldb_feats2joints(mldb_handle* h, const float* feats, int32_t B, int32_t T,
                                 float* joints_out, void* stream) {
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!feats || !joints_out || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  return run_f2j(h, feats, B, T, joints_out, (cudaStream_t)stream);
}

// ----------------------------------------------------------------------------- full sample
extern "C" int mldb_sample(mldb_handle* h, const void* cond, const float* init_noise,
                           const int32_t* lengths, int32_t B, int32_t S_ctx, int32_t T,
                           float* latents_out, float* feats_out, float* joints_out, void* stream) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!cond || !init_noise || !lengths || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  Plan *rp = nullptr, *dp = nullptr;
  TRY(dec_plan(h, B, T, &dp));
  const mldb_config& c = h->cfg;
  // reverse diffusion writes [n_lat, B, d] into the decode plan's staging buffer
  float* z = latents_out;
  if (!z) {
    if (!dp->stage_f32) TRY(dev_alloc(h, (void**)&dp->stage_f32, (size_t)B * c.n_lat * c.latent_dim * sizeof(float)));
    z = dp->stage_f32;
  }
  if (c.arch != MLDB_ARCH_TRANS_ENC) FAIL(MLDB_ERR_UNSUPPORTED, "mldb_sample is built for the latent (VAE) models");
  TRY(run_reverse(h, cond, init_noise, nullptr, lengths, B, S_ctx, T, z, st, &rp));
  TRY(run_decode(h, z, lengths, B, T, feats_out, st, &dp));
  if (joints_out) TRY(run_f2j(h, feats_out ? feats_out : dp->feats, B, T, joints_out, st));
  return MLDB_OK;
}

// Multi-GPU: this rank samples its shard and the finished joints of every rank are gathered into
// joints_global [nranks * B, T, njoints, 3] (k_feats2joints writes straight into this rank's slot, ONE in-place
// ncclAllGather on the handle's side stream).  The call returns after enqueue; the gather of this batch
// overlaps whatever the caller enqueues next on `stream` - call mldb_gather_wait(h, stream) before reading
// joints_global on `stream`, and alternate (at least) two joints_global buffers between consecutive calls.
extern "C" int mldb_sample_gather(mldb_handle* h, const void* cond, const float* init_noise,
                                  const int32_t* lengths, int32_t B, int32_t S_ctx, int32_t T,
                                  float* joints_global, void* stream) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!joints_global) FAIL(MLDB_ERR_INVALID, "bad argument");
  const int64_t count = (int64_t)B * T * h->cfg.njoints * 3;
  cudaStream_t st = (cudaStream_t)stream;
  if (!h->nccl_comm) {      // single rank: the gather is the identity
    return mldb_sample(h, cond, init_noise, lengths, B, S_ctx, T, nullptr, nullptr, joints_global, stream);
  }
  TRY(mldb_gather_begin(h, st));
  TRY(mldb_sample(h, cond, init_noise, lengths, B, S_ctx, T, nullptr, nullptr, joints_global + h->comm_rank * count, stream));
  return mldb_gather_async(h, joints_global, count, st);
}

// Host-buffer entry point.  With a communicator attached joints_host receives the GATHERED motions
// [nranks * B, T, njoints, 3] (every rank holds all of them after the all-gather), else [B, T, njoints, 3].
extern "C" int mldb_sample_host(mldb_handle* h, const void* cond_host, const float* init_noise_host,
                                const int32_t* lengths_host, int32_t B, int32_t S_ctx, int32_t T,
                                float* joints_host, void* stream) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!cond_host || !init_noise_host || !lengths_host || !joints_host || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  const mldb_config& c = h->cfg;
  Plan* dp = nullptr;
  TRY(dec_plan(h, B, T, &dp));
  const bool cfg_on = c.guidance_scale > 1.0f;
  const int Bx = cfg_on ? 2 * B : B;
  const size_t cond_bytes = c.cond_kind == MLDB_COND_TEXT ? (size_t)Bx * S_ctx * c.text_dim * sizeof(float)
                                                         : (size_t)Bx * sizeof(int64_t);
  const size_t noise_bytes = (size_t)B * c.n_lat * c.latent_dim * sizeof(float);
  if (dp->cond_cap < cond_bytes) {
    TRY(dev_alloc(h, (void**)&dp->cond_f, cond_bytes));
    dp->cond_cap = cond_bytes;
  }
  if (!dp->noise_in) {
    TRY(dev_alloc(h, (void**)&dp->noise_in, noise_bytes));
    TRY(dev_alloc(h, (void**)&dp->cond_i, (size_t)B * sizeof(int32_t)));
  }
  const int world = h->nccl_comm ? h->comm_world : 1;
  const size_t joints_elems = (size_t)B * T * c.njoints * 3;
  if (world > 1 && !dp->joints_all) TRY(dev_alloc(h, (void**)&dp->joints_all, world * joints_elems * sizeof(float)));
  CK(cudaMemcpyAsync(dp->cond_f, cond_host, cond_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(dp->noise_in, init_noise_host, noise_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(dp->cond_i, lengths_host, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (world > 1) {
    TRY(mldb_sample_gather(h, dp->cond_f, dp->noise_in, (const int32_t*)dp->cond_i, B, S_ctx, T, dp->joints_all, stream));
    TRY(mldb_gather_wait(h, stream));
    CK(cudaMemcpyAsync(joints_host, dp->joints_all, world * joints_elems * sizeof(float), cudaMemcpyDeviceToHost, st));
    return MLDB_OK;
  }
  TRY(mldb_sample(h, dp->cond_f, dp->noise_in, (const int32_t*)dp->cond_i, B, S_ctx, T, nullptr, nullptr, dp->joints, stream));
  CK(cudaMemcpyAsync(joints_host, dp->joints, joints_elems * sizeof(float), cudaMemcpyDeviceToHost, st));
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- profiling aid
// Time one operator of denoiser layer 0 in isolation on the real workspace of the (B, S_ctx)
// reverse plan: `iters` back-to-back launches bracketed by CUDA events on `stream`.
// op: "qkv" | "attn" | "outproj_ln" | "ffn1" | "ffn2_ln" | "layer".  avg_ms_out: HOST float.
extern "C" int mldb_profile_op(mldb_handle* h, const char* op, int32_t B, int32_t S_ctx, int32_t iters,
                               float* avg_ms_out) {
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!op || !avg_ms_out || iters <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  const mldb_config& c = h->cfg;
  if (c.num_layers == 0 || c.arch != MLDB_ARCH_TRANS_ENC) FAIL(MLDB_ERR_UNSUPPORTED, "needs the trans_enc denoiser");
  const bool cfg_on = c.guidance_scale > 1.0f;
  Plan* p = nullptr;
  TRY(enc_plan(h, 0, B, cfg_on ? 2 * B : B, S_ctx, &p));
  cudaStream_t st = h->cap_stream;
  StackWs& ws = p->ws;
  const EncW& w = h->den.enc[0];
  const int d = ws.d;
  SeqInfo si;
  auto run = [&]() -> int {
    if (!strcmp(op, "qkv")) {
      GemmArgs g; g.a1 = ws.x0; g.K1 = d; g.M = ws.M; g.w = w.in_proj; g.out = ws.qkv; op_gemm(h, g, st);
    } else if (!strcmp(op, "attn")) {
      AttnArgs a; a.q = ws.qkv; a.Lq = ws.L; a.kv = ws.qkv; a.k_col0 = d; a.v_col0 = 2 * d; a.Lk = ws.L;
      a.nseq = ws.nseq; a.heads = c.num_heads; a.hd = d / c.num_heads; a.out = ws.att; op_attn(h, a, st);
    } else if (!strcmp(op, "outproj_ln")) {
      out_proj_ln(h, w.out_proj, w.n1, ws.att, ws.x0, ws.x1, ws.M, d, ws.cf32, st);
    } else if (!strcmp(op, "ffn1")) {
      GemmArgs g; g.a1 = ws.x1; g.K1 = d; g.M = ws.M; g.w = w.l1; g.act = ACT_GELU; g.out = ws.h; op_gemm(h, g, st);
    } else if (!strcmp(op, "ffn2_ln")) {
      GemmArgs g; g.a1 = ws.h; g.K1 = ws.ff; g.M = ws.M; g.w = w.l2;
      LnArgs l; l.res = ws.x1; l.gamma = w.n2.g; l.beta = w.n2.b; l.M = ws.M; l.d = d; l.out = ws.cur[0];
      op_gemm_ln(h, g, l, ws.cf32, st);
    } else if (!strcmp(op, "ffn")) {             // FFN1 + FFN2 the way the stack runs them (pair mode or not)
      ffn_block(h, w.l1, w.l2, w.n2, ws.x1, ws.cur[0], ws, ACT_GELU, st);
    } else if (!strcmp(op, "layer")) {
      enc_layer(h, h->den, w, ws.x0, ws.cur[0], ws, si, st);
    } else {
      FAIL(MLDB_ERR_INVALID, "unknown op %s", op);
    }
    return MLDB_OK;
  };
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int i = 0; i < 3; ++i) TRY(run());
  CK(cudaEventRecord(e0, st));
  for (int i = 0; i < iters; ++i) TRY(run());
  CK(cudaEventRecord(e1, st));
  CK(cudaStreamSynchronize(st));
  float ms = 0.0f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  CK(cudaGetLastError());
  *avg_ms_out = ms / (float)iters;
  return MLDB_OK;
}

// Per-step device times of the reverse loop: the same kernels as the captured graph, launched eagerly on the
// internal stream with a CUDA event between scheduler steps (bench.py's step p50).  cond / init_noise as for
// mldb_diffusion_reverse; ms_out: HOST float[n_steps].  Synchronous.
extern "C" int mldb_profile_steps(mldb_handle* h, const void* cond, const float* init_noise, int32_t B, int32_t S_ctx,
                                  float* ms_out) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!cond || !init_noise || !ms_out || B <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  const mldb_config& c = h->cfg;
  if (c.num_layers == 0 || c.arch != MLDB_ARCH_TRANS_ENC) FAIL(MLDB_ERR_UNSUPPORTED, "needs the trans_enc denoiser");
  if (c.sched_kind != MLDB_SCHED_DDIM) FAIL(MLDB_ERR_UNSUPPORTED, "step profiling is built for the DDIM loop");
  const bool cfg_on = c.guidance_scale > 1.0f;
  Plan* p = nullptr;
  TRY(enc_plan(h, 0, B, cfg_on ? 2 * B : B, S_ctx, &p));
  cudaStream_t st = h->cap_stream;
  const int d = c.latent_dim, nsteps = (int)h->timesteps.size();
  const int64_t per = (int64_t)c.n_lat * d;
  TRY(place_condition(h, p, cond, st));
  CK(cudaMemcpyAsync(p->latents, init_noise, (size_t)B * per * sizeof(float), cudaMemcpyDeviceToDevice, st));
  std::vector<cudaEvent_t> ev(nsteps + 1);
  for (auto& e : ev) CK(cudaEventCreate(&e));
  CK(cudaEventRecord(ev[0], st));
  for (int i = 0; i < nsteps; ++i) {
    denoiser_pass(h, p, p->latents, B, h->d_tt + (size_t)i * d, p->eps, st);
    launch_pdl(k_cfg_sched, dim3(nblk(B * per)), dim3(256), 0, st, (const float*)p->eps, p->latents, (const float*)nullptr,
               (int64_t)(B * per), cfg_on ? 1 : 0, c.guidance_scale, (const StepCoef*)h->d_coefs, i, (const int*)nullptr);
    kcount(h, MLDB_KSTAT_MISC);
    CK(cudaEventRecord(ev[i + 1], st));
  }
  CK(cudaStreamSynchronize(st));
  for (int i = 0; i < nsteps; ++i) CK(cudaEventElapsedTime(&ms_out[i], ev[i], ev[i + 1]));
  for (auto& e : ev) cudaEventDestroy(e);
  CK(cudaGetLastError());
  return check_ops(h);
}

// ----------------------------------------------------------------------------- debug aid
// y = act(A W^T + b) or LayerNorm(A W^T + b + R) through the engine's GEMM operators, so tests can
// compare the wgmma kernels with the CUDA-core kernels (and with torch) shape by shape.
//   A [M,K] fp32 device; W [N,K], bias [N], gamma/beta [N] fp32 HOST (gamma == NULL: no LN);
//   R [M,N] fp32 device or NULL; K1 < K splits A into two concatenated sources (skip connection);
//   out [M,N] fp32 device.  use_tc: 1 tensor-core path, 0 CUDA-core path.  Synchronous.
__global__ void k_split_to_f32(ActBuf X, float* __restrict__ out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = join_f32(X.hi[i], X.lo()[i]);
}
extern "C" int mldb_debug_gemm(mldb_handle* h, const float* A, const float* W, const float* bias,
                               const float* gamma, const float* beta, const float* R, int32_t M, int32_t N,
                               int32_t K, int32_t K1, int32_t act, int32_t use_tc, int32_t split_out, float* out,
                               void* stream) {
  if (!h || !A || !W || !out || M <= 0 || N <= 0 || K <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_alloc0 = h->allocs.size();
  LinW w;
  TRY(pack_linear(h, W, N, K, bias, &w));
  if (K1 <= 0 || K1 >= K) K1 = K;
  ActBuf a1, a2{}, res{}, o{};
  TRY(alloc_act(h, M, K1, &a1));
  k_rows_to_split<<<nblk((int64_t)M * K1), 256, 0, st>>>(a1, A, K, M, K1, 1 << 30, 0, 0, 0, nullptr);
  if (K1 < K) {
    TRY(alloc_act(h, M, K - K1, &a2));
    k_rows_to_split<<<nblk((int64_t)M * (K - K1)), 256, 0, st>>>(a2, A + K1, K, M, K - K1, 1 << 30, 0, 0, 0, nullptr);
  }
  float *g = nullptr, *b = nullptr, *cf32 = nullptr;
  const bool saved = h->use_tc;
  h->use_tc = use_tc != 0;
  GemmArgs ga; ga.a1 = a1; ga.K1 = K1; ga.a2 = a2; ga.K2 = K - K1; ga.M = M; ga.w = w; ga.act = act;
  int rc = MLDB_OK;
  if (gamma) {
    TRY(upload_f32(h, gamma, N, &g));
    TRY(upload_f32(h, beta, N, &b));
    TRY(dev_alloc(h, (void**)&cf32, (size_t)M * N * sizeof(float)));
    TRY(alloc_act(h, M, N, &o));
    if (R) {
      TRY(alloc_act(h, M, N, &res));
      k_rows_to_split<<<nblk((int64_t)M * N), 256, 0, st>>>(res, R, N, M, N, 1 << 30, 0, 0, 0, nullptr);
    }
    LnArgs l; l.res = res; l.gamma = g; l.beta = b; l.M = M; l.d = N; l.out = o;
    op_gemm_ln(h, ga, l, cf32, st);
    k_split_to_f32<<<nblk((int64_t)M * N), 256, 0, st>>>(o, out, (int64_t)M * N);
  } else if (split_out && N % 8 == 0) {
    TRY(alloc_act(h, M, N, &o));                   // the production epilogue: split16 planes
    ga.out = o;
    op_gemm(h, ga, st);
    k_split_to_f32<<<nblk((int64_t)M * N), 256, 0, st>>>(o, out, (int64_t)M * N);
  } else {
    ga.out_f32 = out; ga.ldc = N;
    op_gemm(h, ga, st);
  }
  h->use_tc = saved;
  cudaError_t e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  // release the temporaries
  while (h->allocs.size() > n_alloc0) { cudaFree(h->allocs.back()); h->allocs.pop_back(); }
  if (e != cudaSuccess) FAIL(MLDB_ERR_CUDA, "debug gemm: %s", cudaGetErrorString(e));
  return rc;
}

extern "C" int mldb_debug_ffn(mldb_handle* h, const float* X, const float* W1, const float* b1, const float* W2,
                              const float* b2, const float* gamma, const float* beta, int32_t M, int32_t d,
                              int32_t ff, int32_t mode, float* out, void* stream) {
  if (!h || !X || !W1 || !W2 || !gamma || !beta || !out || M <= 0 || d <= 0 || ff <= 0)
    FAIL(MLDB_ERR_INVALID, "bad argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_alloc0 = h->allocs.size();
  LinW l1, l2;
  LnW n;
  TRY(pack_linear(h, W1, ff, d, b1, &l1));
  TRY(pack_linear(h, W2, d, ff, b2, &l2));
  TRY(upload_f32(h, gamma, d, &n.g));
  TRY(upload_f32(h, beta, d, &n.b));
  StackWs ws;
  ws.M = M; ws.d = d; ws.ff = ff;
  ActBuf x, o;
  TRY(alloc_act(h, M, d, &x));
  TRY(alloc_act(h, M, d, &o));
  TRY(alloc_act(h, M, ff, &ws.h));
  TRY(dev_alloc(h, (void**)&ws.cf32, (size_t)M * d * sizeof(float)));
  k_rows_to_split<<<nblk((int64_t)M * d), 256, 0, st>>>(x, X, d, M, d, 1 << 30, 0, 0, 0, nullptr);
  const bool saved = h->use_tc;
  h->use_tc = mode != 0;
  const int saved_fused = tc_set_ffn_fused(h->tc, mode == 2);
  ffn_block(h, l1, l2, n, x, o, ws, ACT_GELU, st);
  h->use_tc = saved;
  tc_set_ffn_fused(h->tc, saved_fused);
  k_split_to_f32<<<nblk((int64_t)M * d), 256, 0, st>>>(o, out, (int64_t)M * d);
  cudaError_t e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  while (h->allocs.size() > n_alloc0) { cudaFree(h->allocs.back()); h->allocs.pop_back(); }
  if (e != cudaSuccess) FAIL(MLDB_ERR_CUDA, "debug ffn: %s", cudaGetErrorString(e));
  return MLDB_OK;
}

extern "C" int mldb_debug_attention(mldb_handle* h, const float* Q, const float* KV, const int32_t* lengths,
                                    int32_t kv_prefix, int32_t nseq, int32_t Lq, int32_t Lk, int32_t heads, int32_t hd,
                                    int32_t mode, float* out, void* stream) {
  if (!h || !Q || !out || nseq <= 0 || Lq <= 0 || Lk <= 0 || heads <= 0 || hd <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  if (!KV && Lq != Lk) FAIL(MLDB_ERR_INVALID, "a packed QKV input is self-attention: Lq must equal Lk");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_alloc0 = h->allocs.size();
  const int d = heads * hd, Mq = nseq * Lq, Mk = nseq * Lk;
  ActBuf qb, kvb, o;
  TRY(alloc_act(h, Mq, KV ? d : 3 * d, &qb));
  TRY(alloc_act(h, Mq, d, &o));
  rows_to_split(h, qb, Q, qb.cols, Mq, qb.cols, 1 << 30, 0, 0, 0, nullptr, 0, st);
  AttnArgs a; a.q = qb; a.q_col0 = 0; a.Lq = Lq; a.Lk = Lk;
  if (KV) {
    TRY(alloc_act(h, Mk, 2 * d, &kvb));
    rows_to_split(h, kvb, KV, 2 * d, Mk, 2 * d, 1 << 30, 0, 0, 0, nullptr, 0, st);
    a.kv = kvb; a.k_col0 = 0; a.v_col0 = d;
  } else {
    a.kv = qb; a.k_col0 = d; a.v_col0 = 2 * d;
  }
  a.nseq = nseq; a.heads = heads; a.hd = hd; a.lengths = lengths; a.kv_prefix = kv_prefix; a.out = o;
  int rc = MLDB_OK;
  if (mode == 0) simt_attention(a, st);
  else if (mode == 1 && mma_attention_supported(a)) mma_attention(a, st);
  else if (mode == 2 && tc_attention_supported(a)) { if (!tc_attention(a, st)) rc = MLDB_ERR_CUDA; }
  else rc = MLDB_ERR_UNSUPPORTED;
  if (rc == MLDB_OK) k_split_to_f32<<<nblk((int64_t)Mq * d), 256, 0, st>>>(o, out, (int64_t)Mq * d);
  cudaError_t e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  while (h->allocs.size() > n_alloc0) { cudaFree(h->allocs.back()); h->allocs.pop_back(); }
  if (e != cudaSuccess) FAIL(MLDB_ERR_CUDA, "debug attention: %s", cudaGetErrorString(e));
  if (rc == MLDB_ERR_UNSUPPORTED) FAIL(rc, "attention mode %d does not support this shape", mode);
  return rc;
}

// ----------------------------------------------------------------------------- debug timeline
static long long* g_timeline = nullptr;
namespace tc { long long* mldb_timeline_buffer() { return g_timeline; } }
// enable != 0: start (or restart) recording; enable == 0: copy the events recorded since the start into
// out (HOST int64[2 * cap]: {tag | warp << 16 | aux << 24, SM clock} pairs), *count = number of events, stop.
extern "C" int mldb_debug_timeline(int32_t enable, int64_t* out, int32_t cap, int32_t* count) {
  constexpr int WARPS = 32, CAPW = 512;                       // tc_common.cuh: TL_CAPW
  constexpr size_t BYTES = (size_t)WARPS * CAPW * 2 * sizeof(long long);
  if (enable) {
    if (!g_timeline && cudaMalloc((void**)&g_timeline, BYTES) != cudaSuccess) FAIL(MLDB_ERR_CUDA, "timeline buffer");
    CK(cudaMemset(g_timeline, 0, BYTES));
    return MLDB_OK;
  }
  if (!g_timeline) FAIL(MLDB_ERR_STATE, "no timeline is being recorded");
  if (!out || !count || cap <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  CK(cudaDeviceSynchronize());
  std::vector<long long> hbuf((size_t)WARPS * CAPW * 2);
  CK(cudaMemcpy(hbuf.data(), g_timeline, BYTES, cudaMemcpyDeviceToHost));
  int n = 0;
  for (int w = 0; w < WARPS; ++w)
    for (int i = 0; i < CAPW && n < cap; ++i) {
      const long long tag = hbuf[((size_t)w * CAPW + i) * 2], clk = hbuf[((size_t)w * CAPW + i) * 2 + 1];
      if (clk == 0) break;
      out[2 * n] = tag | ((long long)w << 16);                 // {tag | warp << 16 | aux << 24, clock}
      out[2 * n + 1] = clk;
      ++n;
    }
  *count = n;
  cudaFree(g_timeline);
  g_timeline = nullptr;
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- introspection
extern "C" int mldb_kernel_stats(const mldb_handle* h, int64_t* out, int32_t n) {
  if (!h || !out || n <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  for (int i = 0; i < n; ++i) out[i] = i < MLDB_KSTAT_COUNT ? h->kstat[i] : 0;
  return MLDB_OK;
}
extern "C" int mldb_reset_kernel_stats(mldb_handle* h) {
  if (!h) FAIL(MLDB_ERR_INVALID, "null handle");
  for (int i = 0; i < MLDB_KSTAT_COUNT; ++i) h->kstat[i] = 0;
  return MLDB_OK;
}
