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
  c->beta_schedule = MLDB_BETA_SCALED_LINEAR; c->clip_sample = 0;
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
    // the encoder half (actor_vae.py:86-118) is all or none: see mldb_finalize_weights
    spec_add(h, V + "encoder.mu_token", {d});
    spec_add(h, V + "encoder.logvar_token", {d});
    spec_add(h, V + "encoder.skel_embedding.weight", {d, c.vae_nfeats});
    spec_add(h, V + "encoder.skel_embedding.bias", {d});
    spec_add(h, V + "encoder.sequence_pos_encoding.pe", {5000, 1, d});
    for (int i = 0; i < c.vae_layers; ++i)
      spec_layer(h, V + "encoder.seqTransEncoder.layers." + std::to_string(i) + ".", d, c.vae_ff, false);
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
// The scale comes from the finite elements only, so an inf or NaN element poisons its own output column (as in
// torch) and not the precision of every other one; an all-zero or all non-finite W packs at s = 0.
static int pack_linear(mldb_handle* h, const float* W, int N, int K, const float* bias, LinW* out, int Kpad = 0) {
  if (Kpad < K) Kpad = K;
  float mx = 0.0f;
  for (int64_t i = 0; i < (int64_t)N * K; ++i)
    if (std::isfinite(W[i])) mx = std::max(mx, fabsf(W[i]));
  int s = 0;
  if (mx > 0.0f) {
    // clamp before the conversion to int: below mx ~ 5e-35, 16384 / mx overflows to inf
    const float e = floorf(log2f(16384.0f / mx));
    s = (int)std::max(-14.0f, std::min(14.0f, e));
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
// the q rows and the k | v rows of an encoder layer's in_proj as separate operands (enc_layer_selected)
static int pack_trimmed_qkv(mldb_handle* h, const std::string& p, int d, EncW* w) {
  TRY(pack_named(h, p + "self_attn.in_proj_weight", p + "self_attn.in_proj_bias", &w->q_only, 0, d));
  TRY(pack_named(h, p + "self_attn.in_proj_weight", p + "self_attn.in_proj_bias", &w->kv_only, d, 2 * d));
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
  if (!dec) TRY(pack_trimmed_qkv(h, names.back(), d, &s->enc.back()));   // the last block only has to produce
                                                                             // the first few tokens of every sequence
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
// ActorAgnosticEncoder (actor_vae.py:86-118): a plain encoder stack, [mu_token; logvar_token] as a 2-row token
// table, the skel embedding with K zero-padded for the tensor cores, and the encoder's own sine PE table
static int pack_actor_encoder(mldb_handle* h) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim;
  const std::string E = "vae.encoder.";
  StackW* s = &h->venc;
  s->kind = STACK_PLAIN_ENC; s->d = d; s->ff = c.vae_ff; s->heads = c.vae_heads; s->layers = c.vae_layers;
  for (int i = 0; i < c.vae_layers; ++i) {
    const std::string n = E + "seqTransEncoder.layers." + std::to_string(i) + ".";
    s->enc.emplace_back();
    TRY(pack_enc_layer(h, n, d, &s->enc.back()));
    if (i == c.vae_layers - 1) TRY(pack_trimmed_qkv(h, n, d, &s->enc.back()));
  }
  std::vector<float> tok(rt(h, E + "mu_token").host);
  const std::vector<float>& lv = rt(h, E + "logvar_token").host;
  tok.insert(tok.end(), lv.begin(), lv.end());
  TRY(upload_f32(h, tok.data(), tok.size(), &h->global_token));
  TRY(pack_named(h, E + "skel_embedding.weight", E + "skel_embedding.bias", &h->skel_emb, 0, -1, true));
  return upload_pe(h, E + "sequence_pos_encoding.pe", &h->vae_enc_pe, &h->vae_enc_pe_rows);
}

// ----------------------------------------------------------------------------- scheduler
// The scheduler settings the library implements (diffusers DDIMScheduler / DDPMScheduler with epsilon
// prediction, fixed_small variance, clip_sample_range 1.0).
static int check_sched_cfg(const mldb_config& c) {
  if (c.sched_kind != MLDB_SCHED_DDIM && c.sched_kind != MLDB_SCHED_DDPM) FAIL(MLDB_ERR_INVALID, "unknown sched_kind %d", c.sched_kind);
  if (c.beta_schedule != MLDB_BETA_SCALED_LINEAR && c.beta_schedule != MLDB_BETA_LINEAR &&
      c.beta_schedule != MLDB_BETA_SQUAREDCOS_CAP_V2)
    FAIL(MLDB_ERR_INVALID, "unknown beta_schedule %d", c.beta_schedule);
  if (!(c.eta >= 0.0f && c.eta <= 1.0f)) FAIL(MLDB_ERR_INVALID, "eta must lie in [0, 1], got %g", (double)c.eta);
  if (c.num_train_timesteps < 2) FAIL(MLDB_ERR_INVALID, "num_train_timesteps must be >= 2");
  return MLDB_OK;
}

// alphas_cumprod = cumprod(1 - betas) for the configured beta_schedule (fp32 like torch):
//   scaled_linear      betas = linspace(sqrt(b0), sqrt(b1), T, fp32) ** 2
//   linear             betas = linspace(b0, b1, T, fp32)
//   squaredcos_cap_v2  betas = fp32(min(1 - alpha_bar((i+1)/T) / alpha_bar(i/T), 0.999)) in double,
//                      alpha_bar(t) = cos((t + 0.008) / 1.008 * pi / 2) ** 2  (diffusers betas_for_alpha_bar)
static void build_alphas(const mldb_config& c, std::vector<float>* out) {
  // Bit-exact with torch on CPU (checked in tests/test_scheduler.py and test_scheduler_stochastic.py):
  // linspace evaluates start + step*i (first half) / end - step*(T-1-i) (second half) with one rounding
  // (FMA); cumprod accumulates in double (at::acc_type<float> on CPU) and rounds each output.
  const int T = c.num_train_timesteps;
  out->resize(T);
  const bool scaled = c.beta_schedule == MLDB_BETA_SCALED_LINEAR;
  const float s0 = scaled ? (float)sqrt(c.beta_start) : (float)c.beta_start;
  const float s1 = scaled ? (float)sqrt(c.beta_end) : (float)c.beta_end;
  const float step = (s1 - s0) / (float)(T - 1);
  auto alpha_bar = [](double t) { return pow(cos((t + 0.008) / 1.008 * M_PI / 2), 2.0); };
  double prod = 1.0;
  for (int i = 0; i < T; ++i) {
    float beta;
    if (c.beta_schedule == MLDB_BETA_SQUAREDCOS_CAP_V2) {
      const double t1 = (double)i / T, t2 = (double)(i + 1) / T;
      beta = (float)std::min(1.0 - alpha_bar(t2) / alpha_bar(t1), 0.999);
    } else {
      const float v = (i < T / 2) ? fmaf(step, (float)i, s0) : fmaf(-step, (float)(T - 1 - i), s1);
      beta = scaled ? v * v : v;
    }
    const float alpha = 1.0f - beta;
    prod *= (double)alpha;
    (*out)[i] = (float)prod;
  }
}
extern "C" int mldb_scheduler_table(const mldb_config* cfg, float* alphas_cumprod_out) {
  if (!cfg || !alphas_cumprod_out) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(check_sched_cfg(*cfg));
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
  k.clip = c.clip_sample ? 1 : 0;
  if (c.sched_kind == MLDB_SCHED_DDIM) {
    const float a_prev = prev_t >= 0 ? ac[prev_t] : (c.set_alpha_to_one ? 1.0f : ac[0]);
    // variance = (beta_prod_t_prev / beta_prod_t) * (1 - alpha_prod_t / alpha_prod_t_prev);
    // std_dev_t = eta * variance ** 0.5 (0 when eta == 0: c3 is then sqrt(1 - a_prev - 0))
    const float variance = ((1.0f - a_prev) / (1.0f - a_t)) * (1.0f - a_t / a_prev);
    const float std_dev = c.eta * sqrtf(variance);
    k.kind = 0;
    k.c2 = sqrtf(a_prev);
    k.c3 = sqrtf(1.0f - a_prev - std_dev * std_dev);
    k.sigma = std_dev;
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
    if (!simt_attention(a, st)) {
      mldb_set_err("CUDA-core attention: head_dim " + std::to_string(a.hd) + " does not fit shared memory");
      h->op_failed = true;
    }
    kcount(h, MLDB_KSTAT_ATTN_SIMT);
  }
}
// which stream's scratch / flags the fused FFN uses (branches run concurrently, each on its own pair)
static int ffn_scratch_slot(const mldb_handle* h, cudaStream_t st) {
  int k = 0;
  for (int i = 0; i < mldb_handle::MAX_BRANCHES - 1; ++i) if (st == h->br_stream[i]) k = i + 1;
  return k;
}
// the fused FFN block when the shape allows it, else the two GEMMs
static void op_ffn(mldb_handle* h, const GemmArgs& g1, const GemmArgs& g2, const LnArgs& l2, float* cf32, cudaStream_t st) {
  if (h->use_tc && tc_ffn_supported(h->tc, g1, g2, l2)) {
    // one launch: the hidden activations stay in registers (gemm_tc.cu k_ffn_tc)
    const int k = ffn_scratch_slot(h, st);
    if (!tc_ffn(h->tc, g1, g2, l2, h->ffn_scratch[k], h->ffn_flags[k], st)) h->op_failed = true;
    kcount(h, MLDB_KSTAT_FFN_TC);
    return;
  }
  op_gemm(h, g1, st);
  op_gemm_ln(h, g2, l2, cf32, st);
}
// An encoder layer after its attention: x1 = LN1(att W_o^T + b_o + x), then the FFN block on x1 into xout (x1 and
// hbuf are workspaces).  The fused launch (k_ffn_tc with its out-projection prefix, which keeps x1 in shared memory
// and does not write it) runs for at most FUSE_MAX_TILES m-tiles; else (or with fuse == 0: mldb_debug_tail's
// two-kernel arm) the out-projection + LN GEMM and op_ffn, which write x1.  Measured on H100: at 2 m-tiles (one
// prompt) the saved launch and x1 round trip make the whole sample 8 % faster than the two launches; at 24 m-tiles
// (action512) and at 158 (the headline's sub-batches) the fused launch is 4-10 % slower end to end.  Its x tile holds
// att, then x1, then y until the y store has read it, so a tile's loads are not overlapped with the previous tile's
// work, and every ffn_split piece repeats the out-projection.  fuse: 0 never, 1 the size rule, 2 whenever the kernel
// takes the shape (mldb_debug_tail, profile_op "tail_fused").
static void op_tail(mldb_handle* h, const LinW& wo, const LnW& n1, const LinW& l1, const LinW& l2, const LnW& n2,
                    ActBuf att, ActBuf x, ActBuf x1, ActBuf hbuf, ActBuf xout, int M, int d, int ff, float* cf32,
                    cudaStream_t st, int fuse = 1) {
  GemmArgs go; go.a1 = att; go.K1 = d; go.M = M; go.w = wo;
  LnArgs ln1; ln1.res = x; ln1.gamma = n1.g; ln1.beta = n1.b; ln1.M = M; ln1.d = d; ln1.out = x1;
  GemmArgs g1; g1.a1 = x1; g1.K1 = d; g1.M = M; g1.w = l1; g1.act = ACT_GELU; g1.out = hbuf;
  GemmArgs g2; g2.a1 = hbuf; g2.K1 = ff; g2.M = M; g2.w = l2;
  LnArgs ln2; ln2.res = x1; ln2.gamma = n2.g; ln2.beta = n2.b; ln2.M = M; ln2.d = d; ln2.out = xout;
  constexpr int FUSE_MAX_TILES = 2;
  const bool small = (M + 127) / 128 <= FUSE_MAX_TILES;
  if (fuse && (fuse == 2 || small) && h->use_tc && tc_tail_supported(h->tc, go, ln1, g1, g2, ln2)) {
    const int k = ffn_scratch_slot(h, st);
    if (!tc_tail(h->tc, go, ln1, g1, g2, ln2, h->ffn_scratch[k], h->ffn_flags[k], st)) h->op_failed = true;
    kcount(h, MLDB_KSTAT_FFN_TC);
    return;
  }
  op_gemm_ln(h, go, ln1, cf32, st);
  op_ffn(h, g1, g2, ln2, cf32, st);
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
  const bool enc = sw.kind == STACK_SKIP_ENC || sw.kind == STACK_PLAIN_ENC;
  if (!enc) {
    TRY(alloc_act(h, M, d, &ws->x2));
    TRY(alloc_act(h, M, d, &ws->qc));
    TRY(alloc_act(h, nseq * Lmem, 2 * d, &ws->kvm));
    TRY(alloc_act(h, nseq, d, &ws->vrow));
    TRY(dev_alloc(h, (void**)&ws->cvec, (size_t)nseq * d * sizeof(float)));
  }
  if (sw.kind == STACK_SKIP_ENC || sw.kind == STACK_SKIP_DEC) {
    TRY(alloc_act(h, M, d, &ws->cat));
    const int nb = (sw.layers - 1) / 2;
    ws->ys.resize(nb);
    for (int i = 0; i < nb; ++i) TRY(alloc_act(h, M, d, &ws->ys[i]));
  }
  TRY(dev_alloc(h, (void**)&ws->cf32, (size_t)M * d * sizeof(float)));
  if (enc && n_sel > 0) {
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
// QKV projection + self-attention of xin -> ws.att
static void self_attn(mldb_handle* h, const LinW& in_proj, ActBuf xin, StackWs& ws, const SeqInfo& si, int heads,
                      cudaStream_t st) {
  const int d = ws.d;
  GemmArgs g; g.a1 = xin; g.K1 = d; g.M = ws.M; g.w = in_proj; g.out = ws.qkv;
  op_gemm(h, g, st);
  AttnArgs a; a.q = ws.qkv; a.q_col0 = 0; a.Lq = ws.L; a.kv = ws.qkv; a.k_col0 = d; a.v_col0 = 2 * d;
  a.Lk = ws.L; a.nseq = ws.nseq; a.heads = heads; a.hd = d / heads;
  a.lengths = si.lengths; a.kv_prefix = si.kv_prefix; a.len_mod = si.len_mod; a.seq0 = 0; a.out = ws.att;
  op_attn(h, a, st);
}
static void self_attn_block(mldb_handle* h, const LinW& in_proj, const LinW& out_proj, const LnW& n,
                            ActBuf xin, ActBuf xout, StackWs& ws, const SeqInfo& si, int heads,
                            cudaStream_t st) {
  self_attn(h, in_proj, xin, ws, si, heads, st);
  out_proj_ln(h, out_proj, n, ws.att, xin, xout, ws.M, ws.d, ws.cf32, st);
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
  self_attn(h, w.in_proj, xin, ws, si, sw.heads, st);
  op_tail(h, w.out_proj, w.n1, w.l1, w.l2, w.n2, ws.att, xin, ws.x1, ws.h, xout, ws.M, ws.d, ws.ff, ws.cf32, st);
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
  op_tail(h, w.out_proj, w.n1, w.l1, w.l2, w.n2, ws.satt, ws.sx, ws.sx1, ws.sh, ws.sout, R, d, ws.ff, ws.cf32, st);
  return ws.sout;
}

// SkipTransformerEncoder/Decoder.forward (cross_attention.py:41-64, 89-125), the plain
// decoder stacks (cross_attention.py:204-233; torch nn.TransformerDecoder for ActorVae) and
// ActorVae's torch nn.TransformerEncoder (actor_vae.py:114-118, no final norm).
// Returns the buffer holding the last layer's output (before the stack's final norm); the compact
// [nseq * n_sel] rows when the last layer runs trimmed.
static ActBuf run_stack(mldb_handle* h, const StackW& sw, ActBuf x0, ActBuf mem, StackWs& ws,
                        const SeqInfo& si, cudaStream_t st) {
  if (sw.kind == STACK_PLAIN_ENC) {   // only the distribution tokens leave the stack (actor_vae.py:169)
    ActBuf x = x0;
    for (int i = 0; i + 1 < sw.layers; ++i) {
      enc_layer(h, sw, sw.enc[i], x, ws.cur[i & 1], ws, si, st);
      x = ws.cur[i & 1];
    }
    return enc_layer_selected(h, sw, sw.enc.back(), x, ws, si, st);
  }
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
  // every attention shape must have a kernel: the CUDA-core core takes any length, but not any head width
  for (int heads : {cfg->num_heads, cfg->vae_heads})
    if (heads > 0 && !simt_attention_supported(cfg->latent_dim / heads))
      FAIL(MLDB_ERR_UNSUPPORTED, "head_dim %d is too wide for the attention kernels", cfg->latent_dim / heads);
  if (cfg->arch == MLDB_ARCH_TRANS_ENC && cfg->num_layers > 0 && cfg->num_layers % 2 != 1) FAIL(MLDB_ERR_INVALID, "skip encoder needs an odd layer count");
  if (cfg->arch == MLDB_ARCH_TRANS_ENC && cfg->diffusion_only) FAIL(MLDB_ERR_UNSUPPORTED, "diffusion_only requires arch trans_dec");
  if (cfg->vae_kind == MLDB_VAE_MLD && cfg->vae_layers % 2 != 1) FAIL(MLDB_ERR_INVALID, "MldVae needs an odd layer count");
  TRY(check_sched_cfg(*cfg));
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
  // kernel setup: each step records its own message in mldb_last_error() when it fails
  if (!simt_init() || !mma_attention_init()) { delete h; return MLDB_ERR_CUDA; }
  h->tc = tc_create(device);
  if (!h->tc) { delete h; return MLDB_ERR_CUDA; }
  if (!tc_attention_init(device) || !gru_tc_init()) { tc_destroy(h->tc); delete h; return MLDB_ERR_CUDA; }
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
  for (void* p : h->text.ws_allocs) cudaFree(p);
  for (void* p : h->t2m.buf) cudaFree(p);
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
  } else if (!strcmp(name, "t2m_chunk")) {
    h->t2m.chunk = std::max(atoi(value), 0);
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
  if (it == h->raw.end()) FAIL(MLDB_ERR_INVALID, "unexpected state-dict key '%s'", key);
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


// ----------------------------------------------------------------------------- CLIP text tower: spec / pack
static const std::string kTextPrefix = "text_encoder.text_model.";   // MldTextEncoder.text_model (a CLIPModel)

extern "C" void mldb_default_text_config(mldb_text_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = MLDB_TEXT_ABI_VERSION;
  c->vocab_size = 49408; c->max_positions = 77; c->hidden = 768; c->heads = 12; c->layers = 12; c->ff = 3072;
  c->projection_dim = 768; c->eos_token_id = 49407; c->ln_eps = 1e-5f;
}

extern "C" int mldb_text_configure(mldb_handle* h, const mldb_text_config* cfg) {
  if (!h || !cfg) FAIL(MLDB_ERR_INVALID, "null argument");
  if (cfg->abi_version != MLDB_TEXT_ABI_VERSION) FAIL(MLDB_ERR_INVALID, "mldb_text_config abi_version mismatch");
  if (h->finalized) FAIL(MLDB_ERR_STATE, "mldb_text_configure must precede mldb_finalize_weights");
  if (h->text.on) FAIL(MLDB_ERR_STATE, "the text tower is already configured");
  const mldb_text_config& c = *cfg;
  if (c.vocab_size < 1 || c.layers < 1 || c.heads < 1 || c.ff < 1 || c.projection_dim < 1 || !(c.ln_eps > 0.0f))
    FAIL(MLDB_ERR_INVALID, "bad text config");
  if (!text_ln_supported(c.hidden) || c.hidden % c.heads)
    FAIL(MLDB_ERR_UNSUPPORTED, "text hidden size %d: must be a multiple of 128 (<= 1024) and of heads", c.hidden);
  if (!simt_attention_supported(c.hidden / c.heads))
    FAIL(MLDB_ERR_UNSUPPORTED, "text head_dim %d is too wide for the attention kernels", c.hidden / c.heads);
  if (c.max_positions < 1 || c.max_positions > 256) FAIL(MLDB_ERR_UNSUPPORTED, "max_positions must lie in [1, 256]");
  const std::string T = kTextPrefix, M = T + "text_model.";
  const int d = c.hidden;
  spec_add(h, M + "embeddings.token_embedding.weight", {c.vocab_size, d});
  spec_add(h, M + "embeddings.position_embedding.weight", {c.max_positions, d});
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = M + "encoder.layers." + std::to_string(i) + ".";
    for (const char* pr : {"q_proj.", "k_proj.", "v_proj.", "out_proj."}) {
      spec_add(h, p + "self_attn." + pr + "weight", {d, d});
      spec_add(h, p + "self_attn." + pr + "bias", {d});
    }
    spec_ln(h, p + "layer_norm1.", d);
    spec_add(h, p + "mlp.fc1.weight", {c.ff, d});
    spec_add(h, p + "mlp.fc1.bias", {c.ff});
    spec_add(h, p + "mlp.fc2.weight", {d, c.ff});
    spec_add(h, p + "mlp.fc2.bias", {d});
    spec_ln(h, p + "layer_norm2.", d);
  }
  spec_ln(h, M + "final_layer_norm.", d);
  spec_add(h, T + "text_projection.weight", {c.projection_dim, d});
  h->text.cfg = c;
  h->text.on = true;
  return MLDB_OK;
}

static int pack_text(mldb_handle* h) {
  TextW& tw = h->text;
  const mldb_text_config& c = tw.cfg;
  const std::string T = kTextPrefix, M = T + "text_model.";
  const int d = c.hidden;
  TRY(upload_pe(h, M + "embeddings.token_embedding.weight", &tw.tok));
  TRY(upload_pe(h, M + "embeddings.position_embedding.weight", &tw.pos));
  tw.layers.resize(c.layers);
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = M + "encoder.layers." + std::to_string(i) + ".";
    TextLayerW& w = tw.layers[i];
    // one [3d, d] operand: rows q | k | v (the attention kernels' packed-QKV layout)
    std::vector<float> W((size_t)3 * d * d), b((size_t)3 * d);
    const char* names[3] = {"q_proj.", "k_proj.", "v_proj."};
    for (int j = 0; j < 3; ++j) {
      const RawTensor& wt = rt(h, p + "self_attn." + names[j] + "weight");
      const RawTensor& bt = rt(h, p + "self_attn." + names[j] + "bias");
      std::copy(wt.host.begin(), wt.host.end(), W.begin() + (size_t)j * d * d);
      std::copy(bt.host.begin(), bt.host.end(), b.begin() + (size_t)j * d);
    }
    TRY(pack_linear(h, W.data(), 3 * d, d, b.data(), &w.qkv));
    TRY(pack_named(h, p + "self_attn.out_proj.weight", p + "self_attn.out_proj.bias", &w.out));
    TRY(pack_named(h, p + "mlp.fc1.weight", p + "mlp.fc1.bias", &w.fc1));
    TRY(pack_named(h, p + "mlp.fc2.weight", p + "mlp.fc2.bias", &w.fc2));
    TRY(pack_ln(h, p + "layer_norm1.", d, &w.ln1));
    TRY(pack_ln(h, p + "layer_norm2.", d, &w.ln2));
  }
  TRY(pack_ln(h, M + "final_layer_norm.", d, &tw.final_ln));
  TRY(pack_named(h, T + "text_projection.weight", "", &tw.proj));
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- T2M evaluator: spec / pack
static const char* const kT2mText = "t2m_textencoder.";      // MLD attribute names (mld.py:148-164)
static const char* const kT2mMove = "t2m_moveencoder.";
static const char* const kT2mMotion = "t2m_motionencoder.";
static int pad64(int k) { return (k + 63) / 64 * 64; }

extern "C" void mldb_default_t2m_config(mldb_t2m_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = MLDB_T2M_ABI_VERSION;
  c->parts = MLDB_T2M_TEXT | MLDB_T2M_MOVEMENT | MLDB_T2M_MOTION;
  c->dim_word = 300; c->dim_pos_ohot = 15; c->dim_text_hidden = 512; c->dim_coemb_hidden = 512;
  c->dim_pose = 259; c->dim_move_hidden = 512; c->dim_move_latent = 512; c->dim_motion_hidden = 1024;
  c->dim_motion_latent = 512;
}

// nn.GRU(in, H, bidirectional) + the BiGRUCo head (output_net: Linear(2H, H), LayerNorm(H), LeakyReLU, Linear(H, out))
static void spec_gru(mldb_handle* h, const std::string& p, int in, int H, int out) {
  spec_add(h, p + "hidden", {2, 1, H});
  for (const char* sfx : {"", "_reverse"}) {
    spec_add(h, p + "gru.weight_ih_l0" + sfx, {3 * H, in});
    spec_add(h, p + "gru.weight_hh_l0" + sfx, {3 * H, H});
    spec_add(h, p + "gru.bias_ih_l0" + sfx, {3 * H});
    spec_add(h, p + "gru.bias_hh_l0" + sfx, {3 * H});
  }
  spec_add(h, p + "output_net.0.weight", {H, 2 * H});
  spec_add(h, p + "output_net.0.bias", {H});
  spec_ln(h, p + "output_net.1.", H);
  spec_add(h, p + "output_net.3.weight", {out, H});
  spec_add(h, p + "output_net.3.bias", {out});
}

extern "C" int mldb_t2m_configure(mldb_handle* h, const mldb_t2m_config* cfg) {
  if (!h || !cfg) FAIL(MLDB_ERR_INVALID, "null argument");
  if (cfg->abi_version != MLDB_T2M_ABI_VERSION) FAIL(MLDB_ERR_INVALID, "mldb_t2m_config abi_version mismatch");
  if (h->finalized) FAIL(MLDB_ERR_STATE, "mldb_t2m_configure must precede mldb_finalize_weights");
  if (h->t2m.on) FAIL(MLDB_ERR_STATE, "the T2M evaluator is already configured");
  const mldb_t2m_config& c = *cfg;
  if (c.parts < 1 || c.parts > 7) FAIL(MLDB_ERR_INVALID, "parts must be a non-empty MLDB_T2M_* mask");
  if (c.dim_word < 1 || c.dim_pos_ohot < 1 || c.dim_coemb_hidden < 1 || c.dim_pose < 1 || c.dim_motion_latent < 1)
    FAIL(MLDB_ERR_INVALID, "bad T2M config");
  if (c.dim_word % 2 || c.dim_word > 4096) FAIL(MLDB_ERR_UNSUPPORTED, "dim_word must be even and <= 4096");
  if (!gru_shape_supported(c.dim_text_hidden) || !gru_shape_supported(c.dim_motion_hidden))
    FAIL(MLDB_ERR_UNSUPPORTED, "GRU hidden sizes must be multiples of 64 in [64, 1024]");
  for (int v : {c.dim_move_hidden, c.dim_move_latent})
    if (v < 64 || v % 64 || v > 4096) FAIL(MLDB_ERR_UNSUPPORTED, "dim_move_hidden / dim_move_latent must be multiples of 64 up to 4096");
  if (c.dim_coemb_hidden > 4096 || c.dim_motion_latent > 4096 || c.dim_pose > 4096)
    FAIL(MLDB_ERR_UNSUPPORTED, "T2M output / pose widths must be <= 4096");
  if (c.parts & MLDB_T2M_TEXT) {
    const std::string p = kT2mText;
    spec_add(h, p + "pos_emb.weight", {c.dim_word, c.dim_pos_ohot});
    spec_add(h, p + "pos_emb.bias", {c.dim_word});
    spec_add(h, p + "input_emb.weight", {c.dim_text_hidden, c.dim_word});
    spec_add(h, p + "input_emb.bias", {c.dim_text_hidden});
    spec_gru(h, p, c.dim_text_hidden, c.dim_text_hidden, c.dim_coemb_hidden);
  }
  if (c.parts & MLDB_T2M_MOVEMENT) {
    const std::string p = kT2mMove;
    spec_add(h, p + "main.0.weight", {c.dim_move_hidden, c.dim_pose, 4});
    spec_add(h, p + "main.0.bias", {c.dim_move_hidden});
    spec_add(h, p + "main.3.weight", {c.dim_move_latent, c.dim_move_hidden, 4});
    spec_add(h, p + "main.3.bias", {c.dim_move_latent});
    spec_add(h, p + "out_net.weight", {c.dim_move_latent, c.dim_move_latent});
    spec_add(h, p + "out_net.bias", {c.dim_move_latent});
  }
  if (c.parts & MLDB_T2M_MOTION) {
    const std::string p = kT2mMotion;
    spec_add(h, p + "input_emb.weight", {c.dim_motion_hidden, c.dim_move_latent});
    spec_add(h, p + "input_emb.bias", {c.dim_motion_hidden});
    spec_gru(h, p, c.dim_motion_hidden, c.dim_motion_hidden, c.dim_motion_latent);
  }
  h->t2m.cfg = c;
  h->t2m.on = true;
  return MLDB_OK;
}

static int pack_gru(mldb_handle* h, const std::string& p, int H, GruW* g) {
  g->H = H;
  const char* sfx[2] = {"", "_reverse"};
  std::vector<float> W((size_t)6 * H * H), b((size_t)6 * H);
  for (int d = 0; d < 2; ++d) {
    TRY(pack_named(h, p + "gru.weight_ih_l0" + sfx[d], p + "gru.bias_ih_l0" + sfx[d], &g->w_ih[d]));
    const std::vector<float>& w = rt(h, p + "gru.weight_hh_l0" + sfx[d]).host;
    const std::vector<float>& bh = rt(h, p + "gru.bias_hh_l0" + sfx[d]).host;
    for (int gate = 0; gate < 3; ++gate)
      for (int u = 0; u < H; ++u)
        std::copy_n(w.begin() + (size_t)(gate * H + u) * H, H, W.begin() + ((size_t)d * 3 * H + gru_packed_col(gate, u)) * H);
    std::copy(bh.begin(), bh.end(), b.begin() + (size_t)d * 3 * H);
  }
  TRY(pack_linear(h, W.data(), 6 * H, H, nullptr, &g->w_hh));
  TRY(upload_f32(h, b.data(), b.size(), &g->b_hh));
  TRY(upload_f32(h, rt(h, p + "hidden").host.data(), (size_t)2 * H, &g->h0));
  TRY(pack_named(h, p + "output_net.0.weight", p + "output_net.0.bias", &g->head1));
  TRY(pack_ln(h, p + "output_net.1.", H, &g->ln));
  TRY(pack_named(h, p + "output_net.3.weight", p + "output_net.3.bias", &g->head2));
  return MLDB_OK;
}

// Conv1d weight [O, C, 4] -> the GEMM operand [O, 4 * Cp]: column k * Cp + c (zero for c >= C), matching k_im2col_k4s2
static int pack_conv(mldb_handle* h, const std::string& p, int O, int C, int Cp, LinW* out) {
  const std::vector<float>& w = rt(h, p + "weight").host;
  std::vector<float> W((size_t)O * 4 * Cp, 0.0f);
  for (int o = 0; o < O; ++o)
    for (int c = 0; c < C; ++c)
      for (int k = 0; k < 4; ++k) W[(size_t)o * 4 * Cp + (size_t)k * Cp + c] = w[((size_t)o * C + c) * 4 + k];
  return pack_linear(h, W.data(), O, 4 * Cp, rt(h, p + "bias").host.data(), out);
}

static int pack_t2m(mldb_handle* h) {
  T2mW& t = h->t2m;
  const mldb_t2m_config& c = t.cfg;
  if (c.parts & MLDB_T2M_TEXT) {
    const std::string p = kT2mText;
    TRY(pack_named(h, p + "pos_emb.weight", p + "pos_emb.bias", &t.pos_emb, 0, -1, true));
    TRY(pack_named(h, p + "input_emb.weight", p + "input_emb.bias", &t.text_in, 0, -1, true));
    TRY(pack_gru(h, p, c.dim_text_hidden, &t.text_gru));
  }
  if (c.parts & MLDB_T2M_MOVEMENT) {
    const std::string p = kT2mMove;
    TRY(pack_conv(h, p + "main.0.", c.dim_move_hidden, c.dim_pose, (c.dim_pose + 15) / 16 * 16, &t.conv1));
    TRY(pack_conv(h, p + "main.3.", c.dim_move_latent, c.dim_move_hidden, c.dim_move_hidden, &t.conv2));
    TRY(pack_named(h, p + "out_net.weight", p + "out_net.bias", &t.move_out));
  }
  if (c.parts & MLDB_T2M_MOTION) {
    const std::string p = kT2mMotion;
    TRY(pack_named(h, p + "input_emb.weight", p + "input_emb.bias", &t.motion_in));
    TRY(pack_gru(h, p, c.dim_motion_hidden, &t.motion_gru));
  }
  return MLDB_OK;
}

extern "C" int mldb_finalize_weights(mldb_handle* h, void* stream) {
  (void)stream;
  if (!h) FAIL(MLDB_ERR_INVALID, "null handle");
  if (h->finalized) FAIL(MLDB_ERR_STATE, "already finalized");
  const mldb_config& c = h->cfg;
  // ActorVae's encoder keys are all or none: a decoder-only state dict samples and decodes (mldb_vae_encode then
  // refuses), a partial encoder is an incomplete load
  const std::string AE = "vae.encoder.";
  auto is_actor_enc = [&](const std::string& k) { return c.vae_kind == MLDB_VAE_ACTOR && !k.compare(0, AE.size(), AE); };
  bool actor_enc = false;
  for (auto& kv : h->raw)
    if (is_actor_enc(kv.first) && kv.second.loaded) actor_enc = true;
  for (auto& kv : h->raw)
    if (!kv.second.loaded && (actor_enc || !is_actor_enc(kv.first)))
      FAIL(MLDB_ERR_STATE, "missing state-dict key '%s' (strict load)", kv.first.c_str());
  DeviceGuard guard(h->device);
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
    TRY(upload_pe(h, V + "query_pos_encoder.pe", &h->vae_enc_pe, &h->vae_enc_pe_rows));
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
    if (actor_enc) TRY(pack_actor_encoder(h));
  }
  if (h->text.on) TRY(pack_text(h));
  if (h->t2m.on) TRY(pack_t2m(h));
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
  if (k.sigma != 0.0f && !noise)
    FAIL(MLDB_ERR_INVALID, "the step at t = %lld adds noise (%s) and needs the injected N(0,1) noise tensor",
         (long long)timestep, k.kind == 0 ? "DDIM eta > 0" : "DDPM t > 0");
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
    if (e != cudaSuccess) {
      (void)cudaGetLastError();   // the launch error that broke the capture must not fail the next, unrelated call
      FAIL(MLDB_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
    }
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

// Does some step of the current timestep schedule add noise (non-zero std / sigma)?
static bool steps_add_noise(const mldb_handle* h) {
  for (const StepCoef& k : h->coefs_host)
    if (k.sigma != 0.0f) return true;
  return false;
}

static int run_reverse(mldb_handle* h, const void* cond, const float* init_noise, const float* step_noise,
                       const int32_t* lengths, int B, int S, int T, float* latents_out, cudaStream_t st,
                       Plan** plan_out) {
  const mldb_config& c = h->cfg;
  if (c.num_layers == 0) FAIL(MLDB_ERR_STATE, "this handle has no denoiser");
  const bool cfg_on = c.guidance_scale > 1.0f;
  const int Bx = cfg_on ? 2 * B : B;
  if (c.arch == MLDB_ARCH_TRANS_DEC) {
    // no-VAE model: latents are the motion itself, [B, T, F]; DDPM (and DDIM with eta > 0) adds noise at
    // its steps, which the caller injects (step_noise [n_steps, B, T, F]).  One captured step, replayed.
    if (!c.diffusion_only) FAIL(MLDB_ERR_UNSUPPORTED, "arch trans_dec is built for the no-VAE model (diffusion_only)");
    if (!lengths || T <= 0) FAIL(MLDB_ERR_INVALID, "the no-VAE model needs lengths and T");
    const int nsteps = (int)h->timesteps.size();
    const bool needs_noise = steps_add_noise(h);
    if (needs_noise && !step_noise)
      FAIL(MLDB_ERR_INVALID, "this scheduler adds noise at its steps (%s): pass step_noise [%d, %d, %d, %d] (N(0,1) per step)",
           c.sched_kind == MLDB_SCHED_DDIM ? "DDIM eta > 0" : "DDPM", nsteps, B, T, c.nfeats);
    Plan* p = nullptr;
    TRY(decden_plan(h, 5, B, Bx, S, T, &p));
    const int64_t per = (int64_t)T * c.nfeats;
    TRY(place_condition_dec(h, p, cond, st));
    k_dup_lengths<<<nblk(Bx), 256, 0, st>>>(lengths, p->lengths, B, Bx);
    kcount(h, MLDB_KSTAT_MISC);
    CK(cudaMemcpyAsync(p->latents, init_noise, (size_t)B * per * sizeof(float), cudaMemcpyDeviceToDevice, st));
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
  // DDPM (every step with t > 0) and DDIM with eta > 0 (every step) add std * N(0,1) (diffusers
  // scheduler.step draws it): the caller injects the draws
  const float* nz_all = nullptr;
  if (steps_add_noise(h)) {
    if (!step_noise)
      FAIL(MLDB_ERR_INVALID, "this scheduler adds noise at its steps (%s): pass step_noise [%d, %d, %d, %d] (N(0,1) per step)",
           c.sched_kind == MLDB_SCHED_DDIM ? "DDIM eta > 0" : "DDPM", nsteps, B, c.n_lat, d);
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
// the first n elements of a split16 buffer whose rows are contiguous (cols == leading dimension), widened to fp32
__global__ void k_split_to_f32(ActBuf X, float* __restrict__ out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = join_f32(X.hi[i], X.lo()[i]);
}
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
  const bool actor = c.vae_kind == MLDB_VAE_ACTOR;
  if (c.vae_kind != MLDB_VAE_MLD && !actor) FAIL(MLDB_ERR_UNSUPPORTED, "encode needs a VAE (MldVae or ActorVae)");
  if (actor && h->venc.enc.empty())
    FAIL(MLDB_ERR_STATE, "the ActorVae encoder was not loaded: the state dict held no 'vae.encoder.*' keys");
  if (actor && c.n_lat != 1) FAIL(MLDB_ERR_UNSUPPORTED, "the ActorVae encoder yields one latent token, not n_lat = %d", c.n_lat);
  cudaStream_t st = (cudaStream_t)stream;
  const int d = c.latent_dim, G = 2 * c.n_lat, L = G + T;
  if (L > h->vae_enc_pe_rows)
    FAIL(MLDB_ERR_INVALID, "T + %d = %d tokens exceed the encoder's positional table (%d rows)", G, L, h->vae_enc_pe_rows);
  Plan* p = find_plan(h, 2, B, 0, T);
  if (!p) {
    p = add_plan(h, 2, B, 0, T);
    // the last layer runs trimmed to the G distribution rows (ActorVae: always; MldVae: when it has skip blocks)
    TRY(alloc_stack_ws(h, h->venc, B, L, 0, &p->ws, actor || h->venc.layers >= 3 ? G : 0));
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
  // global motion tokens (b, 0..G-1) = token + PE (mld_vae.py:146,157; actor_vae.py:144-165)
  k_rows_to_split<<<nblk((int64_t)B * G * d), 256, 0, st>>>(p->ws.x0, h->global_token, d, B * G, d, G, L, 0, 1, h->vae_enc_pe);
  kcount(h, MLDB_KSTAT_MISC);
  SeqInfo si; si.lengths = p->lengths; si.kv_prefix = G;
  ActBuf x = run_stack(h, h->venc, p->ws.x0, ActBuf{}, p->ws, si, st);
  if (actor) {   // no final norm: the trimmed layer's (b, mu | logvar) rows are the distribution (actor_vae.py:169)
    k_split_to_f32<<<nblk((int64_t)B * G * d), 256, 0, st>>>(x, p->stage_f32, (int64_t)B * G * d);
    kcount(h, MLDB_KSTAT_MISC);
    k_rows_out_permuted<<<nblk((int64_t)B * G * d), 256, 0, st>>>(p->stage_f32, mu, logvar, B, 1, d);
    kcount(h, MLDB_KSTAT_MISC);
    CK(cudaGetLastError());
    return check_ops(h);
  }
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
  k_feats2joints<<<B, 256, 0, st>>>(feats, h->mean, h->stdv, T, F, c.njoints, joints);
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
                           float* latents_out, float* feats_out, float* joints_out, void* stream,
                           const float* step_noise) {
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
  TRY(run_reverse(h, cond, init_noise, step_noise, lengths, B, S_ctx, T, z, st, &rp));
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
                                  float* joints_global, void* stream, const float* step_noise) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!joints_global) FAIL(MLDB_ERR_INVALID, "bad argument");
  const int64_t count = (int64_t)B * T * h->cfg.njoints * 3;
  cudaStream_t st = (cudaStream_t)stream;
  if (!h->nccl_comm) {      // single rank: the gather is the identity
    return mldb_sample(h, cond, init_noise, lengths, B, S_ctx, T, nullptr, nullptr, joints_global, stream, step_noise);
  }
  TRY(mldb_gather_begin(h, st));
  TRY(mldb_sample(h, cond, init_noise, lengths, B, S_ctx, T, nullptr, nullptr, joints_global + h->comm_rank * count, stream,
                  step_noise));
  return mldb_gather_async(h, joints_global, count, st);
}

// Host-buffer entry point.  With a communicator attached joints_host receives the GATHERED motions
// [nranks * B, T, njoints, 3] (every rank holds all of them after the all-gather), else [B, T, njoints, 3].
extern "C" int mldb_sample_host(mldb_handle* h, const void* cond_host, const float* init_noise_host,
                                const int32_t* lengths_host, int32_t B, int32_t S_ctx, int32_t T,
                                float* joints_host, void* stream, const float* step_noise_host) {
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
  // per-step noise [n_steps, B, n_lat, d]: staged in the decode plan's step_noise buffer (unused by decoding)
  const float* step_noise = nullptr;
  if (step_noise_host) {
    const size_t n = h->timesteps.size() * (size_t)B * c.n_lat * c.latent_dim;
    if (dp->noise_cap < n) {
      TRY(dev_alloc(h, (void**)&dp->step_noise, n * sizeof(float)));
      dp->noise_cap = n;
    }
    CK(cudaMemcpyAsync(dp->step_noise, step_noise_host, n * sizeof(float), cudaMemcpyHostToDevice, st));
    step_noise = dp->step_noise;
  }
  if (world > 1) {
    TRY(mldb_sample_gather(h, dp->cond_f, dp->noise_in, (const int32_t*)dp->cond_i, B, S_ctx, T, dp->joints_all, stream,
                           step_noise));
    TRY(mldb_gather_wait(h, stream));
    CK(cudaMemcpyAsync(joints_host, dp->joints_all, world * joints_elems * sizeof(float), cudaMemcpyDeviceToHost, st));
    return MLDB_OK;
  }
  TRY(mldb_sample(h, dp->cond_f, dp->noise_in, (const int32_t*)dp->cond_i, B, S_ctx, T, nullptr, nullptr, dp->joints, stream,
                  step_noise));
  CK(cudaMemcpyAsync(joints_host, dp->joints, joints_elems * sizeof(float), cudaMemcpyDeviceToHost, st));
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- profiling aid
// Time one operator of denoiser layer 0 in isolation on the real workspace of the (B, S_ctx)
// reverse plan: `iters` back-to-back launches bracketed by CUDA events on `stream`.
// op: "qkv" | "attn" | "outproj_ln" | "ffn1" | "ffn2_ln" | "ffn" | "tail" | "tail_fused" | "layer".  "outproj_ln" and
// "ffn" time the standalone kernels; "tail" is both as the encoder layer runs them (op_tail), "tail_fused" the fused
// launch at any row count.
// avg_ms_out: HOST float.
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
    } else if (!strcmp(op, "tail")) {            // out-projection + LN1 + FFN + LN2 the way the stack runs them
      op_tail(h, w.out_proj, w.n1, w.l1, w.l2, w.n2, ws.att, ws.x0, ws.x1, ws.h, ws.cur[0], ws.M, d, ws.ff, ws.cf32, st);
    } else if (!strcmp(op, "tail_fused")) {      // the same with the fused launch whatever the row count
      op_tail(h, w.out_proj, w.n1, w.l1, w.l2, w.n2, ws.att, ws.x0, ws.x1, ws.h, ws.cur[0], ws.M, d, ws.ff, ws.cf32, st, 2);
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


// ----------------------------------------------------------------------------- CLIP text tower: forward
static void op_text_ln(mldb_handle* h, const TextLnArgs& a, cudaStream_t st) { text_ln(a, st); kcount(h, MLDB_KSTAT_TEXT_LN); }

// grow the text workspace to `rows` tokens / `seqs` sequences (outside any capture; synchronises the device)
static int text_workspace(mldb_handle* h, int rows, int seqs) {
  TextW& tw = h->text;
  if (rows <= tw.rows && seqs <= tw.seqs) return MLDB_OK;
  rows = std::max(rows, tw.rows); seqs = std::max(seqs, tw.seqs);
  CK(cudaDeviceSynchronize());                      // the old buffers may still be in use by enqueued work
  for (void* p : tw.ws_allocs) cudaFree(p);
  tw.ws_allocs.clear();
  tw.rows = tw.seqs = 0;
  auto alloc = [&](size_t bytes, void** p) -> int {
    CK(cudaMalloc(p, bytes ? bytes : 16));
    tw.ws_allocs.push_back(*p);
    CK(cudaMemset(*p, 0, bytes));
    return MLDB_OK;
  };
  auto act = [&](int r, int cols, ActBuf* out) -> int {
    const int64_t rp = ((int64_t)r + 127) / 128 * 128;
    TRY(alloc((size_t)2 * rp * cols * sizeof(__half), (void**)&out->hi));
    out->plane_stride = rp * cols; out->rows = r; out->cols = cols;
    return MLDB_OK;
  };
  const mldb_text_config& c = tw.cfg;
  TRY(alloc((size_t)rows * c.hidden * sizeof(float), (void**)&tw.x));
  TRY(act(rows, c.hidden, &tw.a));
  TRY(act(rows, 3 * c.hidden, &tw.qkv));
  TRY(act(rows, c.hidden, &tw.att));
  TRY(act(rows, c.ff, &tw.h));
  TRY(act(seqs, c.hidden, &tw.pooled));
  tw.rows = rows; tw.seqs = seqs;
  return MLDB_OK;
}

extern "C" int mldb_text_encode(mldb_handle* h, const int64_t* ids, int32_t n, int32_t L, int32_t mode, float* out,
                                void* stream) {
  if (!h || !ids || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  TextW& tw = h->text;
  if (!tw.on) FAIL(MLDB_ERR_STATE, "the text tower is not configured (mldb_text_configure)");
  if (!h->finalized) FAIL(MLDB_ERR_STATE, "finalize weights first");
  const mldb_text_config& c = tw.cfg;
  if (n < 1 || L < 1 || L > c.max_positions) FAIL(MLDB_ERR_INVALID, "ids must be [n >= 1, 1 <= L <= %d]", c.max_positions);
  if ((int64_t)n * L > (1 << 30)) FAIL(MLDB_ERR_INVALID, "too many tokens");
  if (mode != MLDB_TEXT_HIDDEN && mode != MLDB_TEXT_POOLED) FAIL(MLDB_ERR_INVALID, "mode must be MLDB_TEXT_HIDDEN or MLDB_TEXT_POOLED");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int M = n * L, d = c.hidden;
  TRY(text_workspace(h, M, n));
  auto rows = [&](ActBuf b, int r) { b.rows = r; return b; };
  const ActBuf a = rows(tw.a, M), qkv = rows(tw.qkv, M), att = rows(tw.att, M), hid = rows(tw.h, M);
  auto ln = [&](int m, const LnW& w) {
    TextLnArgs l; l.mode = m; l.x = tw.x; l.ids = ids; l.L = L; l.tok = tw.tok; l.pos = tw.pos; l.vocab = c.vocab_size;
    l.eos_id = c.eos_token_id; l.gamma = w.g; l.beta = w.b; l.eps = c.ln_eps; l.M = M; l.d = d; l.out = a;
    return l;
  };
  op_text_ln(h, ln(TEXT_LN_EMBED, tw.layers[0].ln1), st);          // x = tok[id] + pos[t]; a = LN1_0(x)
  for (int i = 0; i < c.layers; ++i) {
    const TextLayerW& w = tw.layers[i];
    GemmArgs g; g.a1 = a; g.K1 = d; g.M = M; g.w = w.qkv; g.out = qkv; g.wide_n = 1;
    op_gemm(h, g, st);
    AttnArgs at; at.q = qkv; at.q_col0 = 0; at.Lq = L; at.kv = qkv; at.k_col0 = d; at.v_col0 = 2 * d; at.Lk = L;
    at.nseq = n; at.heads = c.heads; at.hd = d / c.heads; at.causal = 1; at.out = att;
    op_attn(h, at, st);
    GemmArgs go; go.a1 = att; go.K1 = d; go.M = M; go.w = w.out; go.out_f32 = tw.x; go.ldc = d; go.res_f32 = tw.x;
    op_gemm(h, go, st);                                              // x += out_proj(att), in place
    op_text_ln(h, ln(TEXT_LN_ROWS, w.ln2), st);
    GemmArgs g1; g1.a1 = a; g1.K1 = d; g1.M = M; g1.w = w.fc1; g1.act = ACT_QUICKGELU; g1.out = hid; g1.wide_n = 1;
    op_gemm(h, g1, st);
    GemmArgs g2; g2.a1 = hid; g2.K1 = c.ff; g2.M = M; g2.w = w.fc2; g2.out_f32 = tw.x; g2.ldc = d; g2.res_f32 = tw.x;
    op_gemm(h, g2, st);                                              // x += fc2(quick_gelu(fc1(LN2(x))))
    if (i + 1 < c.layers) op_text_ln(h, ln(TEXT_LN_ROWS, tw.layers[i + 1].ln1), st);
  }
  if (mode == MLDB_TEXT_HIDDEN) {
    TextLnArgs l = ln(TEXT_LN_ROWS, tw.final_ln);
    l.out = ActBuf{}; l.out_f32 = out;                             // last_hidden_state, every row
    op_text_ln(h, l, st);
  } else {
    TextLnArgs l = ln(TEXT_LN_EOS, tw.final_ln);
    l.M = n; l.out = rows(tw.pooled, n);                           // only the n eos rows
    op_text_ln(h, l, st);
    GemmArgs gp; gp.a1 = l.out; gp.K1 = d; gp.M = n; gp.w = tw.proj; gp.out_f32 = out; gp.ldc = c.projection_dim;
    gp.wide_n = 1;
    op_gemm(h, gp, st);                                              // text_projection (no bias)
  }
  CK(cudaGetLastError());
  return check_ops(h);
}

// ----------------------------------------------------------------------------- T2M evaluator: forward
// Workspace slot i grown to `bytes` (outside any capture; synchronises the device when it grows).  Zero-filled when
// allocated; every kernel that writes a slot writes all of the region it later reads.
static int t2m_slot(mldb_handle* h, int i, size_t bytes, void** out) {
  T2mW& t = h->t2m;
  if (bytes > t.cap[i]) {
    CK(cudaDeviceSynchronize());                    // the old buffer may still be in use by enqueued work
    cudaFree(t.buf[i]);
    t.buf[i] = nullptr; t.cap[i] = 0;
    CK(cudaMalloc(&t.buf[i], bytes));
    CK(cudaMemset(t.buf[i], 0, bytes));
    t.cap[i] = bytes;
  }
  *out = t.buf[i];
  return MLDB_OK;
}
static int t2m_act(mldb_handle* h, int i, int rows, int cols, ActBuf* out) {
  __half* p = nullptr;
  TRY(t2m_slot(h, i, (size_t)2 * rows * cols * sizeof(__half), (void**)&p));
  out->hi = p; out->plane_stride = (int64_t)rows * cols; out->rows = rows; out->cols = cols;
  return MLDB_OK;
}
// sequences per chunk: the option, else what keeps the chunk's workspace near 1 GiB (whole 128-row tiles when > 128)
static int t2m_chunk(const mldb_handle* h, int B, size_t per_seq) {
  if (h->t2m.chunk > 0) return std::min(B, h->t2m.chunk);
  int c = (int)std::max<size_t>(1, ((size_t)1 << 30) / per_seq);
  if (c > 128) c = c / 128 * 128;
  return std::min(B, c);
}
static size_t gru_bytes_per_seq(int L, int in, int H) {
  return (size_t)L * (4 * in + 24 * H) + (size_t)40 * H;   // x (split16), gi (fp32), state and head
}
static int t2m_ready(mldb_handle* h, int part, const char* name) {
  if (!h->t2m.on || !(h->t2m.cfg.parts & part)) FAIL(MLDB_ERR_STATE, "the T2M %s encoder is not configured (mldb_t2m_configure)", name);
  if (!h->finalized) FAIL(MLDB_ERR_STATE, "finalize weights first");
  return MLDB_OK;
}

// Bidirectional GRU over x [n * L, in] (split16, row b * L + t) and the BiGRUCo head -> out [n, out_dim] fp32.
static int gru_forward(mldb_handle* h, const GruW& g, ActBuf x, const int32_t* lengths, int n, int L, float* out,
                       int out_dim, cudaStream_t st) {
  const int H = g.H, rows_pad = (n + 127) / 128 * 128;
  float* gi = nullptr;
  TRY(t2m_slot(h, 1, (size_t)n * L * 6 * H * sizeof(float), (void**)&gi));
  for (int d = 0; d < 2; ++d) {                    // gi = x W_ih^T + b_ih, every step of both directions
    GemmArgs ga; ga.a1 = x; ga.K1 = x.cols; ga.M = n * L; ga.w = g.w_ih[d]; ga.out_f32 = gi + (size_t)d * 3 * H;
    ga.ldc = 6 * H; ga.wide_n = 1; ga.vec_f32 = 1;
    op_gemm(h, ga, st);
  }
  const size_t plane = (size_t)2 * rows_pad * H;
  __half* hs = nullptr;
  float* hf = nullptr;
  TRY(t2m_slot(h, 3, 2 * 2 * plane * sizeof(__half), (void**)&hs));   // ping-pong split16 state
  TRY(t2m_slot(h, 4, 2 * plane * sizeof(float), (void**)&hf));        // ping-pong fp32 state
  float* gh = nullptr;
  if (!h->use_tc) TRY(t2m_slot(h, 9, plane * 3 * sizeof(float), (void**)&gh));
  auto state = [&](int b) {
    ActBuf a; a.hi = hs + (size_t)b * 2 * plane; a.plane_stride = (int64_t)plane; a.rows = 2 * rows_pad; a.cols = H;
    return a;
  };
  GruStepArgs a;
  a.gi = gi; a.gh = gh; a.b_hh = g.b_hh; a.lengths = lengths; a.w_hh = g.w_hh.w; a.w_plane_stride = g.w_hh.plane_stride;
  a.w_inv_scale = g.w_hh.inv_scale; a.rows = n; a.rows_pad = rows_pad; a.L = L; a.H = H;
  a.h_out = state(0); a.hf_out = hf;
  gru_init_state(a, g.h0, st);
  kcount(h, MLDB_KSTAT_MISC);
  for (int s = 0; s < L; ++s) {
    a.step = s;
    a.h_in = state(s & 1); a.hf_in = hf + (s & 1) * plane;
    a.h_out = state((s + 1) & 1); a.hf_out = hf + ((s + 1) & 1) * plane;
    if (h->use_tc) {
      if (!gru_step_tc(a, st)) h->op_failed = true;
      kcount(h, MLDB_KSTAT_GRU_TC);
    } else {                                       // gemm=simt: h W_hh^T per direction on CUDA cores, then the gates
      for (int d = 0; d < 2; ++d) {
        LinW w = g.w_hh;
        w.w += (size_t)d * 3 * H * H; w.N = 3 * H;
        GemmArgs gg; gg.a1 = rows_of(a.h_in, (int64_t)d * rows_pad, n); gg.K1 = H; gg.M = n; gg.w = w;
        gg.out_f32 = gh + (size_t)d * rows_pad * 3 * H; gg.ldc = 3 * H; gg.wide_n = 1;
        op_gemm(h, gg, st);
      }
      gru_gate_simt(a, st);
      kcount(h, MLDB_KSTAT_MISC);
    }
  }
  // head: cat(h_fwd final, h_bwd final) -> Linear -> LayerNorm -> LeakyReLU -> Linear
  const ActBuf fin = state(L & 1);
  float* cf = nullptr;
  TRY(t2m_slot(h, 5, (size_t)n * H * sizeof(float), (void**)&cf));
  ActBuf ln_out;
  TRY(t2m_act(h, 6, n, H, &ln_out));
  GemmArgs g1; g1.a1 = rows_of(fin, 0, n); g1.K1 = H; g1.a2 = rows_of(fin, rows_pad, n); g1.K2 = H; g1.M = n;
  g1.w = g.head1; g1.out_f32 = cf; g1.ldc = H; g1.vec_f32 = 1;
  op_gemm(h, g1, st);
  LnArgs l; l.c = cf; l.ldc = H; l.gamma = g.ln.g; l.beta = g.ln.b; l.M = n; l.d = H; l.out = ln_out; l.act = ACT_LEAKY;
  op_ln(h, l, st);
  GemmArgs g2; g2.a1 = ln_out; g2.K1 = H; g2.M = n; g2.w = g.head2; g2.out_f32 = out; g2.ldc = out_dim; g2.wide_n = 1;
  g2.vec_f32 = 1;
  op_gemm(h, g2, st);
  return MLDB_OK;
}

extern "C" int mldb_t2m_movement(mldb_handle* h, const float* x, int32_t ld, int32_t B, int32_t T, float* out,
                                 void* stream) {
  if (!h || !x || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(t2m_ready(h, MLDB_T2M_MOVEMENT, "movement"));
  const mldb_t2m_config& c = h->t2m.cfg;
  if (B < 1 || T < 4) FAIL(MLDB_ERR_INVALID, "movement encoder input must be [B >= 1, T >= 4, %d], got B=%d T=%d", c.dim_pose, B, T);
  if (ld < c.dim_pose) FAIL(MLDB_ERR_INVALID, "row stride ld=%d is smaller than dim_pose=%d", ld, c.dim_pose);
  if ((int64_t)B * T * ld > ((int64_t)1 << 40)) FAIL(MLDB_ERR_INVALID, "input too large");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int C = c.dim_pose, Cp = (C + 15) / 16 * 16, hid = c.dim_move_hidden, lat = c.dim_move_latent;
  const int T1 = T / 2, T2 = T1 / 2;
  const size_t per_seq = (size_t)T1 * (16 * Cp + 4 * hid) + (size_t)T2 * (16 * hid + 4 * lat);
  const int Bc = t2m_chunk(h, B, per_seq);
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0);
    ActBuf a1, a2, z;
    float* y1 = nullptr;
    TRY(t2m_act(h, 0, n * T1, 4 * Cp, &a1));
    TRY(t2m_slot(h, 1, (size_t)n * T1 * hid * sizeof(float), (void**)&y1));
    TRY(t2m_act(h, 2, n * T2, 4 * hid, &a2));
    TRY(t2m_act(h, 7, n * T2, lat, &z));
    im2col_k4s2(a1, x + (int64_t)b0 * T * ld, ld, T, C, Cp, T1, n * T1, st);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs g1; g1.a1 = a1; g1.K1 = 4 * Cp; g1.M = n * T1; g1.w = h->t2m.conv1; g1.act = ACT_LEAKY; g1.out_f32 = y1;
    g1.ldc = hid; g1.wide_n = 1; g1.vec_f32 = 1;
    op_gemm(h, g1, st);                            // main.0 + LeakyReLU (dropout: identity in eval)
    im2col_k4s2(a2, y1, hid, T1, hid, hid, T2, n * T2, st);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs g2; g2.a1 = a2; g2.K1 = 4 * hid; g2.M = n * T2; g2.w = h->t2m.conv2; g2.act = ACT_LEAKY; g2.out = z;
    g2.wide_n = 1;
    op_gemm(h, g2, st);                            // main.3 + LeakyReLU
    GemmArgs g3; g3.a1 = z; g3.K1 = lat; g3.M = n * T2; g3.w = h->t2m.move_out; g3.out_f32 = out + (int64_t)b0 * T2 * lat;
    g3.ldc = lat; g3.wide_n = 1; g3.vec_f32 = 1;
    op_gemm(h, g3, st);                            // out_net
  }
  CK(cudaGetLastError());
  return check_ops(h);
}

extern "C" int mldb_t2m_motion(mldb_handle* h, const float* x, const int32_t* lengths, int32_t B, int32_t L, float* out,
                               void* stream) {
  if (!h || !x || !lengths || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(t2m_ready(h, MLDB_T2M_MOTION, "motion"));
  const mldb_t2m_config& c = h->t2m.cfg;
  if (B < 1 || L < 1 || (int64_t)B * L > (1 << 26)) FAIL(MLDB_ERR_INVALID, "motion encoder input must be [B >= 1, L >= 1, %d], got B=%d L=%d", c.dim_move_latent, B, L);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int In = c.dim_move_latent, H = c.dim_motion_hidden;
  const int Bc = t2m_chunk(h, B, gru_bytes_per_seq(L, In + H, H));
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0);
    ActBuf xs, e;
    TRY(t2m_act(h, 0, n * L, In, &xs));
    TRY(t2m_act(h, 2, n * L, H, &e));
    k_f32_to_split_pad<<<nblk((int64_t)n * L * In), 256, 0, st>>>(xs, x + (int64_t)b0 * L * In, In, n * L, In, 1);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs g; g.a1 = xs; g.K1 = In; g.M = n * L; g.w = h->t2m.motion_in; g.out = e; g.wide_n = 1;
    op_gemm(h, g, st);                             // input_emb
    TRY(gru_forward(h, h->t2m.motion_gru, e, lengths + b0, n, L, out + (int64_t)b0 * c.dim_motion_latent,
                    c.dim_motion_latent, st));
  }
  CK(cudaGetLastError());
  return check_ops(h);
}

extern "C" int mldb_t2m_text(mldb_handle* h, const float* word_embs, const float* pos_ohot, const int32_t* lengths,
                             int32_t B, int32_t L, float* out, void* stream) {
  if (!h || !word_embs || !pos_ohot || !lengths || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(t2m_ready(h, MLDB_T2M_TEXT, "text"));
  const mldb_t2m_config& c = h->t2m.cfg;
  if (B < 1 || L < 1 || (int64_t)B * L > (1 << 26)) FAIL(MLDB_ERR_INVALID, "text encoder input must be [B >= 1, L >= 1, *], got B=%d L=%d", B, L);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int W = c.dim_word, P = c.dim_pos_ohot, H = c.dim_text_hidden;
  const int Bc = t2m_chunk(h, B, gru_bytes_per_seq(L, pad64(P) + 2 * W + pad64(W) + H, H));
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0), M = n * L;
    ActBuf ps, xs, e;
    float* xw = nullptr;
    TRY(t2m_act(h, 0, M, pad64(P), &ps));
    TRY(t2m_slot(h, 7, (size_t)M * W * sizeof(float), (void**)&xw));
    TRY(t2m_act(h, 8, M, pad64(W), &xs));
    TRY(t2m_act(h, 2, M, H, &e));
    k_f32_to_split_pad<<<nblk((int64_t)M * ps.cols), 256, 0, st>>>(ps, pos_ohot + (int64_t)b0 * L * P, P, M, P, 1);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs gp; gp.a1 = ps; gp.K1 = ps.cols; gp.M = M; gp.w = h->t2m.pos_emb; gp.out_f32 = xw; gp.ldc = W;
    gp.res_f32 = word_embs + (int64_t)b0 * L * W; gp.wide_n = 1;
    op_gemm(h, gp, st);                            // word_embs + pos_emb(pos_ohot)
    k_f32_to_split_pad<<<nblk((int64_t)M * xs.cols), 256, 0, st>>>(xs, xw, W, M, W, 1);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs g; g.a1 = xs; g.K1 = xs.cols; g.M = M; g.w = h->t2m.text_in; g.out = e; g.wide_n = 1;
    op_gemm(h, g, st);                             // input_emb
    TRY(gru_forward(h, h->t2m.text_gru, e, lengths + b0, n, L, out + (int64_t)b0 * c.dim_coemb_hidden,
                    c.dim_coemb_hidden, st));
  }
  CK(cudaGetLastError());
  return check_ops(h);
}

// ----------------------------------------------------------------------------- debug aid
// y = act(A W^T + b) or LayerNorm(A W^T + b + R) through the engine's GEMM operators, so tests can
// compare the wgmma kernels with the CUDA-core kernels (and with torch) shape by shape.
//   A [M,K] fp32 device; W [N,K], bias [N], gamma/beta [N] fp32 HOST (gamma == NULL: no LN);
//   R [M,N] fp32 device or NULL; K1 < K splits A into two concatenated sources (skip connection);
//   out [M,N] fp32 device.  use_tc: 1 tensor-core path, 0 CUDA-core path.  Synchronous.
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
  GemmArgs ga; ga.a1 = a1; ga.K1 = K1; ga.a2 = a2; ga.K2 = K - K1; ga.M = M; ga.w = w; ga.act = act; ga.wide_n = 1;
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
  } else if (R) {                                  // residual add, fp32 out (in place when R == out)
    ga.res_f32 = R; ga.out_f32 = out; ga.ldc = N;
    op_gemm(h, ga, st);
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

extern "C" int mldb_debug_tail(mldb_handle* h, const float* att, const float* X, const float* Wo, const float* bo,
                               const float* gamma1, const float* beta1, const float* W1, const float* b1,
                               const float* W2, const float* b2, const float* gamma2, const float* beta2, int32_t M,
                               int32_t d, int32_t ff, int32_t mode, int32_t out_rows, float* out, void* stream) {
  if (!h || !att || !X || !Wo || !gamma1 || !beta1 || !W1 || !W2 || !gamma2 || !beta2 || !out || M <= 0 || d <= 0 ||
      ff <= 0 || out_rows < M)
    FAIL(MLDB_ERR_INVALID, "bad argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_alloc0 = h->allocs.size();
  LinW wo, l1, l2;
  LnW n1, n2;
  TRY(pack_linear(h, Wo, d, d, bo, &wo));
  TRY(pack_linear(h, W1, ff, d, b1, &l1));
  TRY(pack_linear(h, W2, d, ff, b2, &l2));
  TRY(upload_f32(h, gamma1, d, &n1.g));
  TRY(upload_f32(h, beta1, d, &n1.b));
  TRY(upload_f32(h, gamma2, d, &n2.g));
  TRY(upload_f32(h, beta2, d, &n2.b));
  ActBuf a, x, x1, hb, o;
  float* cf32 = nullptr;
  TRY(alloc_act(h, M, d, &a));
  TRY(alloc_act(h, M, d, &x));
  TRY(alloc_act(h, M, d, &x1));
  TRY(alloc_act(h, M, ff, &hb));
  TRY(alloc_act(h, out_rows, d, &o));
  TRY(dev_alloc(h, (void**)&cf32, (size_t)M * d * sizeof(float)));
  k_rows_to_split<<<nblk((int64_t)out_rows * d), 256, 0, st>>>(o, out, d, out_rows, d, 1 << 30, 0, 0, 0, nullptr);
  k_rows_to_split<<<nblk((int64_t)M * d), 256, 0, st>>>(a, att, d, M, d, 1 << 30, 0, 0, 0, nullptr);
  k_rows_to_split<<<nblk((int64_t)M * d), 256, 0, st>>>(x, X, d, M, d, 1 << 30, 0, 0, 0, nullptr);
  const bool saved = h->use_tc;
  h->use_tc = mode != 0;
  const int saved_fused = tc_set_ffn_fused(h->tc, 1);
  op_tail(h, wo, n1, l1, l2, n2, a, x, x1, hb, o, M, d, ff, cf32, st, mode == 2 ? 2 : 0);
  h->use_tc = saved;
  tc_set_ffn_fused(h->tc, saved_fused);
  k_split_to_f32<<<nblk((int64_t)out_rows * d), 256, 0, st>>>(o, out, (int64_t)out_rows * d);
  cudaError_t e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  while (h->allocs.size() > n_alloc0) { cudaFree(h->allocs.back()); h->allocs.pop_back(); }
  if (e != cudaSuccess) FAIL(MLDB_ERR_CUDA, "debug tail: %s", cudaGetErrorString(e));
  return MLDB_OK;
}

static int debug_attention(mldb_handle* h, const float* Q, const float* KV, const int32_t* lengths, int32_t kv_prefix,
                           int32_t nseq, int32_t Lq, int32_t Lk, int32_t heads, int32_t hd, int32_t mode, int causal,
                           float* out, void* stream) {
  if (!h || !Q || !out || nseq <= 0 || Lq <= 0 || Lk <= 0 || heads <= 0 || hd <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  if (!KV && Lq != Lk) FAIL(MLDB_ERR_INVALID, "a packed QKV input is self-attention: Lq must equal Lk");
  if (causal && KV) FAIL(MLDB_ERR_INVALID, "causal attention is self-attention: pass a packed QKV input (KV == NULL)");
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
  a.causal = causal;
  int rc = MLDB_OK;
  if (mode == 0 && simt_attention_supported(hd)) { if (!simt_attention(a, st)) rc = MLDB_ERR_UNSUPPORTED; }
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
extern "C" int mldb_debug_attention(mldb_handle* h, const float* Q, const float* KV, const int32_t* lengths,
                                    int32_t kv_prefix, int32_t nseq, int32_t Lq, int32_t Lk, int32_t heads, int32_t hd,
                                    int32_t mode, float* out, void* stream) {
  return debug_attention(h, Q, KV, lengths, kv_prefix, nseq, Lq, Lk, heads, hd, mode, 0, out, stream);
}
extern "C" int mldb_debug_attention_causal(mldb_handle* h, const float* Q, const float* KV, const int32_t* lengths,
                                           int32_t kv_prefix, int32_t nseq, int32_t Lq, int32_t Lk, int32_t heads,
                                           int32_t hd, int32_t mode, float* out, void* stream) {
  return debug_attention(h, Q, KV, lengths, kv_prefix, nseq, Lq, Lk, heads, hd, mode, 1, out, stream);
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
