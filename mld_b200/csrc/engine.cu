// libmldb200 engine: handles and their options, the state-dict spec and weight packing of the sampling models,
// scheduler tables, plans and CUDA-graph capture.  The models' forward passes live in stack.cu (transformer stacks),
// denoiser.cu, vae.cu, text_tower.cu, t2m.cu, a2m.cu, stgcn.cu and smpl.cu.
#include "engine.h"

#include <math.h>
#include <string.h>

#include <algorithm>

#include "gemm_tc.h"
#include "misc_kernels.cuh"

// ----------------------------------------------------------------------------- errors
static thread_local std::string g_err;
void mldb_set_err(const std::string& s) { g_err = s; }
extern "C" const char* mldb_last_error(void) { return g_err.c_str(); }
extern "C" int mldb_abi_version(void) { return MLDB_ABI_VERSION; }

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
void spec_add(mldb_handle* h, const std::string& key, std::vector<int64_t> shape) {
  RawTensor t; t.shape = std::move(shape);
  h->raw[key] = std::move(t);
}
static void spec_attn(mldb_handle* h, const std::string& p, int d) {
  spec_add(h, p + "in_proj_weight", {3 * d, d});
  spec_add(h, p + "in_proj_bias", {3 * d});
  spec_add(h, p + "out_proj.weight", {d, d});
  spec_add(h, p + "out_proj.bias", {d});
}
void spec_ln(mldb_handle* h, const std::string& p, int d) {
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
int dev_alloc(mldb_handle* h, void** p, size_t bytes) {
  CK(cudaMalloc(p, bytes ? bytes : 16));
  h->allocs.push_back(*p);
  return MLDB_OK;
}
// Grow b to at least `bytes`, zero-filled (outside any capture).  Synchronises the device first: enqueued work may
// still use the old buffer.
int may_configure(const mldb_handle* h, int abi_version, int expected, bool on, const char* name, const char* what) {
  if (abi_version != expected) FAIL(MLDB_ERR_INVALID, "mldb_%s_config abi_version mismatch", name);
  if (h->finalized) FAIL(MLDB_ERR_STATE, "mldb_%s_configure must precede mldb_finalize_weights", name);
  if (on) FAIL(MLDB_ERR_STATE, "%s is already configured", what);
  return MLDB_OK;
}
int check_configured(const mldb_handle* h, bool on, const char* name, const char* what) {
  if (!on) FAIL(MLDB_ERR_STATE, "%s is not configured (mldb_%s_configure)", what, name);
  if (!h->finalized) FAIL(MLDB_ERR_STATE, "finalize weights first");
  return MLDB_OK;
}
int eval_chunk(int option, int B, size_t per_seq, int round) {
  if (option > 0) return std::min(B, option);
  int c = (int)std::max<size_t>(1, ((size_t)1 << 30) / per_seq);
  if (c > round) c = c / round * round;
  return std::min(B, c);
}
int grow(GrowBuf& b, size_t bytes) {
  if (bytes <= b.cap) return MLDB_OK;
  CK(cudaDeviceSynchronize());
  cudaFree(b.p);
  b.p = nullptr; b.cap = 0;
  CK(cudaMalloc(&b.p, bytes));
  CK(cudaMemset(b.p, 0, bytes));
  b.cap = bytes;
  return MLDB_OK;
}
int grow_act(GrowBuf& b, int rows, int cols, ActBuf* out) {
  TRY(grow(b, split16_bytes(rows, cols)));
  *out = split16_at(b.p, rows, cols);
  return MLDB_OK;
}
int upload_f32(mldb_handle* h, const float* src, size_t n, float** out) {
  TRY(dev_alloc(h, (void**)out, n * sizeof(float)));
  CK(cudaMemcpy(*out, src, n * sizeof(float), cudaMemcpyHostToDevice));
  return MLDB_OK;
}
const RawTensor& rt(mldb_handle* h, const std::string& k) { return h->raw.at(k); }

// Pack a host [N, K] fp32 matrix into split fp16 planes scaled by 2^s.  Kpad > K zero-pads the rows
// (odd K such as the 263 motion features: the tensor-core GEMM wants K % 64 == 0).
// The scale comes from the finite elements only, so an inf or NaN element poisons its own output column (as in
// torch) and not the precision of every other one; an all-zero or all non-finite W packs at s = 0.
int pack_linear(mldb_handle* h, const float* W, int N, int K, const float* bias, LinW* out, int Kpad) {
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
int pack_named(mldb_handle* h, const std::string& wkey, const std::string& bkey, LinW* out, int row0, int nrows,
               bool pad_k) {
  const RawTensor& w = rt(h, wkey);
  const int K = (int)w.shape.back();
  const int Nall = (int)w.shape[0];
  if (nrows < 0) nrows = Nall;
  const float* b = bkey.empty() ? nullptr : rt(h, bkey).host.data() + row0;
  return pack_linear(h, w.host.data() + (size_t)row0 * K, nrows, K, b, out, pad_k ? (K + 63) / 64 * 64 : 0);
}
int pack_ln(mldb_handle* h, const std::string& p, int d, LnW* out) {
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
int upload_pe(mldb_handle* h, const std::string& key, float** out, int* rows) {
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
  // kernel setup, on this handle's device (the shared-memory opt-ins apply per device): each step records its own
  // message in mldb_last_error() when it fails
  if (!simt_init() || !mma_attention_init() || !tc_attention_init() || !gru_tc_init() ||
      !tconv_tc_init() || !smpl_tc_init()) { delete h; return MLDB_ERR_CUDA; }
  h->tc = tc_create(device);
  if (!h->tc) { delete h; return MLDB_ERR_CUDA; }
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
  } else if (!strcmp(name, "t2m_chunk")) {
    h->t2m.chunk = std::max(atoi(value), 0);
  } else if (!strcmp(name, "a2m_chunk")) {
    h->a2m.chunk = std::max(atoi(value), 0);
  } else if (!strcmp(name, "stgcn_chunk")) {
    h->stgcn.chunk = std::max(atoi(value), 0);
  } else if (!strcmp(name, "smpl_chunk")) {
    h->smpl.chunk = std::max(atoi(value), 0);
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
  if (!h || !key || !data || (!shape && ndim != 0)) FAIL(MLDB_ERR_INVALID, "null argument");
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
  if (h->a2m.on) TRY(pack_a2m(h));
  if (h->stgcn.on) TRY(pack_stgcn(h));
  if (h->smpl.on) TRY(pack_smpl(h));
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
int time_tokens(mldb_handle* h, const int64_t* d_ts, int64_t t_scalar, int n, const float* pe_row, float* out,
                float* scratch_feats, float* scratch_h, cudaStream_t st) {
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
Plan* find_plan(mldb_handle* h, PlanKind kind, int B, int S, int T) {
  char key[64];
  snprintf(key, sizeof key, "%d:%d:%d:%d", kind, B, S, T);
  auto it = h->plans.find(key);
  return it == h->plans.end() ? nullptr : it->second;
}
Plan* add_plan(mldb_handle* h, PlanKind kind, int B, int S, int T) {
  char key[64];
  snprintf(key, sizeof key, "%d:%d:%d:%d", kind, B, S, T);
  Plan* p = new Plan();
  p->kind = kind; p->B = B; p->S = S; p->T = T;
  h->plans[key] = p;
  return p;
}

// an operator could not be enqueued (its tensor maps could not be encoded): the output is unwritten,
// so the call must not report success (mldb_last_error() holds the encoder's message)
int check_ops(mldb_handle* h) {
  if (!h->op_failed) return MLDB_OK;
  h->op_failed = false;
  return MLDB_ERR_CUDA;
}

int run_graphed(mldb_handle* h, Plan* p, cudaStream_t st, const std::function<void(cudaStream_t)>& record) {
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

int check_ready(mldb_handle* h, bool need_sched) {
  if (!h) FAIL(MLDB_ERR_INVALID, "null handle");
  if (!h->finalized) FAIL(MLDB_ERR_STATE, "weights not finalized");
  if (need_sched && h->timesteps.empty()) FAIL(MLDB_ERR_STATE, "call mldb_scheduler_set_timesteps first");
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
