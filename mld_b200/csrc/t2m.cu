// The T2M evaluator (the text, movement and motion encoders behind R-precision and FID).
#include "engine.h"

#include <string.h>

#include <algorithm>

#include "misc_kernels.cuh"

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
  TRY(may_configure(h, cfg->abi_version, MLDB_T2M_ABI_VERSION, h->t2m.on, "t2m", "the T2M evaluator"));
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

int pack_t2m(mldb_handle* h) {
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

// ----------------------------------------------------------------------------- T2M evaluator: forward
// The workspace buffers (T2mW) are shared between encoders and grow to the largest use; every kernel that writes one
// writes all of the region it later reads.

static size_t gru_bytes_per_seq(int L, int in, int H) {
  return (size_t)L * (4 * in + 24 * H) + (size_t)40 * H;   // x (split16), gi (fp32), state and head
}
static int t2m_ready(mldb_handle* h, int part, const char* what) {
  return check_configured(h, h->t2m.on && (h->t2m.cfg.parts & part), "t2m", what);
}

// Bidirectional GRU over x [n * L, in] (split16, row b * L + t) and the BiGRUCo head -> out [n, out_dim] fp32.
static int gru_forward(mldb_handle* h, const GruW& g, ActBuf x, const int32_t* lengths, int n, int L, float* out,
                       int out_dim, cudaStream_t st) {
  T2mW& t = h->t2m;
  const int H = g.H, rows_pad = (n + 127) / 128 * 128;
  ActBuf fin;
  // h0_ld = 0: the learned `hidden` is the initial state of every row
  TRY(op_gru(h, x, g.w_ih, g.w_hh, g.b_hh, g.h0, 0, lengths, n, L, H, 2, t.f32, t.gru, ActBuf{}, &fin, nullptr, st));
  // head: cat(h_fwd final, h_bwd final) -> Linear -> LayerNorm -> LeakyReLU -> Linear
  TRY(grow(t.head_f32, (size_t)n * H * sizeof(float)));
  float* cf = (float*)t.head_f32.p;
  ActBuf ln_out;
  TRY(grow_act(t.head_ln, n, H, &ln_out));
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
  TRY(t2m_ready(h, MLDB_T2M_MOVEMENT, "the T2M movement encoder"));
  const mldb_t2m_config& c = h->t2m.cfg;
  if (B < 1 || T < 4) FAIL(MLDB_ERR_INVALID, "movement encoder input must be [B >= 1, T >= 4, %d], got B=%d T=%d", c.dim_pose, B, T);
  if (ld < c.dim_pose) FAIL(MLDB_ERR_INVALID, "row stride ld=%d is smaller than dim_pose=%d", ld, c.dim_pose);
  if ((int64_t)B * T * ld > ((int64_t)1 << 40)) FAIL(MLDB_ERR_INVALID, "input too large");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  T2mW& t = h->t2m;
  const int C = c.dim_pose, Cp = (C + 15) / 16 * 16, hid = c.dim_move_hidden, lat = c.dim_move_latent;
  const int T1 = T / 2, T2 = T1 / 2;
  const size_t per_seq = (size_t)T1 * (16 * Cp + 4 * hid) + (size_t)T2 * (16 * hid + 4 * lat);
  const int Bc = eval_chunk(t.chunk, B, per_seq, 128);
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0);
    ActBuf a1, a2, z;
    TRY(grow_act(t.in, n * T1, 4 * Cp, &a1));
    TRY(grow(t.f32, (size_t)n * T1 * hid * sizeof(float)));
    float* y1 = (float*)t.f32.p;
    TRY(grow_act(t.emb, n * T2, 4 * hid, &a2));
    TRY(grow_act(t.mid, n * T2, lat, &z));
    im2col_k4s2(a1, x + (int64_t)b0 * T * ld, ld, T, C, Cp, T1, n * T1, st);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs g1; g1.a1 = a1; g1.K1 = 4 * Cp; g1.M = n * T1; g1.w = t.conv1; g1.act = ACT_LEAKY; g1.out_f32 = y1;
    g1.ldc = hid; g1.wide_n = 1; g1.vec_f32 = 1;
    op_gemm(h, g1, st);                            // main.0 + LeakyReLU (dropout: identity in eval)
    im2col_k4s2(a2, y1, hid, T1, hid, hid, T2, n * T2, st);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs g2; g2.a1 = a2; g2.K1 = 4 * hid; g2.M = n * T2; g2.w = t.conv2; g2.act = ACT_LEAKY; g2.out = z;
    g2.wide_n = 1;
    op_gemm(h, g2, st);                            // main.3 + LeakyReLU
    GemmArgs g3; g3.a1 = z; g3.K1 = lat; g3.M = n * T2; g3.w = t.move_out; g3.out_f32 = out + (int64_t)b0 * T2 * lat;
    g3.ldc = lat; g3.wide_n = 1; g3.vec_f32 = 1;
    op_gemm(h, g3, st);                            // out_net
  }
  return ops_done(h);
}

extern "C" int mldb_t2m_motion(mldb_handle* h, const float* x, const int32_t* lengths, int32_t B, int32_t L, float* out,
                               void* stream) {
  if (!h || !x || !lengths || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(t2m_ready(h, MLDB_T2M_MOTION, "the T2M motion encoder"));
  const mldb_t2m_config& c = h->t2m.cfg;
  if (B < 1 || L < 1 || (int64_t)B * L > (1 << 26)) FAIL(MLDB_ERR_INVALID, "motion encoder input must be [B >= 1, L >= 1, %d], got B=%d L=%d", c.dim_move_latent, B, L);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  T2mW& t = h->t2m;
  const int In = c.dim_move_latent, H = c.dim_motion_hidden;
  const int Bc = eval_chunk(t.chunk, B, gru_bytes_per_seq(L, In + H, H), 128);
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0);
    ActBuf xs, e;
    TRY(grow_act(t.in, n * L, In, &xs));
    TRY(grow_act(t.emb, n * L, H, &e));
    k_f32_to_split_pad<<<nblk((int64_t)n * L * In), 256, 0, st>>>(xs, x + (int64_t)b0 * L * In, In, n * L, In, 1);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs g; g.a1 = xs; g.K1 = In; g.M = n * L; g.w = t.motion_in; g.out = e; g.wide_n = 1;
    op_gemm(h, g, st);                             // input_emb
    TRY(gru_forward(h, t.motion_gru, e, lengths + b0, n, L, out + (int64_t)b0 * c.dim_motion_latent,
                    c.dim_motion_latent, st));
  }
  return ops_done(h);
}

extern "C" int mldb_t2m_text(mldb_handle* h, const float* word_embs, const float* pos_ohot, const int32_t* lengths,
                             int32_t B, int32_t L, float* out, void* stream) {
  if (!h || !word_embs || !pos_ohot || !lengths || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(t2m_ready(h, MLDB_T2M_TEXT, "the T2M text encoder"));
  const mldb_t2m_config& c = h->t2m.cfg;
  if (B < 1 || L < 1 || (int64_t)B * L > (1 << 26)) FAIL(MLDB_ERR_INVALID, "text encoder input must be [B >= 1, L >= 1, *], got B=%d L=%d", B, L);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  T2mW& t = h->t2m;
  const int W = c.dim_word, P = c.dim_pos_ohot, H = c.dim_text_hidden;
  const int Bc = eval_chunk(t.chunk, B, gru_bytes_per_seq(L, pad64(P) + 2 * W + pad64(W) + H, H), 128);
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0), M = n * L;
    ActBuf ps, xs, e;
    TRY(grow_act(t.in, M, pad64(P), &ps));
    TRY(grow(t.mid, (size_t)M * W * sizeof(float)));
    float* xw = (float*)t.mid.p;
    TRY(grow_act(t.words, M, pad64(W), &xs));
    TRY(grow_act(t.emb, M, H, &e));
    k_f32_to_split_pad<<<nblk((int64_t)M * ps.cols), 256, 0, st>>>(ps, pos_ohot + (int64_t)b0 * L * P, P, M, P, 1);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs gp; gp.a1 = ps; gp.K1 = ps.cols; gp.M = M; gp.w = t.pos_emb; gp.out_f32 = xw; gp.ldc = W;
    gp.res_f32 = word_embs + (int64_t)b0 * L * W; gp.wide_n = 1;
    op_gemm(h, gp, st);                            // word_embs + pos_emb(pos_ohot)
    k_f32_to_split_pad<<<nblk((int64_t)M * xs.cols), 256, 0, st>>>(xs, xw, W, M, W, 1);
    kcount(h, MLDB_KSTAT_MISC);
    GemmArgs g; g.a1 = xs; g.K1 = xs.cols; g.M = M; g.w = t.text_in; g.out = e; g.wide_n = 1;
    op_gemm(h, g, st);                             // input_emb
    TRY(gru_forward(h, t.text_gru, e, lengths + b0, n, L, out + (int64_t)b0 * c.dim_coemb_hidden,
                    c.dim_coemb_hidden, st));
  }
  return ops_done(h);
}
