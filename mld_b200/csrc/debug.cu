// Profiling and debug hooks: one operator or one step timed in isolation, single operators on caller data (kernel unit
// tests), the kernels' debug timeline.
#include "engine.h"

#include <string.h>

#include <algorithm>

#include "gemm_tc.h"
#include "misc_kernels.cuh"

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
  TRY(enc_plan(h, PLAN_REVERSE, B, cfg_on ? 2 * B : B, S_ctx, &p));
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
  TRY(ops_done(h));
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
  TRY(enc_plan(h, PLAN_REVERSE, B, cfg_on ? 2 * B : B, S_ctx, &p));
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
  return ops_done(h);
}

// ----------------------------------------------------------------------------- debug aid
// The exit of a debug hook: waits for its work on st, then frees its temporaries (every allocation since n_alloc0).
static int debug_exit(mldb_handle* h, size_t n_alloc0, cudaStream_t st, const char* what) {
  cudaError_t e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = cudaGetLastError();
  while (h->allocs.size() > n_alloc0) { cudaFree(h->allocs.back()); h->allocs.pop_back(); }
  if (e != cudaSuccess) FAIL(MLDB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return check_ops(h);
}

// fp32 [rows, cols] (device) -> freshly allocated split16 planes, and back: the debug hooks' split16 outputs start
// from the caller's buffer, so the cells an op must not write can be checked after it
static int debug_to_split(mldb_handle* h, const float* src, int rows, int cols, ActBuf* out, cudaStream_t st) {
  TRY(alloc_act(h, rows, cols, out));
  k_rows_to_split<<<nblk((int64_t)rows * cols), 256, 0, st>>>(*out, src, cols, rows, cols, 1 << 30, 0, 0, 0, nullptr);
  return MLDB_OK;
}
static void debug_from_split(ActBuf x, float* out, cudaStream_t st) {
  k_split_to_f32<<<nblk((int64_t)x.rows * x.cols), 256, 0, st>>>(x, out, (int64_t)x.rows * x.cols);
}

// The largest output row the (in_group, out_group, out_off) map of rows [0, M) addresses, or -1 for a bad map.
static int64_t map_max_row(int M, int in_group, int out_group, int out_off) {
  if (M <= 0 || in_group <= 0 || out_group < 0 || out_off < 0) return -1;
  const int64_t last_seq = (M - 1) / in_group;
  // the last sequence ends at row M - 1; every earlier one is complete
  int64_t mx = last_seq * out_group + out_off + (M - 1 - last_seq * in_group);
  if (last_seq > 0) mx = std::max(mx, (last_seq - 1) * out_group + out_off + in_group - 1);
  return mx;
}

// y = act(A W^T + b) or LayerNorm(A W^T + b + R) through the engine's GEMM operators, with the GEMM's row map and
// output placement (include/mldb.h), so tests can compare the wgmma kernels with the CUDA-core kernels (and with
// torch) shape by shape.
extern "C" int mldb_debug_gemm_rows(mldb_handle* h, const mldb_gemm_rows_args* a, void* stream) {
  if (!h || !a || !a->A || !a->W || !a->out || a->M <= 0 || a->N <= 0 || a->K <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  const int M = a->M, N = a->N, K = a->K;
  const int64_t max_row = map_max_row(M, a->in_group, a->out_group, a->out_off);
  if (max_row < 0 || max_row >= a->out_rows) FAIL(MLDB_ERR_INVALID, "the row map leaves the %d output rows", a->out_rows);
  if (a->out_col0 < 0 || (int64_t)a->out_col0 + N > a->out_cols) FAIL(MLDB_ERR_INVALID, "columns outside the output");
  const int tab_need = a->out_off + std::min(a->in_group, M);
  if (a->addtab && a->tab_rows < tab_need) FAIL(MLDB_ERR_INVALID, "addtab needs %d rows", tab_need);
  if (a->a_kind < A_SPLIT || a->a_kind > A_F32_RELU) FAIL(MLDB_ERR_INVALID, "a_kind %d", a->a_kind);
  if (a->a_kind != A_SPLIT && a->use_tc) FAIL(MLDB_ERR_UNSUPPORTED, "an fp32 A runs on the CUDA-core kernel only");
  const bool identity = a->in_group >= M && a->out_group == 0 && a->out_off == 0 && !a->addtab && !a->zero_lengths;
  if (a->gamma && (!a->beta || !identity || a->out_rows != M || a->out_cols != N || a->out_col0 != 0 ||
                   a->a_kind != A_SPLIT))
    FAIL(MLDB_ERR_INVALID, "the LayerNorm epilogue takes a split16 A, the identity map and an [M, N] output");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_alloc0 = h->allocs.size();
  LinW w;
  TRY(pack_linear(h, a->W, N, K, a->bias, &w));
  const int K1 = (a->K1 <= 0 || a->K1 >= K) ? K : a->K1;
  GemmArgs ga; ga.M = M; ga.w = w; ga.act = a->act; ga.wide_n = 1; ga.vec_f32 = a->vec_f32;
  ga.in_group = a->in_group; ga.out_group = a->out_group; ga.out_off = a->out_off;
  ga.a_kind = a->a_kind;
  if (a->a_kind == A_SPLIT) {
    ActBuf a1, a2{};
    TRY(alloc_act(h, M, K1, &a1));
    k_rows_to_split<<<nblk((int64_t)M * K1), 256, 0, st>>>(a1, a->A, K, M, K1, 1 << 30, 0, 0, 0, nullptr);
    if (K1 < K) {
      TRY(alloc_act(h, M, K - K1, &a2));
      k_rows_to_split<<<nblk((int64_t)M * (K - K1)), 256, 0, st>>>(a2, a->A + K1, K, M, K - K1, 1 << 30, 0, 0, 0, nullptr);
    }
    ga.a1 = a1; ga.K1 = K1; ga.a2 = a2; ga.K2 = K - K1;
  } else {
    ga.a_f32 = a->A; ga.lda = K; ga.K1 = K;
  }
  float* tab = nullptr;
  int32_t* zl = nullptr;
  if (a->addtab) TRY(upload_f32(h, a->addtab, (size_t)a->tab_rows * N, &tab));
  if (a->zero_lengths) {
    const int nseq = (int)((M - 1) / a->in_group + 1);
    TRY(dev_alloc(h, (void**)&zl, (size_t)nseq * sizeof(int32_t)));
    CK(cudaMemcpyAsync(zl, a->zero_lengths, (size_t)nseq * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  ga.addtab = tab; ga.zero_lengths = zl;
  ActBuf o{}, res{};
  float *g = nullptr, *b = nullptr, *cf32 = nullptr;
  if (a->gamma) {
    TRY(upload_f32(h, a->gamma, N, &g));
    TRY(upload_f32(h, a->beta, N, &b));
    TRY(dev_alloc(h, (void**)&cf32, (size_t)M * N * sizeof(float)));
    TRY(debug_to_split(h, a->out, M, N, &o, st));
    if (a->R) TRY(debug_to_split(h, a->R, M, N, &res, st));
  } else if (a->split_out && !a->R) {              // the production epilogue: split16 planes
    TRY(debug_to_split(h, a->out, a->out_rows, a->out_cols, &o, st));
  }
  const bool saved = h->use_tc;
  h->use_tc = a->use_tc != 0;
  if (a->gamma) {
    LnArgs l; l.res = res; l.gamma = g; l.beta = b; l.M = M; l.d = N; l.out = o;
    op_gemm_ln(h, ga, l, cf32, st);
  } else if (o.hi) {
    ga.out = o; ga.out_col0 = a->out_col0;
    op_gemm(h, ga, st);
  } else {                                         // fp32 out (+ residual: in place when R == out)
    ga.out_f32 = a->out + a->out_col0; ga.ldc = a->out_cols;
    if (a->R) ga.res_f32 = a->R + a->out_col0;
    op_gemm(h, ga, st);
  }
  if (o.hi) debug_from_split(o, a->out, st);
  h->use_tc = saved;
  return debug_exit(h, n_alloc0, st, "debug gemm");
}

extern "C" int mldb_debug_gemm(mldb_handle* h, const float* A, const float* W, const float* bias,
                               const float* gamma, const float* beta, const float* R, int32_t M, int32_t N,
                               int32_t K, int32_t K1, int32_t act, int32_t use_tc, int32_t split_out, float* out,
                               void* stream) {
  mldb_gemm_rows_args a{};
  a.A = A; a.W = W; a.bias = bias; a.gamma = gamma; a.beta = beta; a.R = R;
  a.M = M; a.N = N; a.K = K; a.K1 = K1; a.act = act; a.use_tc = use_tc; a.a_kind = A_SPLIT;
  a.in_group = 1 << 30; a.out_group = 0; a.out_off = 0;
  a.split_out = split_out && N % 8 == 0;
  a.out = out; a.out_rows = M; a.out_cols = N; a.out_col0 = 0;
  return mldb_debug_gemm_rows(h, &a, stream);
}

extern "C" int mldb_debug_ln(mldb_handle* h, const mldb_ln_args* a, void* stream) {
  if (!h || !a || !a->gamma || !a->beta || !a->out || a->M <= 0 || a->M_in <= 0 || a->d <= 0 ||
      a->ld_out < a->d || (a->c && a->ldc < a->d) || (a->rowvec && a->rv_group <= 0))
    FAIL(MLDB_ERR_INVALID, "bad argument");
  if (a->d > LN_MAX_D) FAIL(MLDB_ERR_UNSUPPORTED, "LayerNorm rows of %d columns: the CUDA-core kernels take up to %d", a->d, LN_MAX_D);
  if (a->in_group != 0 && (a->in_group < 0 || a->sel_group <= 0)) FAIL(MLDB_ERR_INVALID, "bad row gather");
  // the input row of r: r, or (r / sel_group) * in_group + r % sel_group; the largest is one of the last two
  // sequences' last rows
  auto in_row = [&](int64_t r) { return a->in_group == 0 ? r : (r / a->sel_group) * a->in_group + r % a->sel_group; };
  int64_t mx = in_row(a->M - 1);
  if (a->in_group != 0 && a->M > a->sel_group) mx = std::max(mx, in_row(((a->M - 1) / a->sel_group) * a->sel_group - 1));
  if (mx >= a->M_in) FAIL(MLDB_ERR_INVALID, "the row gather reads past the %d input rows", a->M_in);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_alloc0 = h->allocs.size();
  LnArgs l; l.c = a->c; l.ldc = a->ldc; l.M = a->M; l.d = a->d; l.act = a->act;
  if (a->in_group != 0) { l.sel_group = a->sel_group; l.in_group = a->in_group; }
  float *g = nullptr, *b = nullptr, *rv = nullptr;
  TRY(upload_f32(h, a->gamma, a->d, &g));
  TRY(upload_f32(h, a->beta, a->d, &b));
  l.gamma = g; l.beta = b;
  if (a->rowvec) {
    TRY(upload_f32(h, a->rowvec, (size_t)((a->M_in + a->rv_group - 1) / a->rv_group) * a->d, &rv));
    l.rowvec = rv; l.rv_group = a->rv_group;
  }
  if (a->res) TRY(debug_to_split(h, a->res, a->M_in, a->d, &l.res, st));
  if (a->split_out) TRY(debug_to_split(h, a->out, a->M, a->ld_out, &l.out, st));
  else { l.out_f32 = a->out; l.ld_out = a->ld_out; }
  op_ln(h, l, st);
  if (l.out.hi) debug_from_split(l.out, a->out, st);
  return debug_exit(h, n_alloc0, st, "debug ln");
}

extern "C" int mldb_debug_rows_to_split(mldb_handle* h, const float* src, int32_t ld_src, int32_t M, int32_t d,
                                        int32_t in_group, int32_t out_group, int32_t out_off, int32_t src_bcast,
                                        const float* tab, int32_t tab_rows, int32_t relu, int32_t scalar, float* out,
                                        int32_t out_rows, int32_t out_cols, void* stream) {
  if (!h || !out || M <= 0 || d <= 0 || d > out_cols || (src && ld_src < d)) FAIL(MLDB_ERR_INVALID, "bad argument");
  const int64_t max_row = map_max_row(M, in_group, out_group, out_off);
  if (max_row < 0 || max_row >= out_rows) FAIL(MLDB_ERR_INVALID, "the row map leaves the %d output rows", out_rows);
  const int tab_need = out_off + std::min(in_group, M);
  if (tab && tab_rows < tab_need) FAIL(MLDB_ERR_INVALID, "tab needs %d rows", tab_need);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_alloc0 = h->allocs.size();
  float* tb = nullptr;
  if (tab) TRY(upload_f32(h, tab, (size_t)tab_rows * d, &tb));
  ActBuf x;
  TRY(debug_to_split(h, out, out_rows, out_cols, &x, st));
  if (scalar)
    k_rows_to_split<<<nblk((int64_t)M * d), 256, 0, st>>>(x, src, ld_src, M, d, in_group, out_group, out_off, src_bcast,
                                                          tb, relu);
  else
    rows_to_split(h, x, src, ld_src, M, d, in_group, out_group, out_off, src_bcast, tb, relu, st);
  debug_from_split(x, out, st);
  return debug_exit(h, n_alloc0, st, "debug rows_to_split");
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
  return debug_exit(h, n_alloc0, st, "debug ffn");
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
  return debug_exit(h, n_alloc0, st, "debug tail");
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
  else if (mode == 2 && tc_attention_supported(a)) { if (!tc_attention(a, h->sm_count, st)) rc = MLDB_ERR_CUDA; }
  else rc = MLDB_ERR_UNSUPPORTED;
  if (rc == MLDB_OK) k_split_to_f32<<<nblk((int64_t)Mq * d), 256, 0, st>>>(o, out, (int64_t)Mq * d);
  TRY(debug_exit(h, n_alloc0, st, "debug attention"));
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
