// Operator dispatch (each operator picks the tensor-core kernel when the shape allows it), the transformer-stack
// workspaces, and the encoder / decoder layers and stacks of the denoiser and the VAE.
#include "engine.h"
#include "gemm_tc.h"
#include "misc_kernels.cuh"

// ----------------------------------------------------------------------------- op dispatch
void op_gemm(mldb_handle* h, const GemmArgs& g, cudaStream_t st) {
  if (h->use_tc && tc_gemm_supported(h->tc, g)) {
    if (!tc_gemm(h->tc, g, nullptr, st)) h->op_failed = true;
    kcount(h, MLDB_KSTAT_GEMM_TC);
    return;
  }
  simt_gemm(g, st);
  kcount(h, MLDB_KSTAT_GEMM_SIMT);
}
// GEMM followed by residual + LayerNorm (one fused wgmma kernel when the tile covers a row)
void op_gemm_ln(mldb_handle* h, GemmArgs g, LnArgs l, float* cf32, cudaStream_t st) {
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
void op_ln(mldb_handle* h, const LnArgs& l, cudaStream_t st) { simt_ln(l, st); kcount(h, MLDB_KSTAT_LN_SIMT); }
void op_attn(mldb_handle* h, const AttnArgs& a, cudaStream_t st) {
  if (h->use_tc && h->attn_kind == 0 && tc_attention_supported(a)) {
    if (!tc_attention(a, h->sm_count, st)) h->op_failed = true;
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
int op_gru(mldb_handle* h, ActBuf x, const LinW* w_ih, const LinW& w_hh, const float* b_hh, const float* h0,
           int64_t h0_ld, const int32_t* lengths, int n, int L, int H, int dirs, GrowBuf& gi, GruState& ws,
           ActBuf seq_out, ActBuf* fin, const float** fin_f32, cudaStream_t st) {
  TRY(grow(gi, (size_t)n * L * dirs * 3 * H * sizeof(float)));
  float* gif = (float*)gi.p;
  for (int d = 0; d < dirs; ++d) {                 // gi = x W_ih^T + b_ih, every step of every direction
    GemmArgs g; g.a1 = x; g.K1 = x.cols; g.M = n * L; g.w = w_ih[d]; g.out_f32 = gif + (size_t)d * 3 * H;
    g.ldc = dirs * 3 * H; g.wide_n = 1; g.vec_f32 = 1;
    op_gemm(h, g, st);
  }
  if (h->use_tc && dirs == 1) {
    GruSeqArgs s;
    s.gi = gif; s.b_hh = b_hh; s.h0 = h0; s.lengths = lengths; s.w_hh = w_hh.w; s.w_plane_stride = w_hh.plane_stride;
    s.w_inv_scale = w_hh.inv_scale; s.rows = n; s.L = L; s.H = H; s.seq_out = seq_out;
    if (fin_f32) {
      TRY(grow(ws.h_f32, (size_t)n * H * sizeof(float)));
      *fin_f32 = s.h_last = (float*)ws.h_f32.p;
    }
    // mldb_a2m_configure refuses other H: k_gru_step_tc, the kernel for larger H, runs two directions only
    if (!gru_seq_supported(H) || !gru_seq_tc(s, h->sm_count, st)) h->op_failed = true;
    kcount(h, MLDB_KSTAT_GRU_TC);
    return MLDB_OK;
  }
  const int rows_pad = (n + 127) / 128 * 128;
  const size_t plane = (size_t)dirs * rows_pad * H, state_bytes = split16_bytes(dirs * rows_pad, H);
  TRY(grow(ws.h_split, 2 * state_bytes));
  TRY(grow(ws.h_f32, 2 * plane * sizeof(float)));
  if (!h->use_tc) TRY(grow(ws.gh, plane * 3 * sizeof(float)));
  float *hf = (float*)ws.h_f32.p, *gh = (float*)ws.gh.p;
  auto state = [&](int b) { return split16_at((char*)ws.h_split.p + b * state_bytes, dirs * rows_pad, H); };
  GruStepArgs a;
  a.gi = gif; a.gh = gh; a.b_hh = b_hh; a.lengths = lengths; a.w_hh = w_hh.w; a.w_plane_stride = w_hh.plane_stride;
  a.w_inv_scale = w_hh.inv_scale; a.rows = n; a.rows_pad = rows_pad; a.L = L; a.H = H; a.dirs = dirs; a.h0_ld = h0_ld;
  a.seq_out = seq_out;
  a.h_out = state(0); a.hf_out = hf;
  gru_init_state(a, h0, st);
  kcount(h, MLDB_KSTAT_MISC);
  for (int s = 0; s < L; ++s) {
    a.step = s;
    a.h_in = state(s & 1); a.hf_in = hf + (s & 1) * plane;
    a.h_out = state((s + 1) & 1); a.hf_out = hf + ((s + 1) & 1) * plane;
    if (h->use_tc) {
      if (!gru_step_tc(a, st)) h->op_failed = true;
      kcount(h, MLDB_KSTAT_GRU_TC);
    } else {
      for (int d = 0; d < dirs; ++d) {
        LinW w = w_hh;
        w.w += (size_t)d * 3 * H * H; w.N = 3 * H;
        GemmArgs g; g.a1 = rows_of(a.h_in, (int64_t)d * rows_pad, n); g.K1 = H; g.M = n; g.w = w;
        g.out_f32 = gh + (size_t)d * rows_pad * 3 * H; g.ldc = 3 * H; g.wide_n = 1;
        op_gemm(h, g, st);
      }
      gru_gate_simt(a, st);
      kcount(h, MLDB_KSTAT_MISC);
    }
  }
  if (fin) *fin = state(L & 1);
  if (fin_f32) *fin_f32 = hf + (L & 1) * plane;
  return MLDB_OK;
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
void op_tail(mldb_handle* h, const LinW& wo, const LnW& n1, const LinW& l1, const LinW& l2, const LnW& n2, ActBuf att,
             ActBuf x, ActBuf x1, ActBuf hbuf, ActBuf xout, int M, int d, int ff, float* cf32, cudaStream_t st, int fuse) {
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
// fp32 rows -> split16 rows (+ table row, ReLU) with the (seq, pos) mapping of k_rows_to_split; the
// 128-bit path whenever the shapes allow it
void rows_to_split(mldb_handle* h, ActBuf X, const float* src, int ld_src, int M, int d, int in_group, int out_group,
                   int out_off, int src_bcast, const float* tab, int relu, cudaStream_t st) {
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

// ----------------------------------------------------------------------------- workspaces
int alloc_act(mldb_handle* h, int rows, int cols, ActBuf* out) {
  void* p = nullptr;
  TRY(dev_alloc(h, &p, split16_bytes(rows, cols)));
  CK(cudaMemset(p, 0, split16_bytes(rows, cols)));
  *out = split16_at(p, rows, cols);
  return MLDB_OK;
}
int alloc_stack_ws(mldb_handle* h, const StackW& sw, int nseq, int L, int Lmem, StackWs* ws, int n_sel) {
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

// the workspace rows of sequences [s0, s0 + n): a self-contained workspace for that sub-batch
StackWs ws_slice(const StackWs& ws, int s0, int n) {
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
void out_proj_ln(mldb_handle* h, const LinW& w, const LnW& n, ActBuf att, ActBuf res, ActBuf xout, int M, int d,
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
void ffn_block(mldb_handle* h, const LinW& l1, const LinW& l2, const LnW& n, ActBuf xin, ActBuf xout, StackWs& ws,
               int act, cudaStream_t st) {
  GemmArgs g; g.a1 = xin; g.K1 = ws.d; g.M = ws.M; g.w = l1; g.act = act; g.out = ws.h;
  GemmArgs g2; g2.a1 = ws.h; g2.K1 = ws.ff; g2.M = ws.M; g2.w = l2;
  LnArgs l; l.res = xin; l.gamma = n.g; l.beta = n.b; l.M = ws.M; l.d = ws.d; l.out = xout;
  op_ffn(h, g, g2, l, ws.cf32, st);
}
// TransformerEncoderLayer.forward_post (cross_attention.py:259-272)
void enc_layer(mldb_handle* h, const StackW& sw, const EncW& w, ActBuf xin, ActBuf xout, StackWs& ws,
               const SeqInfo& si, cudaStream_t st) {
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
ActBuf run_stack(mldb_handle* h, const StackW& sw, ActBuf x0, ActBuf mem, StackWs& ws, const SeqInfo& si,
                 cudaStream_t st) {
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
