// CUDA-core (fp32 FFMA) implementations of the path's operators.  These are the on-device
// reference for the wgmma kernels (engine option gemm=simt) and serve the GEMMs whose
// shapes do not fit a tensor-core tile (odd K such as 263/150 motion features, tiny M).
#include "ops.cuh"

#include <stdlib.h>

// ------------------------------------------------------------------------------------ GEMM
namespace {

constexpr int SG_BM = 64, SG_BN = 64, SG_BK = 16;

__device__ __forceinline__ float load_a(const GemmArgs& a, int m, int k) {
  if (a.a_kind == A_SPLIT) {
    if (k < a.K1) {
      int64_t o = (int64_t)m * a.a1.cols + k;
      return join_f32(a.a1.hi[o], a.a1.lo()[o]);
    }
    int64_t o = (int64_t)m * a.a2.cols + (k - a.K1);
    return join_f32(a.a2.hi[o], a.a2.lo()[o]);
  }
  if (k >= a.lda) return 0.0f;               // weights packed with a zero-padded K (odd feature counts)
  float v = a.a_f32[(int64_t)m * a.lda + k];
  return a.a_kind == A_F32_RELU ? fmaxf(v, 0.0f) : v;
}

__global__ void __launch_bounds__(256) k_gemm_simt(const GemmArgs a) {
  __shared__ float As[SG_BK][SG_BM + 4];
  __shared__ float Ws[SG_BK][SG_BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * SG_BM, n0 = blockIdx.x * SG_BN;
  const int K = a.w.K, N = a.w.N, M = a.M;
  const __half* whi = a.w.w;
  const __half* wlo = a.w.w + a.w.plane_stride;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

  const int lr = tid >> 2, lk = (tid & 3) * 4;
  for (int k0 = 0; k0 < K; k0 += SG_BK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = k0 + lk + i;
      const int m = m0 + lr, n = n0 + lr;
      As[lk + i][lr] = (m < M && k < K) ? load_a(a, m, k) : 0.0f;
      float wv = 0.0f;
      if (n < N && k < K) {
        int64_t o = (int64_t)n * K + k;
        wv = join_f32(whi[o], wlo[o]);
      }
      Ws[lk + i][lr] = wv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SG_BK; ++kk) {
      float af[4], bf[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) af[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bf[j] = Ws[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(af[i], bf[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const int seq = m / a.in_group, pos = m - seq * a.in_group;
    const int64_t orow = (int64_t)seq * a.out_group + a.out_off + pos;
    const bool zero = a.zero_lengths != nullptr && pos >= a.zero_lengths[seq];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j] * a.w.inv_scale;
      if (a.w.bias) v += a.w.bias[n];
      if (a.addtab) v += a.addtab[(int64_t)(a.out_off + pos) * N + n];
      v = apply_act(v, a.act);
      if (zero) v = 0.0f;
      if (a.res_f32) v += a.res_f32[orow * a.ldc + n];   // the same thread reads and writes: may run in place
      if (a.out.hi) {
        __half h, l;
        split_f32(v, h, l);
        int64_t o = orow * a.out.cols + a.out_col0 + n;
        a.out.hi[o] = h;
        a.out.lo()[o] = l;
      }
      if (a.out_f32) a.out_f32[orow * a.ldc + n] = v;
    }
  }
}

// ------------------------------------------------------------------------------- LayerNorm
template <int VPL>
__global__ void __launch_bounds__(256) k_ln(const LnArgs a) {
  pdl_trigger();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= a.M) return;
  const int r = warp;
  const int64_t irow = (a.in_group == 0) ? (int64_t)r
                                         : (int64_t)(r / a.sel_group) * a.in_group + r % a.sel_group;
  float v[VPL];
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int n = i * 32 + lane;
    float x = 0.0f;
    if (n < a.d) {
      if (a.c) x += a.c[irow * a.ldc + n];
      if (a.res.hi) {
        int64_t o = irow * a.res.cols + n;
        x += join_f32(a.res.hi[o], a.res.lo()[o]);
      }
      if (a.rowvec) x += a.rowvec[(int64_t)(irow / a.rv_group) * a.d + n];
    }
    v[i] = x;
    s += x;
  }
  const float inv_d = 1.0f / (float)a.d;
  const float mean = warp_sum(s) * inv_d;
  float q = 0.0f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int n = i * 32 + lane;
    float dlt = (n < a.d) ? v[i] - mean : 0.0f;
    q += dlt * dlt;
  }
  const float rstd = rsqrtf(warp_sum(q) * inv_d + 1e-5f);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int n = i * 32 + lane;
    if (n < a.d) v[i] = (v[i] - mean) * rstd * a.gamma[n] + a.beta[n];
  }
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int n = i * 32 + lane;
    if (n >= a.d) continue;
    v[i] = apply_act(v[i], a.act);
    if (a.out.hi) {
      __half h, l;
      split_f32(v[i], h, l);
      int64_t o = (int64_t)r * a.out.cols + n;
      a.out.hi[o] = h;
      a.out.lo()[o] = l;
    }
    if (a.out_f32) a.out_f32[(int64_t)r * a.ld_out + n] = v[i];
  }
}

// ------------------------------------------------------------------------------- attention
// One block per (sequence, head); each warp owns query rows q = warp, warp + nwarps, ...  Softmax over
// the valid keys only (the reference masks padded keys with -inf: cross_attention.py:264-266,
// mld_vae.py:226-232); with a.causal set, query qi sees keys 0..qi only (CLIP's causal mask).
// K and V pass through shared memory as fp32 in chunks of kc keys.  When every valid key fits one chunk
// (kc >= nk, the common case) K and V are loaded once and the scores of pass 1 are kept for pass 2.
// Otherwise the warps step through their query rows together, one row per warp at a time, and stream
// the chunks twice: pass 1 takes the row maximum, pass 2 recomputes the scores, exponentiates and
// accumulates P V.  The per-warp output row lives in shared memory between chunks.  Both ways give the
// same exact two-pass softmax, summed in the same order.
constexpr int ATT_WARPS = 8;
constexpr size_t ATT_SMEM_MAX = 227 * 1024;   // the opt-in set in simt_init

__global__ void __launch_bounds__(ATT_WARPS * 32) k_attn_simt(const AttnArgs a, const int kc) {
  extern __shared__ float sm[];
  const int s = blockIdx.x / a.heads, h = blockIdx.x % a.heads;
  const int hd = a.hd, Lk = a.Lk, Lq = a.Lq;
  int nk = Lk;
  if (a.lengths) {
    const int li = a.len_mod > 0 ? (a.seq0 + s) % a.len_mod : s;
    nk = min(Lk, a.kv_prefix + a.lengths[li]);
  }
  float* Ks = sm;                          // [kc][hd+1]
  float* Vs = Ks + (size_t)kc * (hd + 1);  // [kc][hd]
  float* Qs = Vs + (size_t)kc * hd;        // [ATT_WARPS][hd]
  float* Ps = Qs + ATT_WARPS * hd;         // [ATT_WARPS][kc]
  float* Os = Ps + ATT_WARPS * kc;         // [ATT_WARPS][hd], only when kc < Lk
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const __half* khi = a.kv.hi;
  const __half* klo = a.kv.lo();
  auto load = [&](int c0, int c1, bool with_v) {   // keys [c0, c1) -> chunk rows [0, c1 - c0)
    for (int i = tid; i < (c1 - c0) * hd; i += blockDim.x) {
      const int t = i / hd, d = i - t * hd;
      const int64_t row = (int64_t)s * Lk + c0 + t;
      int64_t ok = row * a.kv.cols + a.k_col0 + h * hd + d;
      Ks[t * (hd + 1) + d] = join_f32(khi[ok], klo[ok]);
      if (with_v) {
        int64_t ov = row * a.kv.cols + a.v_col0 + h * hd + d;
        Vs[t * hd + d] = join_f32(khi[ov], klo[ov]);
      }
    }
  };
  const bool resident = nk <= kc;
  if (resident) {
    load(0, nk, true);
    __syncthreads();
  }
  const float scale = rsqrtf((float)hd);
  float* qv = Qs + warp * hd;
  float* pv = Ps + warp * kc;
  float* ov = Os + warp * hd;
  // block-uniform trip counts: every warp reaches every __syncthreads of the streamed chunks
  for (int q0 = 0; q0 < Lq; q0 += ATT_WARPS) {
    const int qi = q0 + warp;
    const bool active = qi < Lq;
    const int64_t qrow = (int64_t)s * Lq + qi;
    if (active) {
      for (int d = lane; d < hd; d += 32) {
        int64_t o = qrow * a.q.cols + a.q_col0 + h * hd + d;
        qv[d] = join_f32(a.q.hi[o], a.q.lo()[o]) * scale;
      }
    }
    __syncwarp();
    const int nkq = !active ? 0 : (a.causal ? min(nk, qi + 1) : nk);   // causal: keys j <= qi
    // keys any warp of the block needs; at least one chunk, so a row without valid keys is still written (NaN)
    const int nkb = max(1, a.causal ? min(nk, min(q0 + ATT_WARPS, Lq)) : nk);
    auto score = [&](int t, int c0) {
      const float* kr = Ks + (t - c0) * (hd + 1);
      float acc = 0.0f;
#pragma unroll 8
      for (int d = 0; d < hd; ++d) acc = fmaf(qv[d], kr[d], acc);
      return acc;
    };
    float mx = -INFINITY;
    for (int c0 = 0; c0 < nkb; c0 += kc) {
      const int c1 = min(c0 + kc, nkb);
      if (!resident) {
        __syncthreads();
        load(c0, c1, false);
        __syncthreads();
      }
      for (int t = c0 + lane; t < min(c1, nkq); t += 32) {
        const float acc = score(t, c0);
        if (resident) pv[t] = acc;
        mx = fmaxf(mx, acc);
      }
    }
    mx = warp_max(mx);
    float sum = 0.0f;
    for (int c0 = 0; c0 < nkb; c0 += kc) {
      const int c1 = min(c0 + kc, nkb), ce = min(c1, nkq);
      if (!resident) {
        __syncthreads();
        load(c0, c1, true);
        __syncthreads();
      }
      for (int t = c0 + lane; t < ce; t += 32) {
        float e = expf((resident ? pv[t - c0] : score(t, c0)) - mx);
        pv[t - c0] = e;
        sum += e;
      }
      const bool last = c1 == nkb;
      const float inv = last ? 1.0f / warp_sum(sum) : 0.0f;
      __syncwarp();
      if (active) {
        for (int d = lane; d < hd; d += 32) {
          float acc = c0 == 0 ? 0.0f : ov[d];
          for (int t = c0; t < ce; ++t) acc = fmaf(pv[t - c0], Vs[(t - c0) * hd + d], acc);
          if (!last) {
            ov[d] = acc;
            continue;
          }
          acc *= inv;
          __half hh, ll;
          split_f32(acc, hh, ll);
          int64_t o = qrow * a.out.cols + h * hd + d;
          a.out.hi[o] = hh;
          a.out.lo()[o] = ll;
        }
      }
      __syncwarp();
    }
  }
}

// 128-bit version for d = NIT * 256 (the shapes the path uses): a lane owns 8 consecutive columns per 256-column
// group - 16-byte loads of the split16 residual planes, 2 x 16-byte loads of the fp32 inputs, 16-byte stores
template <int NIT>
__global__ void __launch_bounds__(256) k_ln_vec(const LnArgs a) {
  pdl_trigger();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= a.M) return;
  const int r = warp;
  const int64_t irow = (a.in_group == 0) ? (int64_t)r
                                         : (int64_t)(r / a.sel_group) * a.in_group + r % a.sel_group;
  float v[NIT][8];
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < NIT; ++i) {
    const int n = i * 256 + lane * 8;
#pragma unroll
    for (int k = 0; k < 8; ++k) v[i][k] = 0.0f;
    if (a.c) {
      const float4 c0 = *reinterpret_cast<const float4*>(a.c + irow * a.ldc + n), c1 = *reinterpret_cast<const float4*>(a.c + irow * a.ldc + n + 4);
      v[i][0] = c0.x; v[i][1] = c0.y; v[i][2] = c0.z; v[i][3] = c0.w; v[i][4] = c1.x; v[i][5] = c1.y; v[i][6] = c1.z; v[i][7] = c1.w;
    }
    if (a.res.hi) {
      const int64_t o = irow * a.res.cols + n;
      const uint4 h = *reinterpret_cast<const uint4*>(a.res.hi + o), l = *reinterpret_cast<const uint4*>(a.res.lo() + o);
      const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[k]));
        const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[k]));
        v[i][2 * k] += hf.x + lf.x;
        v[i][2 * k + 1] += hf.y + lf.y;
      }
    }
    if (a.rowvec) {
      const float* rv = a.rowvec + (int64_t)(irow / a.rv_group) * a.d + n;
      const float4 r0 = *reinterpret_cast<const float4*>(rv), r1 = *reinterpret_cast<const float4*>(rv + 4);
      v[i][0] += r0.x; v[i][1] += r0.y; v[i][2] += r0.z; v[i][3] += r0.w; v[i][4] += r1.x; v[i][5] += r1.y; v[i][6] += r1.z; v[i][7] += r1.w;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) s += v[i][k];
  }
  const float inv_d = 1.0f / (float)a.d;
  auto normalise = [&](const float* gamma, const float* beta) {
    float sum = 0.0f;
#pragma unroll
    for (int i = 0; i < NIT; ++i)
#pragma unroll
      for (int k = 0; k < 8; ++k) sum += v[i][k];
    const float mean = warp_sum(sum) * inv_d;
    float q = 0.0f;
#pragma unroll
    for (int i = 0; i < NIT; ++i)
#pragma unroll
      for (int k = 0; k < 8; ++k) { const float dlt = v[i][k] - mean; q += dlt * dlt; }
    const float rstd = rsqrtf(warp_sum(q) * inv_d + 1e-5f);
#pragma unroll
    for (int i = 0; i < NIT; ++i) {
      const int n = i * 256 + lane * 8;
      const float4 g0 = *reinterpret_cast<const float4*>(gamma + n), g1 = *reinterpret_cast<const float4*>(gamma + n + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(beta + n), b1 = *reinterpret_cast<const float4*>(beta + n + 4);
      const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int k = 0; k < 8; ++k) v[i][k] = (v[i][k] - mean) * rstd * g[k] + b[k];
    }
  };
  (void)s;
  normalise(a.gamma, a.beta);
  if (a.act != ACT_NONE)
#pragma unroll
    for (int i = 0; i < NIT; ++i)
#pragma unroll
      for (int k = 0; k < 8; ++k) v[i][k] = apply_act(v[i][k], a.act);
#pragma unroll
  for (int i = 0; i < NIT; ++i) {
    const int n = i * 256 + lane * 8;
    if (a.out.hi) {
      uint32_t ph[4], pl[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        __half h0, l0, h1, l1;
        split_f32(v[i][2 * k], h0, l0);
        split_f32(v[i][2 * k + 1], h1, l1);
        const __half2 hh = __halves2half2(h0, h1), ll = __halves2half2(l0, l1);
        ph[k] = *reinterpret_cast<const uint32_t*>(&hh);
        pl[k] = *reinterpret_cast<const uint32_t*>(&ll);
      }
      const int64_t o = (int64_t)r * a.out.cols + n;
      *reinterpret_cast<uint4*>(a.out.hi + o) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
      *reinterpret_cast<uint4*>(a.out.lo() + o) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
    }
    if (a.out_f32) {
      float* dst = a.out_f32 + (int64_t)r * a.ld_out + n;
      *reinterpret_cast<float4*>(dst) = make_float4(v[i][0], v[i][1], v[i][2], v[i][3]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(v[i][4], v[i][5], v[i][6], v[i][7]);
    }
  }
}

}  // namespace

void simt_gemm(const GemmArgs& a, cudaStream_t st) {
  dim3 grid((a.w.N + SG_BN - 1) / SG_BN, (a.M + SG_BM - 1) / SG_BM);
  k_gemm_simt<<<grid, 256, 0, st>>>(a);
}

// d <= LN_MAX_D (k_ln<32> covers 32 x 32 columns; the callers keep d within it)
void simt_ln(const LnArgs& a, cudaStream_t st) {
  const int rows_per_block = 8;
  dim3 grid((a.M + rows_per_block - 1) / rows_per_block);
  // the 128-bit version needs 16-byte aligned rows everywhere it touches
  const bool vec_ok = (a.d == 256 || a.d == 512) && (!a.c || (a.ldc % 4 == 0 && ((uintptr_t)a.c & 15) == 0)) &&
                      (!a.res.hi || (a.res.cols % 8 == 0 && ((uintptr_t)a.res.hi & 15) == 0 && (a.res.plane_stride % 8) == 0)) &&
                      (!a.out.hi || (a.out.cols % 8 == 0 && ((uintptr_t)a.out.hi & 15) == 0 && (a.out.plane_stride % 8) == 0)) &&
                      (!a.out_f32 || (a.ld_out % 4 == 0 && ((uintptr_t)a.out_f32 & 15) == 0)) &&
                      (!a.rowvec || ((uintptr_t)a.rowvec & 15) == 0) && ((uintptr_t)a.gamma & 15) == 0 &&
                      ((uintptr_t)a.beta & 15) == 0;
  if (vec_ok && a.d == 256) launch_pdl(k_ln_vec<1>, grid, dim3(256), 0, st, a);
  else if (vec_ok) launch_pdl(k_ln_vec<2>, grid, dim3(256), 0, st, a);
  else if (a.d <= 256) launch_pdl(k_ln<8>, grid, dim3(256), 0, st, a);
  else if (a.d <= 512) launch_pdl(k_ln<16>, grid, dim3(256), 0, st, a);
  else launch_pdl(k_ln<32>, grid, dim3(256), 0, st, a);
}

// shared memory of k_attn_simt for kc keys per chunk (the output rows only when the keys do not fit one chunk)
static size_t attn_smem(int hd, int Lk, int kc) {
  size_t f = (size_t)kc * (2 * hd + 1) + (size_t)ATT_WARPS * (hd + kc);
  if (kc < Lk) f += (size_t)ATT_WARPS * hd;
  return f * sizeof(float);
}

// Keys per chunk: all Lk when they fit (K and V loaded once), else the most that fit, in whole warps of keys.
// 0: not even one key fits beside the query and output rows (head_dim above ~3200).
static int attn_chunk(int hd, int Lk) {
  if (attn_smem(hd, Lk, Lk) <= ATT_SMEM_MAX) return Lk;
  const size_t fixed = attn_smem(hd, Lk, 0), per_key = (size_t)(2 * hd + 1 + ATT_WARPS) * sizeof(float);
  if (fixed + per_key > ATT_SMEM_MAX) return 0;
  const int kc = (int)((ATT_SMEM_MAX - fixed) / per_key);
  return kc >= 32 ? kc & ~31 : kc;
}

bool simt_attention_supported(int hd) { return hd >= 1 && attn_chunk(hd, 1 << 30) > 0; }

int g_mldb_pdl = 1;

bool simt_init() {
  if (const char* e = getenv("MLDB_PDL")) g_mldb_pdl = atoi(e) != 0;
  return smem_opt_in(k_attn_simt, (int)ATT_SMEM_MAX, "k_attn_simt");
}

bool simt_attention(const AttnArgs& a, cudaStream_t st) {
  const int kc = attn_chunk(a.hd, a.Lk);
  const size_t smem = kc > 0 ? attn_smem(a.hd, a.Lk, kc) : 0;
  if (kc <= 0 || smem > ATT_SMEM_MAX) return false;       // never launch above the opt-in
  k_attn_simt<<<a.nseq * a.heads, ATT_WARPS * 32, smem, st>>>(a, kc);
  return true;
}
