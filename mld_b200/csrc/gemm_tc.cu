// Warpgroup-MMA (wgmma) split-fp16 kernels for sm_90a: the persistent GEMM with fused epilogues
// (k_gemm_tc) and the fused FFN block (k_ffn_tc).
//
//   D[128 x BN] (fp32, registers) = A_hi W_hi^T + A_lo W_hi^T + A_hi W_lo^T        per 128-row tile
//
// A = activations in the split16 format (two fp16 planes, row-major [M, K]); W = nn.Linear weight
// [N, K] (PyTorch's [out, in] layout is already the K-major B operand), also split into hi/lo
// planes.  Three f16 MMAs per K-step reproduce the reference's fp32 GEMM to ~1e-6.
//
// CTA = three warpgroups, one CTA per SM, persistent over tiles: warpgroup 0 gives its registers
// away (setmaxnreg) and its first warp is the TMA producer; warpgroups 1 and 2 each own 64 rows of
// the tile, issue wgmma.mma_async on operands that stream through a ring of 128B-swizzled
// shared-memory tiles (BK = 64 halves = one swizzle row) and run the epilogue on their accumulator
// registers while the producer already fills the ring for the next tile.
// Epilogues (a thread holds column pairs of two rows, a row is spread over the 4 lanes of a quad):
//   fast:      bias + activation -> split16, identity row mapping (the per-layer GEMMs)
//   generic:   + positional table, row remapping, zeroed padding rows, fp32 output, ragged N
//   LayerNorm: BN == N == 256, so a quad owns COMPLETE rows: bias + residual, exact two-pass
//              statistics over the registers with quad shuffles, normalise -> split16.
#include "gemm_tc.h"

#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <string>
#include <string.h>

#include "tc_common.cuh"

void mldb_set_err(const std::string& s);

namespace {
using namespace tc;

constexpr int BM = 128, BK = 64;
constexpr int NUM_THREADS = 384;                     // producer warpgroup + two consumer warpgroups
constexpr int CONSUMER_WARPS = 8;
constexpr int MAX_N = 1024;

// ------------------------------------------------------------------------------ parameters
struct TcParams {
  int M, N, kblocks, kb1;
  int m_tiles, n_tiles;
  float inv_scale;
  const float* bias;
  const float* addtab;
  int act;
  __half* out_hi; __half* out_lo; int ld_out, out_col0;
  float* out_f32; int ldc;
  int in_group, out_group, out_off;
  const int32_t* zero_lengths;
  // residual + LayerNorm epilogue
  const __half* res_hi; const __half* res_lo; int ld_res;
  const float* gamma; const float* beta;
  long long* tl; // debug timeline (nullptr normally)
};

enum { EPI_FAST = 0, EPI_LN = 1, EPI_GENERIC = 2 };     // epilogue variants of k_gemm_tc (see the kernel)

template <int BN>
struct TileCfg {
  static constexpr int A_BYTES = BM * BK * 2;          // one plane of the A tile (16 KB)
  static constexpr int W_BYTES = BN * BK * 2;          // one plane of the W tile
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * W_BYTES;       // 96 KB (BN = 256) / 64 KB
  static constexpr int STAGES = BN == 256 ? 2 : 3;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 + 1024;   // + barriers + alignment slack
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

template <int BN>
__device__ __forceinline__ void wgmma_ss(float (&d)[BN / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (BN == 256) wgmma_ss_n256(d, a, b, acc);
  else if constexpr (BN == 128) wgmma_ss_n128(d, a, b, acc);
  else wgmma_ss_n64(d, a, b, acc);
}
// one k-block (64 deep) of this warpgroup's [64 x BN] tile: 4 x (A_lo.W_hi + A_hi.W_lo + A_hi.W_hi)
template <int BN>
__device__ __forceinline__ void kblock_ss(float (&d)[BN / 2], uint32_t sAh, uint32_t sAl, uint32_t sWh, uint32_t sWl, bool first) {
  uint64_t ah = make_desc(sAh), al = make_desc(sAl), wh = make_desc(sWh), wl = make_desc(sWl);
#pragma unroll
  for (int kk = 0; kk < BK / 16; ++kk) {
    wgmma_ss<BN>(d, al, wh, (first && kk == 0) ? 0u : 1u);
    wgmma_ss<BN>(d, ah, wl, 1u);
    wgmma_ss<BN>(d, ah, wh, 1u);
    ah += 2; al += 2; wh += 2; wl += 2;                // next 16-wide slice: +32 B (>> 4)
  }
}

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ void store_split2(__half* hi, __half* lo, int64_t o, float x0, float x1) {
  uint32_t h, l;
  split2(x0, x1, h, l);
  *reinterpret_cast<uint32_t*>(hi + o) = h;
  *reinterpret_cast<uint32_t*>(lo + o) = l;
}

// y = LayerNorm(acc * sc + bias + residual) * gamma + beta over the 256-wide rows of a [64 x 256] accumulator
// fragment, eps 1e-5.  r_lo: this thread's first row (the second is r_lo + 8), cp: its column offset inside an
// 8-column group.  The statistics are two exact passes over the registers; a row's four lanes are merged with
// shuffles in a fixed order, so the result does not depend on which CTA ran the tile.
__device__ __forceinline__ void ln_epilogue(float (&d)[128], float sc, const float* bias, const __half* res_hi,
                                            const __half* res_lo, int ld_res, const float* gamma, const float* beta,
                                            __half* out_hi, __half* out_lo, int ld_out, int r_lo, int M, int cp) {
  const bool ok0 = r_lo < M, ok1 = r_lo + 8 < M;
  float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int n = 8 * j + cp;
    const float2 b = bias ? __ldg(reinterpret_cast<const float2*>(bias + n)) : make_float2(0.0f, 0.0f);
    float x0 = fmaf(d[4 * j], sc, b.x), x1 = fmaf(d[4 * j + 1], sc, b.y);
    float x2 = fmaf(d[4 * j + 2], sc, b.x), x3 = fmaf(d[4 * j + 3], sc, b.y);
    if (res_hi) {
      if (ok0) {
        const int64_t o = (int64_t)r_lo * ld_res + n;
        const float2 h = __half22float2(*reinterpret_cast<const __half2*>(res_hi + o));
        const float2 l = __half22float2(*reinterpret_cast<const __half2*>(res_lo + o));
        x0 = (x0 + h.x) + l.x; x1 = (x1 + h.y) + l.y;
      }
      if (ok1) {
        const int64_t o = (int64_t)(r_lo + 8) * ld_res + n;
        const float2 h = __half22float2(*reinterpret_cast<const __half2*>(res_hi + o));
        const float2 l = __half22float2(*reinterpret_cast<const __half2*>(res_lo + o));
        x2 = (x2 + h.x) + l.x; x3 = (x3 + h.y) + l.y;
      }
    }
    d[4 * j] = x0; d[4 * j + 1] = x1; d[4 * j + 2] = x2; d[4 * j + 3] = x3;
    s0 += x0 + x1; s1 += x2 + x3;
  }
  const float mean0 = quad_sum(s0) * (1.0f / 256), mean1 = quad_sum(s1) * (1.0f / 256);
  float q0 = 0.0f, q1 = 0.0f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float a0 = d[4 * j] - mean0, a1 = d[4 * j + 1] - mean0, a2 = d[4 * j + 2] - mean1, a3 = d[4 * j + 3] - mean1;
    q0 = fmaf(a0, a0, fmaf(a1, a1, q0));
    q1 = fmaf(a2, a2, fmaf(a3, a3, q1));
  }
  const float rstd0 = rsqrtf(quad_sum(q0) * (1.0f / 256) + 1e-5f), rstd1 = rsqrtf(quad_sum(q1) * (1.0f / 256) + 1e-5f);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int n = 8 * j + cp;
    const float2 g = __ldg(reinterpret_cast<const float2*>(gamma + n)), be = __ldg(reinterpret_cast<const float2*>(beta + n));
    if (ok0)
      store_split2(out_hi, out_lo, (int64_t)r_lo * ld_out + n, fmaf((d[4 * j] - mean0) * rstd0, g.x, be.x),
                   fmaf((d[4 * j + 1] - mean0) * rstd0, g.y, be.y));
    if (ok1)
      store_split2(out_hi, out_lo, (int64_t)(r_lo + 8) * ld_out + n, fmaf((d[4 * j + 2] - mean1) * rstd1, g.x, be.x),
                   fmaf((d[4 * j + 3] - mean1) * rstd1, g.y, be.y));
  }
}

// ------------------------------------------------------------------------------ the kernel
// Persistent: CTA c walks tiles c, c + #CTAs, ...; tile t -> (m = t / n_tiles, n = t % n_tiles).
// EPI selects the epilogue: EPI_FAST = plain, split16 output, identity row mapping, N a whole number of tiles
// (the per-layer GEMMs); EPI_LN = residual + LayerNorm; EPI_GENERIC = plain with everything else (positional
// table, row remapping, zeroed padding rows, fp32 output, ragged N: the per-batch embedding / final-layer
// GEMMs) kept out of the hot kernels' instruction stream.
template <int BN, int EPI, int ACT = ACT_NONE>      // ACT: the fast epilogue's activation (NONE | GELU)
__global__ void __launch_bounds__(NUM_THREADS, 1)
k_gemm_tc(const __grid_constant__ CUtensorMap tmA1h, const __grid_constant__ CUtensorMap tmA1l,
          const __grid_constant__ CUtensorMap tmA2h, const __grid_constant__ CUtensorMap tmA2l,
          const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const TcParams p) {
  static_assert(EPI != EPI_LN || BN == 256, "the LayerNorm epilogue covers a full 256-wide row");
  using Cfg = TileCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment by pointer arithmetic (an integer round trip would lose the shared address space)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);   // [STAGES] TMA tx
  uint64_t* bar_empty = bar_full + STAGES;                                              // [STAGES] one arrival per consumer warp

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // provably warp-uniform
  int tl_n = 0;                                     // debug-timeline event counter of this warp
  tl_event(p.tl, tl_n, 40);                       // kernel entry
  const int ntiles = p.m_tiles * p.n_tiles;
  const int nlocal = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  auto decode = [&](int j, int& m0, int& n0) {
    const int t = (int)blockIdx.x + j * (int)gridDim.x;
    m0 = (t / p.n_tiles) * BM;
    n0 = (t % p.n_tiles) * BN;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmA1h); tma_prefetch_desc(&tmA1l); tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
  }
  pdl_trigger();               // let the next kernel's prologue overlap our tail
  __syncthreads();
  pdl_wait();                  // everything below touches activations of the previous kernel
  tl_event(p.tl, tl_n, 41);                       // the previous kernel has completed

  if (warp < 4) {
    reg_dec<40>();
    if (warp != 0) return;
    // ---------------------------------------------------------------- TMA producer
    // The whole warp walks the loop (uniform control flow), one elected lane issues.
    int kbg = 0;                                   // k-block counter across tiles (ring position)
    for (int j = 0; j < nlocal; ++j) {
      int m0, n0;
      decode(j, m0, n0);
      tl_event(p.tl, tl_n, 1, j);                                    // producer: tile j begins
      for (int kb = 0; kb < p.kblocks; ++kb, ++kbg) {
        const int s = kbg % STAGES;
        mbar_wait(smem_u32(&bar_empty[s]), (((uint32_t)(kbg / STAGES)) & 1u) ^ 1u);
        if (elect_one()) {
          if (kb == 0 && j + 1 < nlocal) {
            // the ring is only two or three k-blocks deep: the NEXT tile's activation rows are pulled into L2
            // one whole tile ahead (weights are L2-resident anyway)
            int m1, n1;
            decode(j + 1, m1, n1);
            if (m1 != m0) {
              for (int k2 = 0; k2 < p.kblocks; ++k2) {
                if (k2 < p.kb1) { tma_prefetch_2d(&tmA1h, k2 * BK, m1); tma_prefetch_2d(&tmA1l, k2 * BK, m1); }
                else { tma_prefetch_2d(&tmA2h, (k2 - p.kb1) * BK, m1); tma_prefetch_2d(&tmA2l, (k2 - p.kb1) * BK, m1); }
              }
            }
          }
          const uint32_t full = smem_u32(&bar_full[s]);
          mbar_expect_tx(full, Cfg::STAGE_BYTES);
          const uint32_t sAh = smem_u32(smem + s * Cfg::STAGE_BYTES), sAl = sAh + Cfg::A_BYTES;
          const uint32_t sWh = sAl + Cfg::A_BYTES, sWl = sWh + Cfg::W_BYTES;
          if (kb < p.kb1) {
            tma_load_2d(sAh, &tmA1h, full, kb * BK, m0);
            tma_load_2d(sAl, &tmA1l, full, kb * BK, m0);
          } else {
            tma_load_2d(sAh, &tmA2h, full, (kb - p.kb1) * BK, m0);
            tma_load_2d(sAl, &tmA2l, full, (kb - p.kb1) * BK, m0);
          }
          tma_load_2d(sWh, &tmWh, full, kb * BK, n0);       // rows >= N are zero-filled (and counted)
          tma_load_2d(sWl, &tmWl, full, kb * BK, n0);
        }
        __syncwarp();
      }
    }
    return;
  }
  // ------------------------------------------------------------------ consumer warpgroups
  reg_inc<232>();
  const int cw = (warp >> 2) - 1;                    // which 64 rows of the tile
  const int cp = 2 * (lane & 3);                     // column offset inside an 8-column group
  float d[BN / 2];
  int kbg = 0;
  for (int it = 0; it < nlocal; ++it) {
    int m0, n0;
    decode(it, m0, n0);
    tl_event(p.tl, tl_n, 2, it);                                     // MMA: tile `it` begins
    for (int kb = 0; kb < p.kblocks; ++kb, ++kbg) {
      const int s = kbg % STAGES;
      mbar_wait(smem_u32(&bar_full[s]), ((uint32_t)(kbg / STAGES)) & 1u);
      const uint32_t sAh = smem_u32(smem + s * Cfg::STAGE_BYTES) + cw * (64 * 128), sAl = sAh + Cfg::A_BYTES;
      const uint32_t sWh = smem_u32(smem + s * Cfg::STAGE_BYTES) + 2 * Cfg::A_BYTES, sWl = sWh + Cfg::W_BYTES;
      wg_fence();
      kblock_ss<BN>(d, sAh, sAl, sWh, sWl, kb == 0);
      wg_commit();
      if (kb > 0) {                                  // the previous k-block's MMAs have retired: free its stage
        wg_wait<1>();
        if (lane == 0) mbar_arrive(smem_u32(&bar_empty[(kbg - 1) % STAGES]));
      }
    }
    wg_wait<0>();
    acc_fence(d);
    if (lane == 0) mbar_arrive(smem_u32(&bar_empty[(kbg - 1) % STAGES]));
    tl_event(p.tl, tl_n, 4, it);                                     // epilogue: accumulator of tile `it` ready

    const int r_lo = m0 + cw * 64 + (warp & 3) * 16 + (lane >> 2);
    if constexpr (EPI == EPI_LN) {
      ln_epilogue(d, p.inv_scale, p.bias, p.res_hi, p.res_lo, p.ld_res, p.gamma, p.beta, p.out_hi, p.out_lo, p.ld_out,
                  r_lo, p.M, cp);
    } else if constexpr (EPI == EPI_FAST) {
      const float sc = p.inv_scale;
      const bool ok0 = r_lo < p.M, ok1 = r_lo + 8 < p.M;
      const int64_t o0 = (int64_t)r_lo * p.ld_out + p.out_col0 + n0 + cp, o1 = o0 + (int64_t)8 * p.ld_out;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + cp));
        float x0 = fmaf(d[4 * j], sc, b.x), x1 = fmaf(d[4 * j + 1], sc, b.y);
        float x2 = fmaf(d[4 * j + 2], sc, b.x), x3 = fmaf(d[4 * j + 3], sc, b.y);
        if (ACT == ACT_GELU) { x0 = gelu_fast(x0); x1 = gelu_fast(x1); x2 = gelu_fast(x2); x3 = gelu_fast(x3); }
        if (ok0) store_split2(p.out_hi, p.out_lo, o0 + 8 * j, x0, x1);
        if (ok1) store_split2(p.out_hi, p.out_lo, o1 + 8 * j, x2, x3);
      }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = r_lo + 8 * h;
        if (m >= p.M) continue;
        int seq = 0, pos = m;
        if (p.in_group < p.M) { seq = m / p.in_group; pos = m - seq * p.in_group; }
        const int64_t orow = (int64_t)seq * p.out_group + p.out_off + pos;
        const bool zero = p.zero_lengths != nullptr && pos >= p.zero_lengths[seq];
        const float* tab = p.addtab ? p.addtab + (int64_t)(p.out_off + pos) * p.N : nullptr;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = n0 + 8 * j + cp + e;
            if (n >= p.N) continue;
            float x = d[4 * j + 2 * h + e] * p.inv_scale + (p.bias ? p.bias[n] : 0.0f);
            if (tab) x += tab[n];
            x = zero ? 0.0f : apply_act(x, p.act);
            if (p.out_hi) {
              __half hh, ll;
              split_f32(x, hh, ll);
              const int64_t o = orow * p.ld_out + p.out_col0 + n;
              p.out_hi[o] = hh; p.out_lo[o] = ll;
            }
            if (p.out_f32) p.out_f32[orow * p.ldc + n] = x;
          }
        }
      }
    }
    tl_event(p.tl, tl_n, 5, it);                                     // epilogue: tile `it` stored
  }
  tl_event(p.tl, tl_n, 42);                       // kernel exit
}

// ------------------------------------------------------------------------------ fused FFN
// y = LayerNorm(res + W2 gelu(W1 x + b1) + b2) for d = 256 as ONE persistent launch in which the
// hidden activations never leave the register file (the unfused pair writes and re-reads 2 x 4 x ff
// bytes per row through HBM, which is what bounds it).  A CTA owns 128-row m-tiles, 64 rows per
// consumer warpgroup; the x tile (both planes, 128 KB) stays in shared memory while the warpgroup
// walks the hidden dimension in 64-column chunks:
//   F1(c): acc1[64 x 64]   = x[64 x 256] . W1[c*64.., :]^T                (4 k-blocks, operands in shared memory)
//   E1(c): acc1 -> *s1 + b1 -> GELU -> split16 A fragments (the accumulator layout of 16 columns IS the
//          register-operand layout of a 16-deep k-step, so the hidden chunk never touches shared memory)
//   F2(c): acc2[64 x 256] += H[64 x 64] . W2[:, c*64..]^T                  (A from registers)
// and finishes with the residual + LayerNorm epilogue on acc2.  The TMA warp streams W1 / W2 through a ring of
// three 32 KB slots, four per chunk: W1 k-blocks 0-1, W1 k-blocks 2-3, W2 hi plane, W2 lo plane.  F2(c)'s last
// group stays in flight under F1(c + 1); the other warpgroup's MMAs cover this one's GELU.
struct FfnParams {
  int M, m_tiles, n_chunks;
  // Work decomposition (see k_ffn_tc): every CTA runs `full` whole m-tiles; the `left` tiles that do
  // not fill another round are cut along the hidden dimension into `parts` pieces, one per CTA.
  int full, left, parts;
  float* scratch;              // [slot][128 rows][256] fp32 partial accumulators of the pieces
  int* flags;                  // [slot] 1 = partial written (reset by the reader)
  int reverse;                 // walk the tiles from the last one down (snake order, see tc_attention)
  long long* tl;
  float inv_s1, inv_s2;
  const float* b1; const float* b2; const float* gamma; const float* beta;
  const __half* res_hi; const __half* res_lo; int ld_res;
  __half* out_hi; __half* out_lo; int ld_out;
};
struct FfnCfg {
  static constexpr int CHUNK = 64;                       // hidden columns per chunk
  static constexpr int X_BYTES = 2 * 4 * BM * 128;       // [plane][k-block][128 rows x 128 B]
  static constexpr int STAGE_BYTES = 32768, STAGES = 3;
  static constexpr int SMEM_BYTES = X_BYTES + STAGES * STAGE_BYTES + 256 + 1024;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
k_ffn_tc(const __grid_constant__ CUtensorMap tmXh, const __grid_constant__ CUtensorMap tmXl,
         const __grid_constant__ CUtensorMap tmW1h, const __grid_constant__ CUtensorMap tmW1l,
         const __grid_constant__ CUtensorMap tmW2h, const __grid_constant__ CUtensorMap tmW2l, const FfnParams p) {
  using Cfg = FfnCfg;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ring = smem + Cfg::X_BYTES;
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(ring + STAGES * Cfg::STAGE_BYTES);   // [STAGES] ring slot filled (TMA tx)
  uint64_t* bar_empty = bar_full + STAGES;    // [STAGES] ring slot consumed (one arrival per consumer warp)
  uint64_t* bar_xfull = bar_empty + STAGES;   // x tile landed
  uint64_t* bar_xempty = bar_xfull + 1;       // ... and read by the tile's last F1

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  int tl_n = 0;
  tl_event(p.tl, tl_n, 40);                       // kernel entry
  const int ncta = (int)gridDim.x, cid = (int)blockIdx.x;
  const int NC = p.n_chunks;
  // Items of this CTA: `full` whole tiles (cid, cid + ncta, ...), then - for the first left * parts CTAs - one
  // PIECE of a leftover tile: hidden chunks [c0, c1) of tile full * ncta + cid / parts.  Pieces 0 .. parts-2 are
  // contributors (their raw fp32 accumulator goes to `scratch`), the last piece is the finisher (adds the
  // contributors' accumulators in piece order, then bias + residual + LayerNorm as for a whole tile).
  // Contributors have lower CTA ids than their finisher, so they are scheduled no later than it.
  struct Item { int mt, c0, c1, mode, piece0; };             // mode: 0 whole tile, 1 contributor, 2 finisher
  auto rev = [&](int t) { return p.reverse ? p.m_tiles - 1 - t : t; };
  const int nlocal = p.full + (cid < p.left * p.parts ? 1 : 0);
  auto item = [&](int j) -> Item {
    if (j < p.full) return Item{rev(cid + j * ncta), 0, NC, 0, 0};
    const int t = cid / p.parts, part = cid - t * p.parts;
    const int c0 = (part * NC + p.parts - 1) / p.parts, c1 = ((part + 1) * NC + p.parts - 1) / p.parts;
    const int slot0 = t * (p.parts - 1);                     // slot of piece k of this tile: slot0 + k
    return Item{rev(p.full * ncta + t), c0, c1, p.parts == 1 ? 0 : (part == p.parts - 1 ? 2 : 1),
                p.parts == 1 ? 0 : slot0 + (part == p.parts - 1 ? 0 : part)};
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), CONSUMER_WARPS);
    }
    mbar_init(smem_u32(bar_xfull), 1);
    mbar_init(smem_u32(bar_xempty), CONSUMER_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmXh); tma_prefetch_desc(&tmXl); tma_prefetch_desc(&tmW1h);
    tma_prefetch_desc(&tmW1l); tma_prefetch_desc(&tmW2h); tma_prefetch_desc(&tmW2l);
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();
  tl_event(p.tl, tl_n, 41);                       // the previous kernel has completed

  if (warp < 4) {
    reg_dec<40>();
    if (warp != 0) return;
    // ---------------------------------------------------------------- TMA producer
    int rc = 0;                                    // ring position
    auto slot_wait = [&]() { mbar_wait(smem_u32(&bar_empty[rc % STAGES]), (((uint32_t)(rc / STAGES)) & 1u) ^ 1u); };
    for (int j = 0; j < nlocal; ++j) {
      const Item it = item(j);
      const int m0 = it.mt * BM;
      mbar_wait(smem_u32(bar_xempty), ((uint32_t)j & 1u) ^ 1u);
      if (elect_one()) {
        const uint32_t full = smem_u32(bar_xfull);
        mbar_expect_tx(full, Cfg::X_BYTES);
        for (int kb = 0; kb < 4; ++kb) {
          tma_load_2d(smem_u32(smem + kb * 16384), &tmXh, full, kb * BK, m0);
          tma_load_2d(smem_u32(smem + 65536 + kb * 16384), &tmXl, full, kb * BK, m0);
        }
        if (j + 1 < nlocal) {                      // next tile's x rows -> L2, a whole tile ahead
          const int m1 = item(j + 1).mt * BM;
          for (int k2 = 0; k2 < 4; ++k2) { tma_prefetch_2d(&tmXh, k2 * BK, m1); tma_prefetch_2d(&tmXl, k2 * BK, m1); }
        }
      }
      __syncwarp();
      for (int c = it.c0; c < it.c1; ++c) {
        for (int half = 0; half < 2; ++half, ++rc) {           // W1 rows [c*64, +64): k-blocks 2*half, 2*half + 1, hi then lo
          slot_wait();
          if (elect_one()) {
            const uint32_t full = smem_u32(&bar_full[rc % STAGES]);
            const uint32_t dst = smem_u32(ring + (rc % STAGES) * Cfg::STAGE_BYTES);
            mbar_expect_tx(full, Cfg::STAGE_BYTES);
            for (int k = 0; k < 2; ++k) {
              tma_load_2d(dst + k * 8192, &tmW1h, full, (2 * half + k) * BK, c * Cfg::CHUNK);
              tma_load_2d(dst + 16384 + k * 8192, &tmW1l, full, (2 * half + k) * BK, c * Cfg::CHUNK);
            }
          }
          __syncwarp();
        }
        for (int pl = 0; pl < 2; ++pl, ++rc) {                 // W2[:, c*64 .. +64): hi plane, then lo plane
          slot_wait();
          if (elect_one()) {
            const uint32_t full = smem_u32(&bar_full[rc % STAGES]);
            mbar_expect_tx(full, Cfg::STAGE_BYTES);
            tma_load_2d(smem_u32(ring + (rc % STAGES) * Cfg::STAGE_BYTES), pl ? &tmW2l : &tmW2h, full, c * Cfg::CHUNK, 0);
          }
          __syncwarp();
        }
      }
    }
    return;
  }
  // ------------------------------------------------------------------ consumer warpgroups
  reg_inc<232>();
  const int cw = (warp >> 2) - 1;
  const int cp = 2 * (lane & 3);
  const uint32_t sX = smem_u32(smem) + cw * (64 * 128);
  float acc2[128];
  float acc1[32];
  uint32_t hh[4][4], hl[4][4];                     // the hidden chunk as A fragments: [16-deep k-step][register]
  int rc = 0;
  auto slot_full = [&](int r) { mbar_wait(smem_u32(&bar_full[r % STAGES]), ((uint32_t)(r / STAGES)) & 1u); };
  auto slot_free = [&](int r) { if (lane == 0) mbar_arrive(smem_u32(&bar_empty[r % STAGES])); };
  for (int j = 0; j < nlocal; ++j) {
    const Item it = item(j);
    const int m0 = it.mt * BM;
    mbar_wait(smem_u32(bar_xfull), (uint32_t)j & 1u);
    tl_event(p.tl, tl_n, 2, j);                                      // x tile landed
    int pend = -1;                                   // ring position of the F2 group still in flight
    for (int c = it.c0; c < it.c1; ++c) {
      // ---- F1(c)
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        slot_full(rc + half);
        const uint32_t w = smem_u32(ring + ((rc + half) % STAGES) * Cfg::STAGE_BYTES);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const uint32_t xh = sX + (2 * half + k) * 16384;
          kblock_ss<64>(acc1, xh, xh + 65536, w + k * 8192, w + 16384 + k * 8192, half == 0 && k == 0);
        }
        wg_commit();
      }
      wg_wait<0>();
      acc_fence(acc1);
      if (pend >= 0) slot_free(pend);
      slot_free(rc); slot_free(rc + 1);
      rc += 2;
      if (c == it.c1 - 1 && lane == 0) mbar_arrive(smem_u32(bar_xempty));     // the x tile may be overwritten
      // ---- E1(c): bias + GELU -> split16 A fragments
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          const int jj = 2 * ks + g, n = c * Cfg::CHUNK + 8 * jj + cp;
          const float2 b = p.b1 ? __ldg(reinterpret_cast<const float2*>(p.b1 + n)) : make_float2(0.0f, 0.0f);
          split2(gelu_fast(fmaf(acc1[4 * jj], p.inv_s1, b.x)), gelu_fast(fmaf(acc1[4 * jj + 1], p.inv_s1, b.y)),
                 hh[ks][2 * g], hl[ks][2 * g]);
          split2(gelu_fast(fmaf(acc1[4 * jj + 2], p.inv_s1, b.x)), gelu_fast(fmaf(acc1[4 * jj + 3], p.inv_s1, b.y)),
                 hh[ks][2 * g + 1], hl[ks][2 * g + 1]);
        }
      }
      // ---- F2(c): H_lo.W2_hi + H_hi.W2_hi on the hi slot, H_hi.W2_lo on the lo slot
      slot_full(rc);
      wg_fence();
      {
        const uint64_t wd = make_desc(smem_u32(ring + (rc % STAGES) * Cfg::STAGE_BYTES));
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          wgmma_rs_n256(acc2, hl[ks], wd + 2 * ks, (c == it.c0 && ks == 0) ? 0u : 1u);
          wgmma_rs_n256(acc2, hh[ks], wd + 2 * ks, 1u);
        }
      }
      wg_commit();
      slot_full(rc + 1);
      {
        const uint64_t wd = make_desc(smem_u32(ring + ((rc + 1) % STAGES) * Cfg::STAGE_BYTES));
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wgmma_rs_n256(acc2, hh[ks], wd + 2 * ks, 1u);
      }
      wg_commit();
      wg_wait<1>();
      slot_free(rc);
      pend = rc + 1;
      rc += 2;
    }
    wg_wait<0>();
    acc_fence(acc2);
    if (pend >= 0) slot_free(pend);
    tl_event(p.tl, tl_n, 4, j);                                      // acc2 complete
    const int rl = cw * 64 + (warp & 3) * 16 + (lane >> 2);          // this thread's first row inside the tile
    if (it.mode == 1) {
      // ---- contributor piece: the raw fp32 accumulator -> scratch, then the flag
      float* const dst = p.scratch + (size_t)it.piece0 * (BM * 256);
#pragma unroll
      for (int jj = 0; jj < 32; ++jj) {
        *reinterpret_cast<float2*>(dst + rl * 256 + 8 * jj + cp) = make_float2(acc2[4 * jj], acc2[4 * jj + 1]);
        *reinterpret_cast<float2*>(dst + (rl + 8) * 256 + 8 * jj + cp) = make_float2(acc2[4 * jj + 2], acc2[4 * jj + 3]);
      }
      __threadfence();
      named_bar_sync(1, CONSUMER_WARPS * 32);
      if (threadIdx.x == 128) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p.flags + it.piece0), "r"(1) : "memory");
      continue;
    }
    const int nparts = it.mode == 2 ? p.parts - 1 : 0;
    if (nparts > 0) {
      // ---- finisher: the contributors' partials must have landed; they are added in piece order
      if (lane == 0) {
        for (int pp = 0; pp < nparts; ++pp) {
          const int* f = p.flags + it.piece0 + pp;
          uint32_t v = 0;
          long long t_end = clock64() + 4000000000ll;      // ~2 s: a lost contributor is a bug, trap instead of hanging
          do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
            if (v == 0 && clock64() > t_end) __trap();
          } while (v == 0);
        }
      }
      __syncwarp();
      for (int pp = 0; pp < nparts; ++pp) {
        const float* src = p.scratch + (size_t)(it.piece0 + pp) * (BM * 256);
#pragma unroll
        for (int jj = 0; jj < 32; ++jj) {
          const float2 a = __ldcg(reinterpret_cast<const float2*>(src + rl * 256 + 8 * jj + cp));
          const float2 b = __ldcg(reinterpret_cast<const float2*>(src + (rl + 8) * 256 + 8 * jj + cp));
          acc2[4 * jj] += a.x; acc2[4 * jj + 1] += a.y; acc2[4 * jj + 2] += b.x; acc2[4 * jj + 3] += b.y;
        }
      }
      named_bar_sync(1, CONSUMER_WARPS * 32);                // everyone is past its partial loads: re-arm the flags
      if (threadIdx.x == 128)
        for (int pp = 0; pp < nparts; ++pp) p.flags[it.piece0 + pp] = 0;
    }
    ln_epilogue(acc2, p.inv_s2, p.b2, p.res_hi, p.res_lo, p.ld_res, p.gamma, p.beta, p.out_hi, p.out_lo, p.ld_out,
                m0 + rl, p.M, cp);
    tl_event(p.tl, tl_n, 5, j);                                      // LN tail done
  }
  tl_event(p.tl, tl_n, 42);                       // kernel exit
}

}  // namespace

// ------------------------------------------------------------------------------ host side
struct TcCtx {
  int device = 0;
  int sm_count = 132;
  int ffn_fused = 1;          // FFN1 + GELU + FFN2 + residual + LayerNorm as one launch (option ffn_fused)
  int ffn_split = 1;          // cut the leftover tiles of the fused FFN along the hidden dimension (option ffn_split)
  tc::PFN_tmapEncodeTiled encode = nullptr;
};

TcCtx* tc_create(int device) {
  TcCtx* c = new TcCtx();
  c->device = device;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
    mldb_set_err("cuTensorMapEncodeTiled is not available from the driver");
    delete c;
    return nullptr;
  }
  c->encode = (tc::PFN_tmapEncodeTiled)fn;
  cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device);
  e = cudaSuccess;
  auto opt_in = [&](auto kernel, int bytes) {
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  };
  opt_in(k_gemm_tc<256, EPI_FAST>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_FAST>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_FAST, ACT_GELU>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_FAST, ACT_GELU>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_GENERIC>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_GENERIC>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_LN>, TileCfg<256>::SMEM_BYTES);
  opt_in(k_ffn_tc, FfnCfg::SMEM_BYTES);
  if (e != cudaSuccess) {
    mldb_set_err(std::string("cudaFuncSetAttribute(k_gemm_tc): ") + cudaGetErrorString(e));
    delete c;
    return nullptr;
  }
  return c;
}
void tc_destroy(TcCtx* c) { delete c; }

// 2-D map over one fp16 plane [rows, cols] (cols contiguous), box = 64 cols x box_rows, 128B swizzle.
// Out-of-bounds rows/cols are zero-filled, so M and N need not be tile multiples.
static bool make_map(const TcCtx* c, CUtensorMap* m, const __half* base, int rows, int cols, int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * sizeof(__half)};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = c->encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

static int pick_bn(const GemmArgs& g) { return (g.w.N % 256 == 0) ? 256 : 128; }

bool tc_gemm_supported(const TcCtx* c, const GemmArgs& g) {
  if (!c) return false;
  if (g.a_kind != A_SPLIT || g.M < 1 || g.w.N > MAX_N) return false;
  if (g.K1 <= 0 || g.K1 % BK || g.K2 % BK || g.a1.cols != g.K1) return false;
  if (g.K2 > 0 && g.a2.cols != g.K2) return false;
  if (g.w.K != g.K1 + g.K2) return false;
  if (((uintptr_t)g.a1.hi & 15) || ((uintptr_t)g.w.w & 15)) return false;
  if (g.out.hi && ((g.out.cols % 8) || (g.out_col0 % 8))) return false;
  return true;
}

bool tc_gemm_ln_supported(const TcCtx* c, const GemmArgs& g, const LnArgs& l) {
  if (!tc_gemm_supported(c, g)) return false;
  if (g.w.N != 256 || l.d != 256 || g.act != ACT_NONE) return false;
  if (l.in_group != 0 || l.c != nullptr || l.out_f32 != nullptr || !l.out.hi) return false;
  if (l.out.cols != 256 || (l.res.hi && l.res.cols != 256)) return false;
  if (l.gamma2 || l.rowvec) return false;
  if (g.addtab || g.zero_lengths || g.in_group < g.M || g.out_group != 0 || g.out_off != 0) return false;
  return true;
}

static void fill_params(const GemmArgs& g, const LnArgs* ln, int bn, TcParams* out) {
  TcParams p{};
  p.M = g.M; p.N = g.w.N; p.kblocks = g.w.K / BK; p.kb1 = g.K1 / BK;
  p.inv_scale = g.w.inv_scale; p.bias = g.w.bias; p.addtab = g.addtab; p.act = g.act;
  p.in_group = g.in_group; p.out_group = g.out_group; p.out_off = g.out_off; p.zero_lengths = g.zero_lengths;
  if (ln) {
    p.out_hi = ln->out.hi; p.out_lo = ln->out.lo(); p.ld_out = ln->out.cols; p.out_col0 = 0;
    p.res_hi = ln->res.hi; p.res_lo = ln->res.hi ? ln->res.lo() : nullptr; p.ld_res = ln->res.cols;
    p.gamma = ln->gamma; p.beta = ln->beta;
  } else {
    p.out_hi = g.out.hi; p.out_lo = g.out.hi ? g.out.lo() : nullptr; p.ld_out = g.out.cols; p.out_col0 = g.out_col0;
    p.out_f32 = g.out_f32; p.ldc = g.ldc;
  }
  p.m_tiles = (g.M + BM - 1) / BM;
  p.n_tiles = (g.w.N + bn - 1) / bn;
  p.tl = tc::mldb_timeline_buffer();
  *out = p;
}

static bool map_fail(const char* what, int M, int N, int K) {
  char buf[160];
  snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%s M=%d N=%d K=%d)", what, M, N, K);
  mldb_set_err(buf);
  return false;
}

bool tc_gemm(TcCtx* c, const GemmArgs& g, const LnArgs* ln, cudaStream_t st) {
  CUtensorMap mA1h, mA1l, mA2h, mA2l, mWh, mWl;
  const int bn = ln ? 256 : pick_bn(g);
  bool ok = make_map(c, &mA1h, g.a1.hi, g.M, g.K1, BM) && make_map(c, &mA1l, g.a1.lo(), g.M, g.K1, BM);
  if (g.K2 > 0) ok = ok && make_map(c, &mA2h, g.a2.hi, g.M, g.K2, BM) && make_map(c, &mA2l, g.a2.lo(), g.M, g.K2, BM);
  else { mA2h = mA1h; mA2l = mA1l; }
  ok = ok && make_map(c, &mWh, g.w.w, g.w.N, g.w.K, bn) && make_map(c, &mWl, g.w.w + g.w.plane_stride, g.w.N, g.w.K, bn);
  if (!ok) return map_fail("gemm", g.M, g.w.N, g.w.K);
  TcParams p;
  fill_params(g, ln, bn, &p);
  // the fast plain epilogue: split16 output, identity row mapping, N a whole number of tiles
  const bool fast = !ln && g.out.hi && !g.out_f32 && !g.addtab && !g.zero_lengths && g.in_group >= g.M &&
                    g.out_group == 0 && g.out_off == 0 && g.w.N % bn == 0 && g.w.bias != nullptr &&
                    (g.act == ACT_NONE || g.act == ACT_GELU);
  const int ntiles = p.m_tiles * p.n_tiles;
  dim3 grid(ntiles < c->sm_count ? ntiles : c->sm_count);
#define MLDB_LAUNCH(BN_, ...)                                                                                      \
  launch_pdl(k_gemm_tc<BN_, __VA_ARGS__>, grid, dim3(NUM_THREADS), TileCfg<BN_>::SMEM_BYTES, st, mA1h, mA1l, mA2h, \
             mA2l, mWh, mWl, p)
#define MLDB_LAUNCH_SHAPE(...)                                                       \
  do {                                                                               \
    if (bn == 256) MLDB_LAUNCH(256, __VA_ARGS__); else MLDB_LAUNCH(128, __VA_ARGS__); \
  } while (0)
  if (ln)                             MLDB_LAUNCH(256, EPI_LN);
  else if (fast && g.act == ACT_GELU) MLDB_LAUNCH_SHAPE(EPI_FAST, ACT_GELU);
  else if (fast)                      MLDB_LAUNCH_SHAPE(EPI_FAST);
  else                                MLDB_LAUNCH_SHAPE(EPI_GENERIC);
#undef MLDB_LAUNCH_SHAPE
#undef MLDB_LAUNCH
  return true;
}

// FFN block (linear1 + GELU + linear2 + residual + LayerNorm) as one launch, d = 256.
int tc_set_ffn_split(TcCtx* c, int on) {
  if (!c) return 0;
  const int old = c->ffn_split;
  c->ffn_split = on;
  return old;
}
int tc_set_ffn_fused(TcCtx* c, int on) {
  if (!c) return 0;
  const int old = c->ffn_fused;
  c->ffn_fused = on;
  return old;
}
bool tc_ffn_supported(const TcCtx* c, const GemmArgs& g1, const GemmArgs& g2, const LnArgs& l2) {
  if (!c || !c->ffn_fused) return false;
  if (!tc_gemm_supported(c, g1) || !tc_gemm_ln_supported(c, g2, l2)) return false;
  if (g1.K1 != 256 || g1.K2 > 0 || g2.K2 > 0 || g1.M != g2.M) return false;
  if (g1.w.N % FfnCfg::CHUNK || g1.w.N > MAX_N || g1.w.N != g2.K1) return false;
  if (g1.act != ACT_GELU || g1.out_f32 || g1.addtab || g1.zero_lengths) return false;
  if (g1.in_group < g1.M || g1.out_group != 0 || g1.out_off != 0) return false;
  return true;
}
bool tc_ffn(TcCtx* c, const GemmArgs& g1, const GemmArgs& g2, const LnArgs& l2, float* scratch, int* flags, cudaStream_t st) {
  CUtensorMap mXh, mXl, mW1h, mW1l, mW2h, mW2l;
  const int m_tiles = (g1.M + BM - 1) / BM;
  const bool ok = make_map(c, &mXh, g1.a1.hi, g1.M, g1.K1, BM) && make_map(c, &mXl, g1.a1.lo(), g1.M, g1.K1, BM) &&
                  make_map(c, &mW1h, g1.w.w, g1.w.N, g1.w.K, FfnCfg::CHUNK) &&
                  make_map(c, &mW1l, g1.w.w + g1.w.plane_stride, g1.w.N, g1.w.K, FfnCfg::CHUNK) &&
                  make_map(c, &mW2h, g2.w.w, g2.w.N, g2.w.K, 256) &&
                  make_map(c, &mW2l, g2.w.w + g2.w.plane_stride, g2.w.N, g2.w.K, 256);
  if (!ok) return map_fail("ffn", g1.M, g1.w.N, g1.w.K);
  FfnParams p{};
  p.M = g1.M; p.m_tiles = m_tiles; p.n_chunks = g1.w.N / FfnCfg::CHUNK;
  p.tl = tc::mldb_timeline_buffer();
  p.inv_s1 = g1.w.inv_scale; p.inv_s2 = g2.w.inv_scale;
  p.b1 = g1.w.bias; p.b2 = g2.w.bias; p.gamma = l2.gamma; p.beta = l2.beta;
  p.res_hi = l2.res.hi; p.res_lo = l2.res.hi ? l2.res.lo() : nullptr; p.ld_res = l2.res.cols;
  p.out_hi = l2.out.hi; p.out_lo = l2.out.lo(); p.ld_out = l2.out.cols;
  const int ncta_max = c->sm_count;
  // whole rounds of tiles, then the leftover tiles cut along the hidden dimension so that the last round
  // uses (nearly) every SM instead of `left` of them (FfnParams).  scratch == nullptr, the ffn_split option
  // off or left * 2 > SMs: the leftover tiles run as whole tiles.
  p.full = m_tiles / ncta_max; p.left = m_tiles % ncta_max; p.parts = 1;
  p.scratch = scratch; p.flags = flags;
  if (p.left > 0 && scratch && flags && c->ffn_split) {
    const int parts = std::min(p.n_chunks, ncta_max / p.left);
    if (parts >= 2 && (size_t)p.left * (parts - 1) * (BM * 256 * 4) <= TC_FFN_SCRATCH_BYTES) p.parts = parts;
  }
  const int ncta = p.full > 0 ? ncta_max : p.left * p.parts;
  static const int snake = [] { const char* e = getenv("MLDB_SNAKE"); return (e && !strcmp(e, "0")) ? 0 : 1; }();
  p.reverse = snake;
  launch_pdl(k_ffn_tc, dim3(ncta), dim3(NUM_THREADS), FfnCfg::SMEM_BYTES, st, mXh, mXl, mW1h, mW1l, mW2h, mW2l, p);
  return true;
}
