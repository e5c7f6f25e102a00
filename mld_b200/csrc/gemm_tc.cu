// Warpgroup-MMA (wgmma) split-fp16 kernels for sm_90a: the persistent GEMM with fused epilogues
// (k_gemm_tc), the fused FFN block (k_ffn_tc) and the K = 256 projection (k_proj_tc).
//
//   D[128 x BN] (fp32, registers) = A_hi W_hi^T + A_lo W_hi^T + A_hi W_lo^T        per 128-row tile
//
// A = activations in the split16 format (two fp16 planes, row-major [M, K]); W = nn.Linear weight
// [N, K] (PyTorch's [out, in] layout is already the K-major B operand), also split into hi/lo
// planes.  Three f16 MMAs per K-step reproduce the reference's fp32 GEMM to ~1e-6.
//
// k_gemm_tc: CTA = three warpgroups, one CTA per SM, persistent over tiles: warpgroup 0 gives its
// registers away (setmaxnreg) and its first warp is the TMA producer; warpgroups 1 and 2 each own 64
// rows of the tile, issue wgmma.mma_async on operands that stream through a ring of 128B-swizzled
// shared-memory tiles (BK = 64 halves = one swizzle row) and run the epilogue on their accumulator
// registers while the producer already fills the ring for the next tile.  k_ffn_tc keeps the two
// consumer warpgroups and drops the producer one (see there): its body needs more than the 168
// registers per thread a 384-thread CTA allows.
// Epilogues (a thread holds column pairs of two rows, a row is spread over the 4 lanes of a quad):
//   fast:      bias + activation -> split16, identity row mapping (the per-layer GEMMs)
//   generic:   + positional table, row remapping, zeroed padding rows, fp32 output, ragged N
//   LayerNorm: BN == N == 256, so a quad owns COMPLETE rows: bias + residual, exact two-pass
//              statistics over the registers with quad shuffles, normalise -> split16.
//   residual:  bias + fp32 residual R -> fp32 (may run in place, out == R: the text tower's residual stream).
//   fp32:      bias + activation -> fp32 with float2 stores, identity row mapping (GemmArgs::vec_f32: the T2M evaluator).
#include "gemm_tc.h"

#include <algorithm>

#include "tc_common.cuh"

namespace {
using namespace tc;

constexpr int MMA_THREADS = 256;                     // k_ffn_tc, k_proj_tc: the two MMA warpgroups only
constexpr int MAX_N = 1024;
constexpr int MAX_N_WIDE = 4096;                     // GemmArgs::wide_n

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
  const float* res_f32;                              // EPI_RES: [M, N] fp32, leading dimension ldc (may alias out_f32)
  int in_group, out_group, out_off;
  const int32_t* zero_lengths;
  // residual + LayerNorm epilogue
  const __half* res_hi; const __half* res_lo; int ld_res;
  const float* gamma; const float* beta;
  long long* tl; // debug timeline (nullptr normally)
};

enum { EPI_FAST = 0, EPI_LN = 1, EPI_GENERIC = 2, EPI_RES = 3, EPI_F32 = 4 };     // epilogue variants of k_gemm_tc (see the kernel)

// [A hi | A lo | W hi | W lo] stages (tc_common.cuh): two of 96 KB at BN = 256, three of 64 KB at BN = 128
template <int BN>
using TileCfg = StageLayout<BN, BN == 256 ? 2 : 3>;

// The fast epilogue's math on 8-column group j of an accumulator fragment: x[0..1] = act(d * sc + b) of this
// thread's first row, x[2..3] of its second.  b: the bias of the thread's column pair in group j.
template <int ACT, int N>
__device__ __forceinline__ void fast_group(const float (&d)[N], int j, float sc, float2 b, float (&x)[4]) {
  x[0] = fmaf(d[4 * j], sc, b.x); x[1] = fmaf(d[4 * j + 1], sc, b.y);
  x[2] = fmaf(d[4 * j + 2], sc, b.x); x[3] = fmaf(d[4 * j + 3], sc, b.y);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (ACT == ACT_GELU) x[e] = gelu_fast(x[e]);
    if (ACT == ACT_QUICKGELU) x[e] = quick_gelu_f(x[e]);
    if (ACT == ACT_LEAKY) x[e] = apply_act(x[e], ACT_LEAKY);
  }
}

// 4 x 4 transpose across the lanes of a quad: lane l holds v[g] = word l of group g and gets word g of group l.
// Two shuffle rounds of two words each.
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4], int l) {
  const bool b2 = l & 2, b1 = l & 1;
  uint32_t r0 = __shfl_xor_sync(0xffffffffu, b2 ? v[0] : v[2], 2), r1 = __shfl_xor_sync(0xffffffffu, b2 ? v[1] : v[3], 2);
  if (b2) { v[0] = r0; v[1] = r1; } else { v[2] = r0; v[3] = r1; }
  r0 = __shfl_xor_sync(0xffffffffu, b1 ? v[0] : v[1], 1); r1 = __shfl_xor_sync(0xffffffffu, b1 ? v[2] : v[3], 1);
  if (b1) { v[0] = r0; v[2] = r1; } else { v[1] = r0; v[3] = r1; }
}

// Ring producer of the two-warpgroup kernels (k_ffn_tc, k_proj_tc), run by warp 0 between its own MMAs: load every
// position up to `need` (blocking on its slot: warp 0 reads that position next), then those whose slot is already
// free.  Warp-uniform.
template <int S, class Load>
__device__ __forceinline__ void ring_produce(int& q_next, int total, int need, const Ring<S>& ring, Load&& load) {
  while (q_next < total) {
    if (q_next <= need) ring.wait_empty(q_next);
    else if (!__shfl_sync(0xffffffffu, (int)ring.test_empty(q_next), 0)) break;
    load(q_next++);
  }
}

// y = LayerNorm(acc * sc + bias + residual) * gamma + beta over the 256-wide rows of a [64 x 256] accumulator
// fragment, eps 1e-5.  cp: this thread's column offset inside an 8-column group.  The residual and the output go
// through the caller: res(j, x) adds the residual of 8-column group j to x[0..1] (first row) and x[2..3] (second
// row); out(j, y) stores group j's normalised values in the same layout.  The statistics are two exact passes over
// the registers; a row's four lanes are merged with shuffles in a fixed order, so the result does not depend on
// which CTA ran the tile, nor on where the residual came from.
template <class Res, class Out>
__device__ __forceinline__ void ln_rows(float (&d)[128], float sc, const float* bias, const float* gamma,
                                        const float* beta, int cp, Res&& res, Out&& out) {
  float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int n = 8 * j + cp;
    const float2 b = bias ? __ldg(reinterpret_cast<const float2*>(bias + n)) : make_float2(0.0f, 0.0f);
    float x[4] = {fmaf(d[4 * j], sc, b.x), fmaf(d[4 * j + 1], sc, b.y), fmaf(d[4 * j + 2], sc, b.x),
                  fmaf(d[4 * j + 3], sc, b.y)};
    res(j, x);
    d[4 * j] = x[0]; d[4 * j + 1] = x[1]; d[4 * j + 2] = x[2]; d[4 * j + 3] = x[3];
    s0 += x[0] + x[1]; s1 += x[2] + x[3];
  }
  const float mean0 = quad_sum(s0) * (1.0f / 256), mean1 = quad_sum(s1) * (1.0f / 256);
  float q0 = 0.0f, q1 = 0.0f;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float a0 = d[4 * j] - mean0, a1 = d[4 * j + 1] - mean0, a2 = d[4 * j + 2] - mean1, a3 = d[4 * j + 3] - mean1;
    d[4 * j] = a0; d[4 * j + 1] = a1; d[4 * j + 2] = a2; d[4 * j + 3] = a3;
    q0 = fmaf(a0, a0, fmaf(a1, a1, q0));
    q1 = fmaf(a2, a2, fmaf(a3, a3, q1));
  }
  const float rstd0 = rsqrtf(quad_sum(q0) * (1.0f / 256) + 1e-5f), rstd1 = rsqrtf(quad_sum(q1) * (1.0f / 256) + 1e-5f);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int n = 8 * j + cp;
    const float2 g = __ldg(reinterpret_cast<const float2*>(gamma + n)), be = __ldg(reinterpret_cast<const float2*>(beta + n));
    const float y[4] = {fmaf(d[4 * j] * rstd0, g.x, be.x), fmaf(d[4 * j + 1] * rstd0, g.y, be.y),
                        fmaf(d[4 * j + 2] * rstd1, g.x, be.x), fmaf(d[4 * j + 3] * rstd1, g.y, be.y)};
    out(j, y);
  }
}

// ln_rows with the residual read from and the output written to split16 planes in global memory (k_gemm_tc).
// r_lo: this thread's first row (the second is r_lo + 8); rows >= M are neither read nor written.
__device__ __forceinline__ void ln_epilogue(float (&d)[128], float sc, const float* bias, const __half* res_hi,
                                            const __half* res_lo, int ld_res, const float* gamma, const float* beta,
                                            __half* out_hi, __half* out_lo, int ld_out, int r_lo, int M, int cp) {
  const bool ok0 = r_lo < M, ok1 = r_lo + 8 < M;
  ln_rows(d, sc, bias, gamma, beta, cp,
          [&](int j, float (&x)[4]) {
            if (!res_hi) return;
            const int n = 8 * j + cp;
            if (ok0) {
              const int64_t o = (int64_t)r_lo * ld_res + n;
              const float2 h = __half22float2(*reinterpret_cast<const __half2*>(res_hi + o));
              const float2 l = __half22float2(*reinterpret_cast<const __half2*>(res_lo + o));
              x[0] = (x[0] + h.x) + l.x; x[1] = (x[1] + h.y) + l.y;
            }
            if (ok1) {
              const int64_t o = (int64_t)(r_lo + 8) * ld_res + n;
              const float2 h = __half22float2(*reinterpret_cast<const __half2*>(res_hi + o));
              const float2 l = __half22float2(*reinterpret_cast<const __half2*>(res_lo + o));
              x[2] = (x[2] + h.x) + l.x; x[3] = (x[3] + h.y) + l.y;
            }
          },
          [&](int j, const float (&y)[4]) {
            const int n = 8 * j + cp;
            if (ok0) store_split2(out_hi, out_lo, (int64_t)r_lo * ld_out + n, y[0], y[1]);
            if (ok1) store_split2(out_hi, out_lo, (int64_t)(r_lo + 8) * ld_out + n, y[2], y[3]);
          });
}

// ln_rows in place on a [128 x 256] split16 tile in shared memory, laid out as TMA writes it with 128B swizzle:
// [plane][k-block][row][128 B], 16-byte chunk c of row r at chunk c ^ (r & 7).  The residual is read from the tile
// and the result written back over it; every thread touches only its own elements (rows rl, rl + 8 of the tile,
// rl & 7 = lane / 4), and a warp's accesses of one group fall in 8 distinct 16-byte chunks: no bank conflicts.
__device__ __forceinline__ void ln_tile(float (&d)[128], float sc, const float* bias, const float* gamma,
                                        const float* beta, uint8_t* tile, int rl, int lane, int cp) {
  uint8_t* const row0 = tile + rl * 128 + cp * 2;
  const int sw = lane >> 2;
  auto at = [&](int j, int h, int plane) {
    return reinterpret_cast<__half2*>(row0 + plane * 65536 + h * 1024 + (j >> 3) * 16384 + (((j & 7) ^ sw) << 4));
  };
  ln_rows(d, sc, bias, gamma, beta, cp,
          [&](int j, float (&x)[4]) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float2 hi = __half22float2(*at(j, h, 0)), lo = __half22float2(*at(j, h, 1));
              x[2 * h] = (x[2 * h] + hi.x) + lo.x; x[2 * h + 1] = (x[2 * h + 1] + hi.y) + lo.y;
            }
          },
          [&](int j, const float (&y)[4]) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              uint32_t hi, lo;
              split2(y[2 * h], y[2 * h + 1], hi, lo);
              *reinterpret_cast<uint32_t*>(at(j, h, 0)) = hi;
              *reinterpret_cast<uint32_t*>(at(j, h, 1)) = lo;
            }
          });
}

// ------------------------------------------------------------------------------ the kernel
// Persistent: CTA c walks tiles c, c + #CTAs, ...; tile t -> (m = t / n_tiles, n = t % n_tiles).
// EPI selects the epilogue: EPI_FAST = plain, split16 output, identity row mapping, N a whole number of tiles
// (the per-layer GEMMs); EPI_LN = residual + LayerNorm; EPI_GENERIC = plain with everything else (positional
// table, row remapping, zeroed padding rows, fp32 output, ragged N: the per-batch embedding / final-layer
// GEMMs) kept out of the hot kernels' instruction stream; EPI_RES = bias + fp32 residual -> fp32, N even;
// EPI_F32 = bias + activation -> fp32, identity row mapping, N even.
struct GemmTile { int m0, n0; };
template <int BN, int EPI, int ACT = ACT_NONE>      // ACT: the fast / fp32 epilogue's activation (NONE | GELU | QUICKGELU | LEAKY)
__global__ void __launch_bounds__(WS_THREADS, 1)
k_gemm_tc(const __grid_constant__ CUtensorMap tmA1h, const __grid_constant__ CUtensorMap tmA1l,
          const __grid_constant__ CUtensorMap tmA2h, const __grid_constant__ CUtensorMap tmA2l,
          const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const TcParams p) {
  static_assert(EPI != EPI_LN || BN == 256, "the LayerNorm epilogue covers a full 256-wide row");
  const auto tile = [&](int j) {
    const int t = (int)blockIdx.x + j * (int)gridDim.x;
    return GemmTile{(t / p.n_tiles) * BM, (t % p.n_tiles) * BN};
  };
  ws_cta<TileCfg<BN>>(
      tmA1h, tmA1l, tmWh, tmWl, p.tl, p.kblocks, [&] { return persistent_count(p.m_tiles * p.n_tiles); }, tile,
      [&](const GemmTile& t, int kb, const auto& s, uint32_t full) {
        if (kb < p.kb1) {
          tma_load_2d(s.ah, &tmA1h, full, kb * BK, t.m0);
          tma_load_2d(s.al, &tmA1l, full, kb * BK, t.m0);
        } else {
          tma_load_2d(s.ah, &tmA2h, full, (kb - p.kb1) * BK, t.m0);
          tma_load_2d(s.al, &tmA2l, full, (kb - p.kb1) * BK, t.m0);
        }
        tma_load_2d(s.wh, &tmWh, full, kb * BK, t.n0);   // rows >= N are zero-filled (and counted)
        tma_load_2d(s.wl, &tmWl, full, kb * BK, t.n0);
      },
      [&](const GemmTile& t, float (&d)[BN / 2], const TileThread& th) {
        const int r_lo = t.m0 + th.row(), n0 = t.n0, cp = th.cp;
        if constexpr (EPI == EPI_LN) {
          ln_epilogue(d, p.inv_scale, p.bias, p.res_hi, p.res_lo, p.ld_res, p.gamma, p.beta, p.out_hi, p.out_lo, p.ld_out,
                      r_lo, p.M, cp);
        } else if constexpr (EPI == EPI_FAST) {
          const bool ok0 = r_lo < p.M, ok1 = r_lo + 8 < p.M;
          const int64_t o0 = (int64_t)r_lo * p.ld_out + p.out_col0 + n0 + cp, o1 = o0 + (int64_t)8 * p.ld_out;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            float x[4];
            fast_group<ACT>(d, j, p.inv_scale, __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + cp)), x);
            if (ok0) store_split2(p.out_hi, p.out_lo, o0 + 8 * j, x[0], x[1]);
            if (ok1) store_split2(p.out_hi, p.out_lo, o1 + 8 * j, x[2], x[3]);
          }
        } else if constexpr (EPI == EPI_RES) {
          // each element of R is read and then overwritten by the same thread: in place is safe (plain loads, no __ldg)
          const float sc = p.inv_scale;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int n = n0 + 8 * j + cp;
            if (n >= p.N) continue;                    // N even: a column pair is in or out together
            const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + n)) : make_float2(0.0f, 0.0f);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (r_lo + 8 * h >= p.M) continue;
              const int64_t o = (int64_t)(r_lo + 8 * h) * p.ldc + n;
              const float2 r = *reinterpret_cast<const float2*>(p.res_f32 + o);
              *reinterpret_cast<float2*>(p.out_f32 + o) =
                  make_float2(fmaf(d[4 * j + 2 * h], sc, b.x) + r.x, fmaf(d[4 * j + 2 * h + 1], sc, b.y) + r.y);
            }
          }
        } else if constexpr (EPI == EPI_F32) {
          const float sc = p.inv_scale;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int n = n0 + 8 * j + cp;
            if (n >= p.N) continue;                    // N even: a column pair is in or out together
            const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + n)) : make_float2(0.0f, 0.0f);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (r_lo + 8 * h >= p.M) continue;
              const float x0 = apply_act(fmaf(d[4 * j + 2 * h], sc, b.x), ACT), x1 = apply_act(fmaf(d[4 * j + 2 * h + 1], sc, b.y), ACT);
              *reinterpret_cast<float2*>(p.out_f32 + (int64_t)(r_lo + 8 * h) * p.ldc + n) = make_float2(x0, x1);
            }
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
      },
      [&](const GemmTile& t, int j, int ntiles, int kb) {
        if (kb == 0 && j + 1 < ntiles) {
          // the ring is only two or three k-blocks deep: the NEXT tile's activation rows are pulled into L2
          // one whole tile ahead (weights are L2-resident anyway)
          const int m1 = tile(j + 1).m0;
          if (m1 != t.m0) {
            for (int k2 = 0; k2 < p.kblocks; ++k2) {
              if (k2 < p.kb1) { tma_prefetch_2d(&tmA1h, k2 * BK, m1); tma_prefetch_2d(&tmA1l, k2 * BK, m1); }
              else { tma_prefetch_2d(&tmA2h, (k2 - p.kb1) * BK, m1); tma_prefetch_2d(&tmA2l, (k2 - p.kb1) * BK, m1); }
            }
          }
        }
      });
}

// ------------------------------------------------------------------------------ fused FFN
// y = LayerNorm(x + W2 gelu(W1 x + b1) + b2) for d = 256 as ONE persistent launch in which the
// hidden activations never leave the register file (the unfused pair writes and re-reads 2 x 4 x ff
// bytes per row through HBM, which is what bounds it).  A CTA owns 128-row m-tiles, 64 rows per
// consumer warpgroup; the x tile (both planes, 128 KB) stays in shared memory while the warpgroup
// walks the hidden dimension in 64-column chunks:
//   F1(c): acc1[64 x 64]   = x[64 x 256] . W1[c*64.., :]^T                (4 k-blocks, operands in shared memory)
//   E1(c): acc1 -> *s1 + b1 -> GELU -> split16 A fragments (the accumulator layout of 16 columns IS the
//          register-operand layout of a 16-deep k-step, so the hidden chunk never touches shared memory)
//   F2(c): acc2[64 x 256] += H[64 x 64] . W2[:, c*64..]^T                  (A from registers)
// and finishes with the residual + LayerNorm epilogue on acc2: the residual is x, read from the x tile, and y is
// written over it and leaves through one TMA store per warpgroup (64 rows, rows >= M clipped by the tensor map).
// With FfnParams::prefix (tc_tail) the tile first holds the attention output `att` and the item begins with the
// block's out-projection + residual + LayerNorm, so that x1 = LN1(att W_o^T + b_o + x) is produced in the x tile:
//   P(kb): acc2 = sum over k-blocks kb of att . W_o^T   (kblock_ss<256> over k-blocks 0..3: k_gemm_tc<256, EPI_LN>'s
//          order, so x1 has the bits of the two-kernel path)
//   once att k-block kb has been read by both warpgroups, k-block kb of the layer input x is loaded over it;
//   LN1:   acc2 * s0 + b_o + x -> LayerNorm -> x1 (split16, in place in the x tile), then the FFN as above.
// W_o, W1 and W2 stream through a ring of three 32 KB slots: eight positions per item for W_o (k-block kb's hi /
// lo plane at 2 kb / 2 kb + 1), then four per chunk: W1 k-blocks 0-1, W1 k-blocks 2-3, W2 hi plane, W2 lo plane.
// F2(c)'s last group stays in flight under F1(c + 1); the other warpgroup's MMAs cover this one's GELU.
// CTA = the two MMA warpgroups only, 256 threads, one CTA per SM.  ptxas compiles a kernel under 65536 / (threads
// rounded up to whole warpgroups) registers per thread whatever setmaxnreg does at run time: 168 with a third
// (producer) warpgroup, which this body (~208) does not fit - it spilled and had its wgmma serialised - and 255
// without one.  The TMA loads are a handful of instructions, so warp 0 issues them between its own MMAs.
struct FfnParams {
  int M, m_tiles, n_chunks;
  // Work decomposition (see k_ffn_tc): every CTA runs `full` whole m-tiles; the `left` tiles that do
  // not fill another round are cut along the hidden dimension into `parts` pieces, one per CTA.
  int full, left, parts;
  float* scratch;              // [slot][128 rows][256] fp32 partial accumulators of the pieces
  int* flags;                  // [slot] 1 = partial written (reset by the reader)
  int reverse;                 // walk the tiles from the last one down (snake order, see tc_attention)
  int prefix;                  // 1: every item (each piece too) starts with the out-projection + LN1 (tc_tail)
  long long* tl;
  float inv_s0, inv_s1, inv_s2;
  const float* b0; const float* gamma1; const float* beta1;   // the prefix's out-projection bias and LayerNorm
  const float* b1; const float* b2; const float* gamma; const float* beta;
};
struct FfnCfg {
  static constexpr int CHUNK = 64;                       // hidden columns per chunk
  static constexpr int X_BYTES = 2 * 4 * BM * 128;       // [plane][k-block][128 rows x 128 B]
  static constexpr int STAGE_BYTES = 32768, STAGES = 3;
  static constexpr int SMEM_BYTES = X_BYTES + STAGES * STAGE_BYTES + 256 + 1024;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

// tmX: the FFN input x (with the prefix: the layer input, LN1's residual); tmA / tmWo: the attention output and
// W_o (read with the prefix only); tmY: the output planes, 64-row boxes.
__global__ void __launch_bounds__(MMA_THREADS, 1)
k_ffn_tc(const __grid_constant__ CUtensorMap tmXh, const __grid_constant__ CUtensorMap tmXl,
         const __grid_constant__ CUtensorMap tmW1h, const __grid_constant__ CUtensorMap tmW1l,
         const __grid_constant__ CUtensorMap tmW2h, const __grid_constant__ CUtensorMap tmW2l,
         const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
         const __grid_constant__ CUtensorMap tmWoh, const __grid_constant__ CUtensorMap tmWol,
         const __grid_constant__ CUtensorMap tmYh, const __grid_constant__ CUtensorMap tmYl, const FfnParams p) {
  using Cfg = FfnCfg;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
  uint8_t* ring = smem + Cfg::X_BYTES;
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(ring + STAGES * Cfg::STAGE_BYTES);
  const Ring<STAGES> wring{bar_full, bar_full + STAGES};                 // the weight ring
  const Ring<4> xring{bar_full + 2 * STAGES, bar_full + 2 * STAGES + 4};  // slot kb: k-block kb of the x tile

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  int tl_n = 0;
  tl_event(p.tl, tl_n, 40);                       // kernel entry
  const int ncta = (int)gridDim.x, cid = (int)blockIdx.x;
  const int NC = p.n_chunks;
  // Items of this CTA: `full` whole tiles (cid, cid + ncta, ...), then - for the first left * parts CTAs - one
  // PIECE of a leftover tile: hidden chunks [c0, c1) of tile full * ncta + cid / parts.  Pieces 0 .. parts-2 are
  // contributors (their raw fp32 accumulator goes to `scratch`), the last piece is the finisher (adds the
  // contributors' accumulators in piece order, then bias + residual + LayerNorm as for a whole tile).
  // Contributors have lower CTA ids than their finisher, so they are scheduled no later than it.  With the prefix
  // every piece computes x1 itself (LN1 is deterministic: the same bits in every piece).
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
  // ring positions of this CTA: PRE for the out-projection, then four per chunk, of every item in item order
  const int PRE = p.prefix ? 8 : 0;
  const int per_tile = PRE + 4 * NC;
  int total = p.full * per_tile;
  if (nlocal > p.full) {
    const Item it = item(p.full);
    total += PRE + 4 * (it.c1 - it.c0);
  }
  // x-tile fills: XG per item and k-block ([att,] x), item after item; fill v is k-block v & 3's (v >> 2)-th
  const int XG = p.prefix ? 2 : 1;
  const int xtotal = nlocal * 4 * XG;

  if (threadIdx.x == 0) {
    wring.init(CONSUMER_WARPS);
    xring.init(CONSUMER_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmXh); tma_prefetch_desc(&tmXl); tma_prefetch_desc(&tmW1h);
    tma_prefetch_desc(&tmW1l); tma_prefetch_desc(&tmW2h); tma_prefetch_desc(&tmW2l);
    tma_prefetch_desc(&tmYh); tma_prefetch_desc(&tmYl);
    if (p.prefix) { tma_prefetch_desc(&tmAh); tma_prefetch_desc(&tmAl); tma_prefetch_desc(&tmWoh); tma_prefetch_desc(&tmWol); }
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();
  tl_event(p.tl, tl_n, 41);                       // the previous kernel has completed

  // ---------------------------------------------------------------- TMA issue (warp 0, one elected lane)
  // Ring position q holds, for its item: q < PRE: plane q & 1 (hi, lo) of W_o's k-block q >> 1 (all 256 rows); then
  // for chunk c, (q - PRE) % 4 = 0 / 1: W1 rows [c*64, +64), k-blocks 0-1 / 2-3, hi then lo; 2 / 3: the hi / lo
  // plane of W2[:, c*64 .. +64).  It is loaded once position q - 3 (same slot) has been freed by all eight warps.
  int q_next = 0, x_next = 0;                      // next ring position / next x-tile fill
  auto load_slot = [&](int q) {
    const int j = min(q / per_tile, p.full);
    const Item it = item(j);
    const int r = q - j * per_tile;
    if (elect_one()) {
      const uint32_t full = wring.full_bar(q);
      const uint32_t dst = smem_u32(ring + (q % STAGES) * Cfg::STAGE_BYTES);
      mbar_expect_tx(full, Cfg::STAGE_BYTES);
      if (r < PRE) {
        tma_load_2d(dst, (r & 1) ? &tmWol : &tmWoh, full, (r >> 1) * BK, 0);
      } else {
        const int c = it.c0 + ((r - PRE) >> 2), k = (r - PRE) & 3;
        if (k < 2) {
          for (int kk = 0; kk < 2; ++kk) {
            tma_load_2d(dst + kk * 8192, &tmW1h, full, (2 * k + kk) * BK, c * Cfg::CHUNK);
            tma_load_2d(dst + 16384 + kk * 8192, &tmW1l, full, (2 * k + kk) * BK, c * Cfg::CHUNK);
          }
        } else {
          tma_load_2d(dst, k == 3 ? &tmW2l : &tmW2h, full, c * Cfg::CHUNK, 0);
        }
      }
    }
    __syncwarp();
  };
  auto load_x = [&](int v) {                       // fill v: k-block v & 3 of item v / (4 XG), both planes
    if (elect_one()) {
      const int j = v / (4 * XG), kb = v & 3;
      const bool att = p.prefix && (v >> 2) == j * XG;       // the item's first fill with the prefix: att
      const int m0 = item(j).mt * BM;
      const uint32_t full = smem_u32(&xring.full[kb]);
      mbar_expect_tx(full, 2 * BM * 128);
      tma_load_2d(smem_u32(smem + kb * 16384), att ? &tmAh : &tmXh, full, kb * BK, m0);
      tma_load_2d(smem_u32(smem + 65536 + kb * 16384), att ? &tmAl : &tmXl, full, kb * BK, m0);
      if (att && kb == 0)                          // this item's residual rows -> L2 while att is consumed
        for (int k2 = 0; k2 < 4; ++k2) { tma_prefetch_2d(&tmXh, k2 * BK, m0); tma_prefetch_2d(&tmXl, k2 * BK, m0); }
      if (v % (4 * XG) == 0 && j + 1 < nlocal) {   // the next item's rows -> L2, a whole item ahead
        const int m1 = item(j + 1).mt * BM;
        for (int k2 = 0; k2 < 4; ++k2) {
          tma_prefetch_2d(&tmXh, k2 * BK, m1); tma_prefetch_2d(&tmXl, k2 * BK, m1);
          if (p.prefix) { tma_prefetch_2d(&tmAh, k2 * BK, m1); tma_prefetch_2d(&tmAl, k2 * BK, m1); }
        }
      }
    }
    __syncwarp();
  };
  // Load every x-tile fill up to `need_x` and ring position up to `need` (blocking: warp 0 reads them next), then
  // those whose slot is already free.  Warp 0 blocks only where the other warpgroup can always make progress:
  //   - on x fills at the start of an item (freed by the previous item's last reads of the tile: its y store, or a
  //     contributor's last F1, which need nothing that has not been loaded) and, with the prefix, before LN1 (the
  //     residual over att k-block kb, freed by the out-projection MMAs of kb, which need only att and W_o);
  //   - on ring position q, whose slot frees when position q - 3 has been read.  Freeing position q never needs a
  //     load past q + 2 (a W_o k-block's planes q, q + 1 retire before q + 2 is asked for; F1 / F2 as before), so
  //     warp 0 never waits on its own warpgroup, and the other warpgroup's readers of q - 3 need at most positions
  //     up to q - 1 and the x fills of their item.  Warp 0 has issued those fills itself before asking for any
  //     position past the out-projection (it needs them for its own LN1 / F1).
  // Called by warp 0 only, warp-uniformly.
  auto produce = [&](int need, int need_x) {
    ring_produce(x_next, xtotal, need_x, xring, load_x);
    ring_produce(q_next, total, need, wring, load_slot);
  };

  // ------------------------------------------------------------------ both warpgroups: MMA + epilogue
  const int cw = warp >> 2;                        // which 64 rows of the tile
  const int cp = 2 * (lane & 3);
  const int rl = cw * 64 + (warp & 3) * 16 + (lane >> 2);          // this thread's first row inside the tile
  const uint32_t sX = smem_u32(smem) + cw * (64 * 128);
  float acc2[128];
  float acc1[32];
  uint32_t hh[4][4], hl[4][4];                     // the hidden chunk as A fragments: [16-deep k-step][register]
  int rc = 0;
  auto slot_full = [&](int r) { wring.wait_full(r); };
  auto slot_free = [&](int r) { if (lane == 0) wring.release(r); };
  auto x_full = [&](int kb, uint32_t par) { mbar_wait(smem_u32(&xring.full[kb]), par); };
  auto x_free = [&](int kb) { if (lane == 0) mbar_arrive(smem_u32(&xring.empty[kb])); };
  for (int j = 0; j < nlocal; ++j) {
    const Item it = item(j);
    const int m0 = it.mt * BM;
    const uint32_t xpar = (uint32_t)(j * XG) & 1u;               // parity of the item's first fill of each k-block
    if (warp == 0) produce(-1, 4 * j * XG + 3);
    if (p.prefix) {
      // ---- P(kb): acc2 = att . W_o^T.  A k-block holds two of the three ring slots, so its MMAs retire (and free
      // them, and the att k-block for the residual) before the next k-block's second plane is asked for: keeping
      // two k-blocks in flight would need four slots, and warp 0 would wait on a slot only its own warpgroup frees.
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) {
        if (warp == 0) produce(rc + 1, -1);
        x_full(kb, xpar);
        slot_full(rc); slot_full(rc + 1);
        const uint32_t wh = smem_u32(ring + (rc % STAGES) * Cfg::STAGE_BYTES);
        const uint32_t wl = smem_u32(ring + ((rc + 1) % STAGES) * Cfg::STAGE_BYTES);
        wg_fence();
        kblock_ss<256>(acc2, sX + kb * 16384, sX + 65536 + kb * 16384, wh, wl, kb == 0);
        wg_commit();
        wg_wait<0>();
        slot_free(rc); slot_free(rc + 1); x_free(kb);
        rc += 2;
        if (warp == 0) produce(-1, -1);            // the next k-block's hi plane goes into a slot freed earlier
        tl_event(p.tl, tl_n, 60, kb);                                // out-projection k-block kb retired
      }
      acc_fence(acc2);
      // ---- LN1: x1 = LN(acc2 * s0 + b_o + x) over the residual x, in place
      if (warp == 0) produce(-1, 4 * j * XG + 7);
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) x_full(kb, xpar ^ 1u);
      ln_tile(acc2, p.inv_s0, p.b0, p.gamma1, p.beta1, smem, rl, lane, cp);
      fence_async_smem();
      named_bar_sync(2 + cw, 128);                 // this warpgroup's 64 rows of x1 are written: its F1 may read them
      tl_event(p.tl, tl_n, 61, j);                                   // LN1 done
    } else {
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) x_full(kb, xpar);
    }
    tl_event(p.tl, tl_n, 2, j);                                      // x tile ready
    int pend = -1;                                   // ring position of the F2 group still in flight
    for (int c = it.c0; c < it.c1; ++c) {
      // ---- F1(c)
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        if (warp == 0) produce(rc + half, -1);
        slot_full(rc + half);
        tl_event(p.tl, tl_n, 10 + half, c);                          // W1 k-blocks 2 * half, +1 landed
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
      tl_event(p.tl, tl_n, 13, c);                                   // F1(c) retired
      if (pend >= 0) slot_free(pend);
      slot_free(rc); slot_free(rc + 1);
      rc += 2;
      if (c == it.c1 - 1 && it.mode == 1)          // a contributor does not read the x tile again
        for (int kb = 0; kb < 4; ++kb) x_free(kb);
      if (warp == 0) produce(-1, -1);
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
      tl_event(p.tl, tl_n, 14, c);                                   // GELU done
      // ---- F2(c): H_lo.W2_hi + H_hi.W2_hi on the hi slot, H_hi.W2_lo on the lo slot
      if (warp == 0) produce(rc, -1);
      slot_full(rc);
      tl_event(p.tl, tl_n, 12, c);                                   // W2 hi plane landed
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
      if (warp == 0) produce(rc + 1, -1);
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
      if (warp == 0) produce(-1, -1);
    }
    wg_wait<0>();
    acc_fence(acc2);
    if (pend >= 0) slot_free(pend);
    if (warp == 0) produce(-1, -1);
    tl_event(p.tl, tl_n, 4, j);                                      // acc2 complete
    if (it.mode == 1) {
      // ---- contributor piece: the raw fp32 accumulator -> scratch, then the flag
      float* const dst = p.scratch + (size_t)it.piece0 * (BM * 256);
#pragma unroll
      for (int jj = 0; jj < 32; ++jj) {
        *reinterpret_cast<float2*>(dst + rl * 256 + 8 * jj + cp) = make_float2(acc2[4 * jj], acc2[4 * jj + 1]);
        *reinterpret_cast<float2*>(dst + (rl + 8) * 256 + 8 * jj + cp) = make_float2(acc2[4 * jj + 2], acc2[4 * jj + 3]);
      }
      __threadfence();
      named_bar_sync(1, MMA_THREADS);
      if (threadIdx.x == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p.flags + it.piece0), "r"(1) : "memory");
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
      named_bar_sync(1, MMA_THREADS);                        // everyone is past its partial loads: re-arm the flags
      if (threadIdx.x == 0)
        for (int pp = 0; pp < nparts; ++pp) p.flags[it.piece0 + pp] = 0;
    }
    // ---- LN2: y = LN(acc2 * s2 + b2 + x) over the residual in the x tile, in place; then out through TMA
    ln_tile(acc2, p.inv_s2, p.b2, p.gamma, p.beta, smem, rl, lane, cp);
    fence_async_smem();
    named_bar_sync(2 + cw, 128);                   // this warpgroup's 64 rows of y are in the tile
    tl_event(p.tl, tl_n, 62, j);                                     // LN2 done
    if ((warp & 3) == 0) {
      // one thread per warpgroup stores its 64 rows and, once the stores have read the tile, frees it (4 arrivals
      // per warpgroup) for the next item's fills
      if (elect_one()) {
        if (m0 + cw * 64 < p.M) {
#pragma unroll
          for (int kb = 0; kb < 4; ++kb) {
            const uint32_t src = smem_u32(smem + kb * 16384 + cw * 8192);
            tma_store_2d(&tmYh, src, kb * BK, m0 + cw * 64);
            tma_store_2d(&tmYl, src + 65536, kb * BK, m0 + cw * 64);
          }
          bulk_commit();
          bulk_wait_read<0>();
        }
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) mbar_arrive_cnt(smem_u32(&xring.empty[kb]), 4);
      }
      __syncwarp();
      tl_event(p.tl, tl_n, 63, j);                                   // the y store has read the tile
    }
  }
  tl_event(p.tl, tl_n, 42);                       // kernel exit
}

// ------------------------------------------------------------------------------ K = 256 projection
// out = act(A W^T * s + b) -> split16 for K = 256 with one A source and N a multiple of 128 (the fast epilogue's
// shapes): the QKV / kv / q projections of the encoder layers and the VAE's d = 256 projections.  With only four
// k-blocks, k_gemm_tc spends about as long in its epilogue as in its MMAs, and both warpgroups reach the epilogue
// together, so nothing overlaps it.  Here the CTA is k_ffn_tc's F1 with a store epilogue:
//   - the two MMA warpgroups only (256 threads, 255 registers), warp 0 issues the TMA loads between its MMAs;
//   - the 128 x 256 A tile (both planes, 128 KB, one barrier pair per k-block) stays in shared memory while W
//     streams through three 32 KB ring slots, one k-block of a 128-column chunk per slot;
//   - each warpgroup keeps two 64 x 128 accumulators: the epilogue of chunk i - 1 runs while chunk i's k-blocks 1
//     and 2 are on the tensor cores.
// Work items are (m-tile, chunk) pairs in m-major order; each CTA takes one contiguous range of near-equal
// length and walks it upwards (the GEMMs' direction in the snake order), loading each A tile it touches once.
// The per-element accumulation order is kblock_ss's over k-blocks 0..3, as in k_gemm_tc, so the outputs are
// identical to k_gemm_tc's.
struct ProjParams {
  int M, n_chunks, items;                        // items = m-tiles x n_chunks
  float inv_scale;
  const float* bias;
  __half* out_hi; __half* out_lo; int ld_out, out_col0;
  long long* tl;
};
struct ProjCfg {
  static constexpr int CHUNK = 128;                      // output columns per chunk
  static constexpr int A_BYTES = 2 * 4 * BM * 128;       // [plane][k-block][128 rows x 128 B], as k_ffn_tc's x tile
  static constexpr int STAGE_BYTES = 2 * CHUNK * 128, STAGES = 3;   // one k-block of a chunk, both planes
  static constexpr int SMEM_BYTES = A_BYTES + STAGES * STAGE_BYTES + 256 + 1024;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

template <int ACT>                                     // the fast epilogue's activation (NONE | GELU | QUICKGELU | LEAKY)
__global__ void __launch_bounds__(MMA_THREADS, 1)
k_proj_tc(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
          const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const ProjParams p) {
  using Cfg = ProjCfg;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
  uint8_t* ring = smem + Cfg::A_BYTES;
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(ring + STAGES * Cfg::STAGE_BYTES);
  const Ring<STAGES> wring{bar_full, bar_full + STAGES};                 // the weight ring
  // slot k: k-block k of the A tile, freed by the last chunk of its tile
  const Ring<4> aring{bar_full + 2 * STAGES, bar_full + 2 * STAGES + 4};

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  int tl_n = 0;
  tl_event(p.tl, tl_n, 40);                       // kernel entry
  const int NC = p.n_chunks;
  // this CTA's items [t0, t0 + n), n >= 1 (the grid is at most the item count); local item i, local A tile j
  const int t0 = (int)((long long)blockIdx.x * p.items / gridDim.x);
  const int n = (int)((long long)(blockIdx.x + 1) * p.items / gridDim.x) - t0;
  const int mt0 = t0 / NC, ntiles = (t0 + n - 1) / NC - mt0 + 1;
  auto tile_of = [&](int i) { return (t0 + i) / NC - mt0; };
  auto first_of_tile = [&](int i) { return i == 0 || (t0 + i) % NC == 0; };
  auto last_of_tile = [&](int i) { return i == n - 1 || (t0 + i + 1) % NC == 0; };

  if (threadIdx.x == 0) {
    wring.init(CONSUMER_WARPS);
    aring.init(CONSUMER_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmAh); tma_prefetch_desc(&tmAl); tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();
  tl_event(p.tl, tl_n, 41);                       // the previous kernel has completed

  // ---------------------------------------------------------------- TMA issue (warp 0, one elected lane)
  // Two rings, both filled by ring_produce: W position q = 4 i + k (k-block k of item i's chunk) in slot q % 3, and
  // A position a = 4 j + k (k-block k of local tile j) in k-block slot k.  Freeing W position q never needs a load
  // past q + 2, and A k-block k of tile j is freed by MMAs that only need W positions and A tiles up to tile j, so
  // the other warpgroup can always free what warp 0 waits on.
  int q_next = 0, a_next = 0;
  auto load_w = [&](int q) {
    if (elect_one()) {
      const int c = (t0 + (q >> 2)) % NC, k = q & 3;
      const uint32_t full = wring.full_bar(q);
      const uint32_t dst = smem_u32(ring + (q % STAGES) * Cfg::STAGE_BYTES);
      mbar_expect_tx(full, Cfg::STAGE_BYTES);
      tma_load_2d(dst, &tmWh, full, k * BK, c * Cfg::CHUNK);         // rows >= N are zero-filled (and counted)
      tma_load_2d(dst + Cfg::STAGE_BYTES / 2, &tmWl, full, k * BK, c * Cfg::CHUNK);
    }
    __syncwarp();
  };
  auto load_a = [&](int a) {
    if (elect_one()) {
      const int j = a >> 2, k = a & 3, m0 = (mt0 + j) * BM;
      const uint32_t full = smem_u32(&aring.full[k]);
      mbar_expect_tx(full, 2 * BM * 128);
      tma_load_2d(smem_u32(smem + k * 16384), &tmAh, full, k * BK, m0);
      tma_load_2d(smem_u32(smem + 65536 + k * 16384), &tmAl, full, k * BK, m0);
      if (k == 0 && j + 1 < ntiles)                // the next tile's rows -> L2, a whole tile ahead
        for (int k2 = 0; k2 < 4; ++k2) { tma_prefetch_2d(&tmAh, k2 * BK, m0 + BM); tma_prefetch_2d(&tmAl, k2 * BK, m0 + BM); }
    }
    __syncwarp();
  };
  auto produce = [&](int need_w, int need_a) {     // warp 0 only, warp-uniformly
    ring_produce(a_next, 4 * ntiles, need_a, aring, load_a);
    ring_produce(q_next, 4 * n, need_w, wring, load_w);
  };

  // ------------------------------------------------------------------ both warpgroups: MMA + epilogue
  const int cw = warp >> 2;                        // which 64 rows of the tile
  const int cp = 2 * (lane & 3);
  const uint32_t sA = smem_u32(smem) + cw * (64 * 128);
  float acc0[64], acc1[64];
  auto retire = [&](int q) {                       // this warp's MMAs of W position q have retired
    if (lane == 0) {
      wring.release(q);
      if (last_of_tile(q >> 2)) mbar_arrive(smem_u32(&aring.empty[q & 3]));
    }
  };
  // The fast epilogue's math, then a quad transpose per four 8-column groups, so that each lane stores one group
  // of a row as 16 B per plane: a warp store writes 64 B row pieces instead of k_gemm_tc's 16 B ones.
  auto epilogue = [&](const float (&d)[64], int i) {
    const int t = t0 + i, r_lo = (t / NC) * BM + cw * 64 + (warp & 3) * 16 + (lane >> 2), n0 = (t % NC) * Cfg::CHUNK;
    const int l = lane & 3;
    const bool ok0 = r_lo < p.M, ok1 = r_lo + 8 < p.M;
    const int64_t o0 = (int64_t)r_lo * p.ld_out + p.out_col0 + n0 + 8 * l, o1 = o0 + (int64_t)8 * p.ld_out;
    tl_event(p.tl, tl_n, 52, i);                                     // epilogue of item i begins
#pragma unroll
    for (int jb = 0; jb < Cfg::CHUNK / 32; ++jb) {
      uint32_t h0[4], l0[4], h1[4], l1[4];        // [group jb * 4 + g]: hi / lo words of the first / second row
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const int j = 4 * jb + g;
        float x[4];
        fast_group<ACT>(d, j, p.inv_scale, __ldg(reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + cp)), x);
        split2(x[0], x[1], h0[g], l0[g]);
        split2(x[2], x[3], h1[g], l1[g]);
      }
      quad_transpose(h0, l); quad_transpose(l0, l); quad_transpose(h1, l); quad_transpose(l1, l);
      if (ok0) {
        *reinterpret_cast<uint4*>(p.out_hi + o0 + 32 * jb) = make_uint4(h0[0], h0[1], h0[2], h0[3]);
        *reinterpret_cast<uint4*>(p.out_lo + o0 + 32 * jb) = make_uint4(l0[0], l0[1], l0[2], l0[3]);
      }
      if (ok1) {
        *reinterpret_cast<uint4*>(p.out_hi + o1 + 32 * jb) = make_uint4(h1[0], h1[1], h1[2], h1[3]);
        *reinterpret_cast<uint4*>(p.out_lo + o1 + 32 * jb) = make_uint4(l1[0], l1[1], l1[2], l1[3]);
      }
    }
    tl_event(p.tl, tl_n, 53, i);                                     // ... stores issued
  };
  // Item i into `cur`.  After issuing each k-block, wait for the one before it and free its W slot (and A k-block);
  // item i - 1 is complete once k-block 0 has been issued, and its epilogue runs behind k-blocks 1 and 2.
  auto step = [&](int i, float (&cur)[64], float (&prev)[64]) {
    const bool fresh = first_of_tile(i);
    const int j = tile_of(i);
    tl_event(p.tl, tl_n, 50, i);                                     // item i begins
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int q = 4 * i + k;
      if (warp == 0) produce(q, fresh ? 4 * j + k : -1);
      if (fresh) {
        mbar_wait(aring.full_bar(k), aring.phase(4 * j));     // position 4 j + k
        if (k == 0) tl_event(p.tl, tl_n, 51, j);                    // A k-block 0 of tile j landed
      }
      wring.wait_full(q);
      const uint32_t w = smem_u32(ring + (q % STAGES) * Cfg::STAGE_BYTES), a = sA + k * 16384;
      wg_fence();
      kblock_ss<128>(cur, a, a + 65536, w, w + Cfg::STAGE_BYTES / 2, k == 0);
      wg_commit();
      if (k == 2) {
        if (warp == 0) produce(q + 1, -1);         // k-block 3's load must not wait behind the epilogue
        if (i > 0) epilogue(prev, i - 1);
      }
      if (q > 0) {
        wg_wait<1>();
        retire(q - 1);
      }
      if (k == 0 && i > 0) acc_fence(prev);
    }
  };
  for (int i = 0; i < n; i += 2) {
    step(i, acc0, acc1);
    if (i + 1 < n) step(i + 1, acc1, acc0);
  }
  wg_wait<0>();
  retire(4 * n - 1);
  if ((n - 1) & 1) {
    acc_fence(acc1);
    epilogue(acc1, n - 1);
  } else {
    acc_fence(acc0);
    epilogue(acc0, n - 1);
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
};

TcCtx* tc_create(int device) {
  if (!tc::tmap_encoder()) return nullptr;
  TcCtx* c = new TcCtx();
  c->device = device;
  cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device);
  bool ok = true;
  auto opt_in = [&](auto kernel, int bytes) { ok = ok && smem_opt_in(kernel, bytes, "k_gemm_tc"); };
  opt_in(k_gemm_tc<256, EPI_FAST>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_FAST>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_FAST, ACT_GELU>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_FAST, ACT_GELU>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_GENERIC>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_GENERIC>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_FAST, ACT_QUICKGELU>, TileCfg<256>::SMEM_BYTES);
  opt_in(k_gemm_tc<128, EPI_FAST, ACT_QUICKGELU>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_RES>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_RES>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_LN>, TileCfg<256>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_FAST, ACT_LEAKY>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_FAST, ACT_LEAKY>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_F32>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_F32>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_gemm_tc<256, EPI_F32, ACT_LEAKY>, TileCfg<256>::SMEM_BYTES); opt_in(k_gemm_tc<128, EPI_F32, ACT_LEAKY>, TileCfg<128>::SMEM_BYTES);
  opt_in(k_ffn_tc, FfnCfg::SMEM_BYTES);
  opt_in(k_proj_tc<ACT_NONE>, ProjCfg::SMEM_BYTES); opt_in(k_proj_tc<ACT_GELU>, ProjCfg::SMEM_BYTES);
  opt_in(k_proj_tc<ACT_QUICKGELU>, ProjCfg::SMEM_BYTES); opt_in(k_proj_tc<ACT_LEAKY>, ProjCfg::SMEM_BYTES);
  if (!ok) {
    delete c;
    return nullptr;
  }
  return c;
}
void tc_destroy(TcCtx* c) { delete c; }

static int pick_bn(const GemmArgs& g) { return (g.w.N % 256 == 0) ? 256 : 128; }

bool tc_gemm_supported(const TcCtx* c, const GemmArgs& g) {
  if (!c) return false;
  if (g.a_kind != A_SPLIT || g.M < 1 || g.w.N > (g.wide_n ? MAX_N_WIDE : MAX_N)) return false;
  if (g.K1 <= 0 || g.K1 % BK || g.K2 % BK || g.a1.cols != g.K1) return false;
  if (g.K2 > 0 && g.a2.cols != g.K2) return false;
  if (g.w.K != g.K1 + g.K2) return false;
  if (((uintptr_t)g.a1.hi & 15) || ((uintptr_t)g.w.w & 15)) return false;
  if (g.out.hi && ((g.out.cols % 8) || (g.out_col0 % 8))) return false;
  if (g.res_f32 && (!g.out_f32 || g.out.hi || g.act != ACT_NONE || g.addtab || g.zero_lengths || g.in_group < g.M ||
                    g.out_group != 0 || g.out_off != 0 || (g.w.N % 2) || (g.ldc % 2) || ((uintptr_t)g.out_f32 & 7) ||
                    ((uintptr_t)g.res_f32 & 7)))
    return false;
  return true;
}

bool tc_gemm_ln_supported(const TcCtx* c, const GemmArgs& g, const LnArgs& l) {
  if (!tc_gemm_supported(c, g)) return false;
  if (g.w.N != 256 || l.d != 256 || g.act != ACT_NONE) return false;
  if (l.in_group != 0 || l.c != nullptr || l.out_f32 != nullptr || !l.out.hi) return false;
  if (l.out.cols != 256 || (l.res.hi && l.res.cols != 256)) return false;
  if (l.rowvec) return false;
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
    p.out_f32 = g.out_f32; p.ldc = g.ldc; p.res_f32 = g.res_f32;
  }
  p.m_tiles = (g.M + BM - 1) / BM;
  p.n_tiles = (g.w.N + bn - 1) / bn;
  p.tl = tc::mldb_timeline_buffer();
  *out = p;
}

// k_proj_tc: the fast epilogue with K = 256 from one A source (every N here is a multiple of 128)
static bool tc_proj(TcCtx* c, const GemmArgs& g, cudaStream_t st) {
  CUtensorMap mAh, mAl, mWh, mWl;
  const bool ok = make_map(&mAh, g.a1.hi, g.M, g.K1, BM) && make_map(&mAl, g.a1.lo(), g.M, g.K1, BM) &&
                  make_map(&mWh, g.w.w, g.w.N, g.w.K, ProjCfg::CHUNK) &&
                  make_map(&mWl, g.w.w + g.w.plane_stride, g.w.N, g.w.K, ProjCfg::CHUNK);
  if (!ok) return false;
  ProjParams p{};
  p.M = g.M; p.n_chunks = g.w.N / ProjCfg::CHUNK; p.items = (g.M + BM - 1) / BM * p.n_chunks;
  p.inv_scale = g.w.inv_scale; p.bias = g.w.bias;
  p.out_hi = g.out.hi; p.out_lo = g.out.lo(); p.ld_out = g.out.cols; p.out_col0 = g.out_col0;
  p.tl = tc::mldb_timeline_buffer();
  const dim3 grid(p.items < c->sm_count ? p.items : c->sm_count);
  switch (g.act) {
    case ACT_GELU: launch_pdl(k_proj_tc<ACT_GELU>, grid, dim3(MMA_THREADS), ProjCfg::SMEM_BYTES, st, mAh, mAl, mWh, mWl, p); break;
    case ACT_QUICKGELU: launch_pdl(k_proj_tc<ACT_QUICKGELU>, grid, dim3(MMA_THREADS), ProjCfg::SMEM_BYTES, st, mAh, mAl, mWh, mWl, p); break;
    case ACT_LEAKY: launch_pdl(k_proj_tc<ACT_LEAKY>, grid, dim3(MMA_THREADS), ProjCfg::SMEM_BYTES, st, mAh, mAl, mWh, mWl, p); break;
    default: launch_pdl(k_proj_tc<ACT_NONE>, grid, dim3(MMA_THREADS), ProjCfg::SMEM_BYTES, st, mAh, mAl, mWh, mWl, p); break;
  }
  return true;
}

bool tc_gemm(TcCtx* c, const GemmArgs& g, const LnArgs* ln, cudaStream_t st) {
  const int bn = ln ? 256 : pick_bn(g);
  // the fast plain epilogue: split16 output, identity row mapping, N a whole number of tiles
  const bool fast = !ln && g.out.hi && !g.out_f32 && !g.addtab && !g.zero_lengths && g.in_group >= g.M &&
                    g.out_group == 0 && g.out_off == 0 && g.w.N % bn == 0 && g.w.bias != nullptr &&
                    (g.act == ACT_NONE || g.act == ACT_GELU || g.act == ACT_QUICKGELU || g.act == ACT_LEAKY);
  // K = 256 from one source: keep the A tile on the SM and overlap each chunk's epilogue with the next chunk's MMAs
  // (16-byte stores: both output planes 16-byte aligned)
  if (fast && g.K1 == 256 && g.K2 == 0 && ((uintptr_t)g.out.hi & 15) == 0 && ((uintptr_t)g.out.lo() & 15) == 0)
    return tc_proj(c, g, st);
  CUtensorMap mA1h, mA1l, mA2h, mA2l, mWh, mWl;
  bool ok = make_map(&mA1h, g.a1.hi, g.M, g.K1, BM) && make_map(&mA1l, g.a1.lo(), g.M, g.K1, BM);
  if (g.K2 > 0) ok = ok && make_map(&mA2h, g.a2.hi, g.M, g.K2, BM) && make_map(&mA2l, g.a2.lo(), g.M, g.K2, BM);
  else { mA2h = mA1h; mA2l = mA1l; }
  ok = ok && make_map(&mWh, g.w.w, g.w.N, g.w.K, bn) && make_map(&mWl, g.w.w + g.w.plane_stride, g.w.N, g.w.K, bn);
  if (!ok) return false;
  TcParams p;
  fill_params(g, ln, bn, &p);
  // the vectorised fp32 epilogue, for callers that ask for it (vec_f32)
  const bool f32 = !ln && g.vec_f32 && !g.out.hi && g.out_f32 && !g.res_f32 && !g.addtab && !g.zero_lengths &&
                   g.in_group >= g.M && g.out_group == 0 && g.out_off == 0 && g.w.N % 2 == 0 && g.ldc % 2 == 0 &&
                   ((uintptr_t)g.out_f32 & 7) == 0 && (g.act == ACT_NONE || g.act == ACT_LEAKY);
  const int ntiles = p.m_tiles * p.n_tiles;
  dim3 grid(ntiles < c->sm_count ? ntiles : c->sm_count);
#define MLDB_LAUNCH(BN_, ...)                                                                                      \
  launch_pdl(k_gemm_tc<BN_, __VA_ARGS__>, grid, dim3(WS_THREADS), TileCfg<BN_>::SMEM_BYTES, st, mA1h, mA1l, mA2h, \
             mA2l, mWh, mWl, p)
#define MLDB_LAUNCH_SHAPE(...)                                                       \
  do {                                                                               \
    if (bn == 256) MLDB_LAUNCH(256, __VA_ARGS__); else MLDB_LAUNCH(128, __VA_ARGS__); \
  } while (0)
  if (ln)                             MLDB_LAUNCH(256, EPI_LN);
  else if (g.res_f32)                 MLDB_LAUNCH_SHAPE(EPI_RES);
  else if (fast && g.act == ACT_GELU) MLDB_LAUNCH_SHAPE(EPI_FAST, ACT_GELU);
  else if (fast && g.act == ACT_QUICKGELU) MLDB_LAUNCH_SHAPE(EPI_FAST, ACT_QUICKGELU);
  else if (fast && g.act == ACT_LEAKY) MLDB_LAUNCH_SHAPE(EPI_FAST, ACT_LEAKY);
  else if (f32 && g.act == ACT_LEAKY) MLDB_LAUNCH_SHAPE(EPI_F32, ACT_LEAKY);
  else if (f32)                       MLDB_LAUNCH_SHAPE(EPI_F32);
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
  // the residual is the FFN input itself (the kernel reads it from its x tile); y leaves through TMA stores
  if (l2.res.hi != g1.a1.hi || l2.res.plane_stride != g1.a1.plane_stride) return false;
  if (!planes_aligned16(g1.a1) || !planes_aligned16(l2.out)) return false;
  return true;
}
bool tc_tail_supported(const TcCtx* c, const GemmArgs& go, const LnArgs& l1, const GemmArgs& g1, const GemmArgs& g2,
                       const LnArgs& l2) {
  if (!tc_gemm_ln_supported(c, go, l1) || !tc_ffn_supported(c, g1, g2, l2)) return false;
  if (go.K1 != 256 || go.K2 > 0 || go.M != g1.M || !l1.res.hi) return false;
  // the FFN's input is LN1's output (x1, which the fused kernel keeps in shared memory)
  if (g1.a1.hi != l1.out.hi || g1.a1.plane_stride != l1.out.plane_stride) return false;
  return planes_aligned16(go.a1) && planes_aligned16(l1.res);
}

// k_ffn_tc, standalone (go == nullptr: x = g1.a1) or with the out-projection prefix (x = l1->res, att = go->a1)
static bool launch_ffn(TcCtx* c, const GemmArgs* go, const LnArgs* l1, const GemmArgs& g1, const GemmArgs& g2,
                       const LnArgs& l2, float* scratch, int* flags, cudaStream_t st) {
  CUtensorMap mXh, mXl, mW1h, mW1l, mW2h, mW2l, mAh, mAl, mWoh, mWol, mYh, mYl;
  const int M = g1.M, m_tiles = (M + BM - 1) / BM;
  const ActBuf x = go ? l1->res : g1.a1;
  bool ok = make_map(&mXh, x.hi, M, 256, BM) && make_map(&mXl, x.lo(), M, 256, BM) &&
            make_map(&mW1h, g1.w.w, g1.w.N, g1.w.K, FfnCfg::CHUNK) &&
            make_map(&mW1l, g1.w.w + g1.w.plane_stride, g1.w.N, g1.w.K, FfnCfg::CHUNK) &&
            make_map(&mW2h, g2.w.w, g2.w.N, g2.w.K, 256) &&
            make_map(&mW2l, g2.w.w + g2.w.plane_stride, g2.w.N, g2.w.K, 256) &&
            make_map(&mYh, l2.out.hi, M, 256, 64) && make_map(&mYl, l2.out.lo(), M, 256, 64);
  if (go) {
    ok = ok && make_map(&mAh, go->a1.hi, M, 256, BM) && make_map(&mAl, go->a1.lo(), M, 256, BM) &&
         make_map(&mWoh, go->w.w, go->w.N, go->w.K, 256) && make_map(&mWol, go->w.w + go->w.plane_stride, go->w.N, go->w.K, 256);
  } else {
    mAh = mXh; mAl = mXl; mWoh = mW2h; mWol = mW2l;   // not read
  }
  if (!ok) return false;
  FfnParams p{};
  p.M = M; p.m_tiles = m_tiles; p.n_chunks = g1.w.N / FfnCfg::CHUNK;
  p.tl = tc::mldb_timeline_buffer();
  p.prefix = go ? 1 : 0;
  if (go) { p.inv_s0 = go->w.inv_scale; p.b0 = go->w.bias; p.gamma1 = l1->gamma; p.beta1 = l1->beta; }
  p.inv_s1 = g1.w.inv_scale; p.inv_s2 = g2.w.inv_scale;
  p.b1 = g1.w.bias; p.b2 = g2.w.bias; p.gamma = l2.gamma; p.beta = l2.beta;
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
  p.reverse = tc::snake_order();
  launch_pdl(k_ffn_tc, dim3(ncta), dim3(MMA_THREADS), FfnCfg::SMEM_BYTES, st, mXh, mXl, mW1h, mW1l, mW2h, mW2l, mAh,
             mAl, mWoh, mWol, mYh, mYl, p);
  return true;
}
bool tc_ffn(TcCtx* c, const GemmArgs& g1, const GemmArgs& g2, const LnArgs& l2, float* scratch, int* flags, cudaStream_t st) {
  return launch_ffn(c, nullptr, nullptr, g1, g2, l2, scratch, flags, st);
}
bool tc_tail(TcCtx* c, const GemmArgs& go, const LnArgs& l1, const GemmArgs& g1, const GemmArgs& g2, const LnArgs& l2,
             float* scratch, int* flags, cudaStream_t st) {
  return launch_ffn(c, &go, &l1, g1, g2, l2, scratch, flags, st);
}
