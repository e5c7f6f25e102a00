// The ST-GCN's temporal convolution on sm_90a (k_tconv_tc): one st_gcn block's (9, 1) convolution, its residual and
// the block's final ReLU as ONE implicit GEMM, with no im2col buffer.
//
//   D[128 x C] = sum over k-blocks (tap, c0) of  X_tap[128 x 64] . W[:, tap C + c0 ..]^T       (split16, kblock_ss)
//
// The activations are split16 rows (n * T + t) * 24 + v, i.e. planes of shape [nseq][T][24][C].  A tile is 8 joints
// x 16 output frames of one sequence (128 rows, 64 per consumer warpgroup), so k_gemm_tc's two-consumer layout and
// register budget carry over unchanged.  Its A operand for tap `tap` is one TMA box of a 4-D tensor map over those
// planes: channels c0 .. c0 + 63, joints 8 vt .. 8 vt + 7, frames s t0 + tap - 4 + s i (i < 16), sequence n.  The
// box is one sequence deep, so no tile reads another sequence's frames, and the frames outside [0, T) are TMA's
// out-of-bounds zero fill: the convolution's padding.  Stride 2 is the frame dimension's traversal stride in the map
// (a 32-frame box at element stride 2 holds 16 frames).  A residual convolution (1 x 1, stride s) is a tenth K
// segment over the block input, read through its own map with the same stride; an identity residual is added in the
// epilogue.  Tile rows are frame-major inside the box (row = 8 i + joint), so the epilogue scatters each thread's two
// rows (frames i, i + 1 of one joint) to their global rows.
#include "ops.cuh"

#include <algorithm>

#include "tc_common.cuh"

namespace {
using namespace tc;

constexpr int BM = 128, BK = 64;
constexpr int NUM_THREADS = 384;                     // producer warpgroup + two consumer warpgroups (k_gemm_tc's layout)
constexpr int CONSUMER_WARPS = 8;
constexpr int JOINTS = 24, TILE_V = 8, TILE_T = 16;  // a tile: 8 joints x 16 output frames
constexpr int TAPS = 9, PAD = 4;

template <int BN>
struct TconvCfg {
  static constexpr int A_BYTES = BM * BK * 2;          // one plane of the A tile (16 KB)
  static constexpr int W_BYTES = BN * BK * 2;          // one plane of the W tile
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * W_BYTES;
  static constexpr int STAGES = BN == 256 ? 2 : (BN == 128 ? 3 : 4);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 + 1024;   // + barriers + alignment slack
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
};

struct TconvParams {
  int nseq, T_out, t_blocks;
  int kc, ktap, kblocks;             // k-blocks per tap (C / 64), of the nine taps (9 kc), in all (+ C_res / 64)
  int stride;
  float inv_scale;
  const float* bias;
  const __half* res_hi; const __half* res_lo;          // identity residual (null: none or a residual convolution)
  __half* out_hi; __half* out_lo;                      // split16 output (null: out_f32)
  float* out_f32;
};

__device__ __forceinline__ void store_split2(__half* hi, __half* lo, int64_t o, float x0, float x1) {
  uint32_t h, l;
  split2(x0, x1, h, l);
  *reinterpret_cast<uint32_t*>(hi + o) = h;
  *reinterpret_cast<uint32_t*>(lo + o) = l;
}

// Persistent: CTA c walks tiles c, c + #CTAs, ...; tile -> (sequence, 16-frame block, 8-joint group), the joint group
// fastest so that the three tiles reading the same frames run side by side.
template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
k_tconv_tc(const __grid_constant__ CUtensorMap tmXh, const __grid_constant__ CUtensorMap tmXl,
           const __grid_constant__ CUtensorMap tmRh, const __grid_constant__ CUtensorMap tmRl,
           const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const TconvParams p) {
  using Cfg = TconvCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);   // [STAGES] TMA tx
  uint64_t* bar_empty = bar_full + STAGES;                                              // [STAGES] one arrival per consumer warp

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int ntiles = p.nseq * p.t_blocks * 3;
  const int nlocal = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  auto decode = [&](int j, int& n, int& t0, int& vt) {
    const int t = (int)blockIdx.x + j * (int)gridDim.x;
    vt = t % 3;
    const int r = t / 3;
    t0 = (r % p.t_blocks) * TILE_T;
    n = r / p.t_blocks;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmXh); tma_prefetch_desc(&tmXl); tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();                  // everything below touches activations of the previous kernel

  if (warp < 4) {
    reg_dec<40>();
    if (warp != 0) return;
    // ---------------------------------------------------------------- TMA producer (one elected lane issues)
    int kbg = 0;
    for (int j = 0; j < nlocal; ++j) {
      int n, t0, vt;
      decode(j, n, t0, vt);
      const int f0 = p.stride * t0;                  // input frame of the tile's first output frame at tap 4
      for (int kb = 0; kb < p.kblocks; ++kb, ++kbg) {
        const int s = kbg % STAGES;
        mbar_wait(smem_u32(&bar_empty[s]), (((uint32_t)(kbg / STAGES)) & 1u) ^ 1u);
        if (elect_one()) {
          const uint32_t full = smem_u32(&bar_full[s]);
          mbar_expect_tx(full, Cfg::STAGE_BYTES);
          const uint32_t sAh = smem_u32(smem + s * Cfg::STAGE_BYTES), sAl = sAh + Cfg::A_BYTES;
          const uint32_t sWh = sAl + Cfg::A_BYTES, sWl = sWh + Cfg::W_BYTES;
          if (kb < p.ktap) {
            const int tap = kb / p.kc, c0 = (kb - tap * p.kc) * BK;
            tma_load_4d(sAh, &tmXh, full, c0, vt * TILE_V, f0 + tap - PAD, n);
            tma_load_4d(sAl, &tmXl, full, c0, vt * TILE_V, f0 + tap - PAD, n);
          } else {
            const int c0 = (kb - p.ktap) * BK;
            tma_load_4d(sAh, &tmRh, full, c0, vt * TILE_V, f0, n);
            tma_load_4d(sAl, &tmRl, full, c0, vt * TILE_V, f0, n);
          }
          tma_load_2d(sWh, &tmWh, full, kb * BK, 0);
          tma_load_2d(sWl, &tmWl, full, kb * BK, 0);
        }
        __syncwarp();
      }
    }
    return;
  }
  // ------------------------------------------------------------------ consumer warpgroups
  reg_inc<232>();
  const int cw = (warp >> 2) - 1;                    // which 64 rows (8 frames) of the tile
  const int cp = 2 * (lane & 3);                     // column offset inside an 8-column group
  float d[BN / 2];
  int kbg = 0;
  for (int it = 0; it < nlocal; ++it) {
    int n, t0, vt;
    decode(it, n, t0, vt);
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

    // this thread's rows: tile rows r and r + 8 = frames t and t + 1 of joint v
    const int t = t0 + cw * 8 + (warp & 3) * 2, v = vt * TILE_V + (lane >> 2);
    const float sc = p.inv_scale;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (t + h >= p.T_out) continue;
      const int64_t o = (((int64_t)n * p.T_out + t + h) * JOINTS + v) * BN + cp;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + 8 * j + cp));
        float x0 = fmaf(d[4 * j + 2 * h], sc, b.x), x1 = fmaf(d[4 * j + 2 * h + 1], sc, b.y);
        if (p.res_hi) {
          const float2 rh = __half22float2(*reinterpret_cast<const __half2*>(p.res_hi + o + 8 * j));
          const float2 rl = __half22float2(*reinterpret_cast<const __half2*>(p.res_lo + o + 8 * j));
          x0 = (x0 + rh.x) + rl.x; x1 = (x1 + rh.y) + rl.y;
        }
        x0 = x0 < 0.0f ? 0.0f : x0; x1 = x1 < 0.0f ? 0.0f : x1;      // torch.relu: a NaN stays NaN
        if (p.out_hi) store_split2(p.out_hi, p.out_lo, o + 8 * j, x0, x1);
        else *reinterpret_cast<float2*>(p.out_f32 + o + 8 * j) = make_float2(x0, x1);
      }
    }
  }
}

// A split16 plane [nseq * T * 24, C] seen as [nseq][T][24][C]: boxes of 64 channels x 8 joints x 16 frames (every
// stride-th frame) x 1 sequence.
bool frames_map(CUtensorMap* m, const __half* base, int nseq, int T, int C, int stride) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)JOINTS, (cuuint64_t)T, (cuuint64_t)nseq};
  const cuuint64_t strides[3] = {(cuuint64_t)C * sizeof(__half), (cuuint64_t)JOINTS * C * sizeof(__half),
                                 (cuuint64_t)T * JOINTS * C * sizeof(__half)};
  const cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)TILE_V, (cuuint32_t)(TILE_T * stride), 1u};
  const cuuint32_t estr[4] = {1u, 1u, (cuuint32_t)stride, 1u};
  return encode_plane_map(m, base, 4, dims, strides, box, estr);
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

bool tconv_tc_init() {
  return smem_opt_in(k_tconv_tc<64>, TconvCfg<64>::SMEM_BYTES, "k_tconv_tc<64>") &&
         smem_opt_in(k_tconv_tc<128>, TconvCfg<128>::SMEM_BYTES, "k_tconv_tc<128>") &&
         smem_opt_in(k_tconv_tc<256>, TconvCfg<256>::SMEM_BYTES, "k_tconv_tc<256>");
}

bool tconv_tc_supported(const TconvArgs& a) {
  if (a.C != 64 && a.C != 128 && a.C != 256) return false;
  if ((a.stride != 1 && a.stride != 2) || a.nseq < 1 || a.T_in < 1 || a.T_out != (a.T_in - 1) / a.stride + 1) return false;
  if (a.x.cols != a.C || !aligned16(a.x.hi) || !aligned16(a.x.lo())) return false;
  int kres = 0;
  if (a.res.hi) {
    if (a.res.cols != a.C_res || !aligned16(a.res.hi) || !aligned16(a.res.lo())) return false;
    if (a.res_conv) {
      if (a.C_res < 64 || a.C_res % 64) return false;
      kres = a.C_res;
    } else if (a.C_res != a.C || a.stride != 1) {
      return false;
    }
  }
  if (a.w.N != a.C || a.w.K != TAPS * a.C + kres || !aligned16(a.w.w) || !a.w.bias) return false;
  if (a.out.hi ? a.out.cols != a.C : !a.out_f32) return false;
  return true;
}

bool tconv_tc(const TconvArgs& a, int sm_count, cudaStream_t st) {
  CUtensorMap mXh, mXl, mRh, mRl, mWh, mWl;
  bool ok = frames_map(&mXh, a.x.hi, a.nseq, a.T_in, a.C, a.stride) &&
            frames_map(&mXl, a.x.lo(), a.nseq, a.T_in, a.C, a.stride);
  if (a.res.hi && a.res_conv)
    ok = ok && frames_map(&mRh, a.res.hi, a.nseq, a.T_in, a.C_res, a.stride) &&
         frames_map(&mRl, a.res.lo(), a.nseq, a.T_in, a.C_res, a.stride);
  else { mRh = mXh; mRl = mXl; }
  ok = ok && make_map(&mWh, a.w.w, a.w.N, a.w.K, a.C) && make_map(&mWl, a.w.w + a.w.plane_stride, a.w.N, a.w.K, a.C);
  if (!ok) return false;
  TconvParams p{};
  p.nseq = a.nseq; p.T_out = a.T_out; p.t_blocks = (a.T_out + TILE_T - 1) / TILE_T;
  p.kc = a.C / BK; p.ktap = TAPS * p.kc; p.kblocks = a.w.K / BK; p.stride = a.stride;
  p.inv_scale = a.w.inv_scale; p.bias = a.w.bias;
  if (a.res.hi && !a.res_conv) { p.res_hi = a.res.hi; p.res_lo = a.res.lo(); }
  if (a.out.hi) { p.out_hi = a.out.hi; p.out_lo = a.out.lo(); } else p.out_f32 = a.out_f32;
  const int ntiles = a.nseq * p.t_blocks * 3;
  const dim3 grid((unsigned)std::min(ntiles, std::max(sm_count, 1)));
  if (a.C == 64) launch_pdl(k_tconv_tc<64>, grid, dim3(NUM_THREADS), TconvCfg<64>::SMEM_BYTES, st, mXh, mXl, mRh, mRl, mWh, mWl, p);
  else if (a.C == 128) launch_pdl(k_tconv_tc<128>, grid, dim3(NUM_THREADS), TconvCfg<128>::SMEM_BYTES, st, mXh, mXl, mRh, mRl, mWh, mWl, p);
  else launch_pdl(k_tconv_tc<256>, grid, dim3(NUM_THREADS), TconvCfg<256>::SMEM_BYTES, st, mXh, mXl, mRh, mRl, mWh, mWl, p);
  return true;
}
