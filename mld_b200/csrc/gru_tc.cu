// The recurrent step of the bidirectional GRU of the T2M evaluator (t2m_motionenc.py / t2m_textenc.py) on wgmma,
// plus its CUDA-core twin, the state initialisation and the im2col of the movement encoder's strided convolutions.
//
// One launch of k_gru_step_tc advances every sequence of a batch chunk by one step in BOTH directions:
//   gh[dir] = h_{s-1}[dir] . W_hh[dir]^T        (split16 A and B, three f16 MMAs per k-step, fp32 accumulation)
// followed by the gate epilogue (torch.nn.GRU, gate rows r | z | n):
//   r = sigmoid(gi_r + gh_r + b_hr), z = sigmoid(gi_z + gh_z + b_hz), n = tanh(gi_n + r * (gh_n + b_hn)),
//   h_s = (1 - z) * n + z * h_{s-1}
// where gi = x_t W_ih^T + b_ih was computed for every step beforehand by one GEMM per direction.  The forward
// direction reads step t = s, the backward direction t = len - 1 - s, so each sequence's backward pass starts at its
// own last valid step (pack_padded_sequence).  Rows with s >= len copy their state through unchanged, so after the
// last step the output buffer holds every row's final state.  Nothing is read at t >= len.
//
// W_hh of both directions is one [2 * 3H, H] operand whose rows are interleaved per 32-unit tile: inside a tile of
// 96 rows, 8-row group j = 3 * jj + g holds gate g of units 8 * jj .. 8 * jj + 7.  The accumulator fragment of a
// thread holds columns 8 j + cp, 8 j + cp + 1 of every group j, so the r, z and n pre-activations of its units land
// in its own registers and the epilogue needs no shuffle or shared memory.
//
// CTA = three warpgroups as in k_gemm_tc (gemm_tc.cu): warp 0 streams the A (state) and W_hh k-blocks through a
// ring of 128B-swizzled stages with TMA, warpgroups 1 and 2 each own 64 rows of the 128-row tile.  Grid =
// (H / 32 unit tiles, row tiles, 2 directions); no CTA waits on another, steps are ordered by the stream.
#include "ops.cuh"
#include "tc_common.cuh"

namespace {
using namespace tc;

constexpr int BM = 128, BK = 64, BN = 96, UNITS = 32;        // a tile: 128 rows x 32 hidden units (96 gate columns)
constexpr int NUM_THREADS = 384, CONSUMER_WARPS = 8;
constexpr int A_BYTES = BM * BK * 2, W_BYTES = BN * BK * 2;  // one plane: 16 KB / 12 KB
constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * W_BYTES;       // 56 KB
constexpr int STAGES = 4;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 + 1024;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");

// accurate expf / tanhf (not the fast intrinsics): the recurrence compounds their error over up to 49 steps
__device__ __forceinline__ float gru_cell(float gr, float gz, float gn, float hr, float hz, float hn, float h) {
  const float r = 1.0f / (1.0f + expf(-(gr + hr)));
  const float z = 1.0f / (1.0f + expf(-(gz + hz)));
  const float n = tanhf(gn + r * hn);
  return (1.0f - z) * n + z * h;
}

// one (row, direction, unit) of the step: hh_* = the three h W_hh^T columns of the unit, already scaled
__device__ __forceinline__ void gru_update(const GruStepArgs& a, int dir, int m, int u, float hh_r, float hh_z, float hh_n) {
  const int H = a.H;
  const int64_t o = ((int64_t)dir * a.rows_pad + m) * H + u;
  const float hp = a.hf_in[o];
  int len = a.lengths[m];
  len = len < 0 ? 0 : (len > a.L ? a.L : len);
  float hn = hp;
  if (a.step < len) {
    const int t = dir ? len - 1 - a.step : a.step;
    const float* g = a.gi + ((int64_t)m * a.L + t) * (6 * H) + dir * 3 * H;
    const float* b = a.b_hh + dir * 3 * H;
    hn = gru_cell(g[u], g[H + u], g[2 * H + u], hh_r + b[u], hh_z + b[H + u], hh_n + b[2 * H + u], hp);
  }
  a.hf_out[o] = hn;
  __half hi, lo;
  split_f32(hn, hi, lo);
  a.h_out.hi[o] = hi;
  a.h_out.lo()[o] = lo;
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
k_gru_step_tc(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
              const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const GruStepArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* bar_empty = bar_full + STAGES;
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int nt = (int)blockIdx.x, m0 = (int)blockIdx.y * BM, dir = (int)blockIdx.z;
  const int kblocks = a.H / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_empty[s]), CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmAh); tma_prefetch_desc(&tmAl); tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();                  // the previous step's state (and gi) are complete

  if (warp < 4) {
    reg_dec<40>();
    if (warp != 0) return;
    const int arow = dir * a.rows_pad + m0, wrow = dir * 3 * a.H + nt * BN;
    for (int kb = 0; kb < kblocks; ++kb) {
      const int s = kb % STAGES;
      mbar_wait(smem_u32(&bar_empty[s]), (((uint32_t)(kb / STAGES)) & 1u) ^ 1u);
      if (elect_one()) {
        const uint32_t full = smem_u32(&bar_full[s]);
        mbar_expect_tx(full, STAGE_BYTES);
        const uint32_t sAh = smem_u32(smem + s * STAGE_BYTES), sAl = sAh + A_BYTES;
        const uint32_t sWh = sAl + A_BYTES, sWl = sWh + W_BYTES;
        tma_load_2d(sAh, &tmAh, full, kb * BK, arow);
        tma_load_2d(sAl, &tmAl, full, kb * BK, arow);
        tma_load_2d(sWh, &tmWh, full, kb * BK, wrow);
        tma_load_2d(sWl, &tmWl, full, kb * BK, wrow);
      }
      __syncwarp();
    }
    return;
  }
  reg_inc<232>();
  const int cw = (warp >> 2) - 1;
  const int cp = 2 * (lane & 3);
  float d[BN / 2];
  for (int kb = 0; kb < kblocks; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(smem_u32(&bar_full[s]), ((uint32_t)(kb / STAGES)) & 1u);
    const uint32_t base = smem_u32(smem + s * STAGE_BYTES);
    wg_fence();
    kblock_ss<BN>(d, base + cw * (64 * 128), base + A_BYTES + cw * (64 * 128), base + 2 * A_BYTES,
                  base + 2 * A_BYTES + W_BYTES, kb == 0);
    wg_commit();
    if (kb > 0) {
      wg_wait<1>();
      if (lane == 0) mbar_arrive(smem_u32(&bar_empty[(kb - 1) % STAGES]));
    }
  }
  wg_wait<0>();
  acc_fence(d);

  // gate epilogue.  Every load of a row (state, gi, biases) is issued before any store, so the loads of the 8
  // (unit, row) pairs overlap instead of each waiting behind the previous pair's stores.
  const int r_lo = m0 + cw * 64 + (warp & 3) * 16 + (lane >> 2);
  const int H = a.H, u0 = nt * UNITS + cp;
  const float sc = a.w_inv_scale;
  float bh[4][2][3];
#pragma unroll
  for (int jj = 0; jj < 4; ++jj)
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
      for (int g = 0; g < 3; ++g) bh[jj][e][g] = __ldg(a.b_hh + dir * 3 * H + g * H + u0 + 8 * jj + e);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = r_lo + 8 * h;
    if (m >= a.rows) continue;
    int len = __ldg(a.lengths + m);
    len = len < 0 ? 0 : (len > a.L ? a.L : len);
    const bool live = a.step < len;
    const int64_t so = ((int64_t)dir * a.rows_pad + m) * H + u0;
    const float* gi = a.gi + ((int64_t)m * a.L + (dir ? len - 1 - a.step : a.step)) * (6 * H) + dir * 3 * H + u0;
    float hp[4][2], gv[4][2][3];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        hp[jj][e] = __ldg(a.hf_in + so + 8 * jj + e);
#pragma unroll
        for (int g = 0; g < 3; ++g) gv[jj][e][g] = live ? __ldg(gi + g * H + 8 * jj + e) : 0.0f;
      }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = 2 * h + e;
        const float hn = live ? gru_cell(gv[jj][e][0], gv[jj][e][1], gv[jj][e][2], d[4 * (3 * jj) + c] * sc + bh[jj][e][0],
                                         d[4 * (3 * jj + 1) + c] * sc + bh[jj][e][1], d[4 * (3 * jj + 2) + c] * sc + bh[jj][e][2],
                                         hp[jj][e])
                              : hp[jj][e];
        const int64_t o = so + 8 * jj + e;
        a.hf_out[o] = hn;
        __half hi, lo;
        split_f32(hn, hi, lo);
        a.h_out.hi[o] = hi;
        a.h_out.lo()[o] = lo;
      }
  }
}

// CUDA-core gate step (gemm=simt): gh [2 * rows_pad, 3H] fp32 in the packed column order, from k_gemm_simt
__global__ void __launch_bounds__(256) k_gru_gate_simt(const GruStepArgs a) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)2 * a.rows * a.H) return;
  const int u = (int)(idx % a.H);
  const int m = (int)((idx / a.H) % a.rows);
  const int dir = (int)(idx / ((int64_t)a.H * a.rows));
  const float* g = a.gh + ((int64_t)dir * a.rows_pad + m) * (3 * a.H);
  gru_update(a, dir, m, u, g[gru_packed_col(0, u)], g[gru_packed_col(1, u)], g[gru_packed_col(2, u)]);
}

__global__ void k_gru_init(GruStepArgs a, const float* __restrict__ h0) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)2 * a.rows * a.H) return;
  const int u = (int)(idx % a.H);
  const int m = (int)((idx / a.H) % a.rows);
  const int dir = (int)(idx / ((int64_t)a.H * a.rows));
  const int64_t o = ((int64_t)dir * a.rows_pad + m) * a.H + u;
  const float v = h0[dir * a.H + u];
  a.hf_out[o] = v;
  __half hi, lo;
  split_f32(v, hi, lo);
  a.h_out.hi[o] = hi;
  a.h_out.lo()[o] = lo;
}

// out[b * T_out + t, k * Cp + c] = src[(b * T_in + 2t + k - 1) * ld + c] for c < C and 0 <= 2t + k - 1 < T_in, else 0
// (Conv1d(k = 4, stride 2, padding 1) as a GEMM; split16 output, K = 4 * Cp)
__global__ void k_im2col_k4s2(ActBuf X, const float* __restrict__ src, int64_t ld, int T_in, int C, int Cp, int T_out,
                              int rows) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int K = 4 * Cp;
  if (idx >= (int64_t)rows * K) return;
  const int col = (int)(idx % K);
  const int r = (int)(idx / K);
  const int k = col / Cp, c = col - k * Cp;
  const int b = r / T_out, t = r - b * T_out;
  const int ti = 2 * t + k - 1;
  const float v = (c < C && ti >= 0 && ti < T_in) ? src[((int64_t)b * T_in + ti) * ld + c] : 0.0f;
  __half hi, lo;
  split_f32(v, hi, lo);
  X.hi[idx] = hi;
  X.lo()[idx] = lo;
}

}  // namespace

bool gru_tc_init() {
  return smem_opt_in(k_gru_step_tc, SMEM_BYTES, "k_gru_step_tc");
}

bool gru_shape_supported(int H) { return H >= 64 && H <= 1024 && H % 64 == 0; }

bool gru_step_tc(const GruStepArgs& a, cudaStream_t st) {
  CUtensorMap mAh, mAl, mWh, mWl;
  const bool ok = make_map(&mAh, a.h_in.hi, 2 * a.rows_pad, a.H, BM) && make_map(&mAl, a.h_in.lo(), 2 * a.rows_pad, a.H, BM) &&
                  make_map(&mWh, a.w_hh, 6 * a.H, a.H, BN) && make_map(&mWl, a.w_hh + a.w_plane_stride, 6 * a.H, a.H, BN);
  if (!ok) return false;
  const dim3 grid((unsigned)(a.H / UNITS), (unsigned)((a.rows + BM - 1) / BM), 2);
  launch_pdl(k_gru_step_tc, grid, dim3(NUM_THREADS), SMEM_BYTES, st, mAh, mAl, mWh, mWl, a);
  return true;
}

void gru_gate_simt(const GruStepArgs& a, cudaStream_t st) {
  const int64_t n = (int64_t)2 * a.rows * a.H;
  k_gru_gate_simt<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a);
}

void gru_init_state(const GruStepArgs& a, const float* h0, cudaStream_t st) {
  const int64_t n = (int64_t)2 * a.rows * a.H;
  k_gru_init<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, h0);
}

void im2col_k4s2(ActBuf X, const float* src, int64_t ld, int T_in, int C, int Cp, int T_out, int rows, cudaStream_t st) {
  const int64_t n = (int64_t)rows * 4 * Cp;
  k_im2col_k4s2<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(X, src, ld, T_in, C, Cp, T_out, rows);
}
