// The recurrent step of the bidirectional GRU of the T2M evaluator (t2m_motionenc.py / t2m_textenc.py) on wgmma,
// plus its CUDA-core twin, the state initialisation and the im2col of the movement encoder's strided convolutions;
// and k_gru_seq_tc, one whole layer of the action classifier's unidirectional GRU per launch (below).
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
// CTA = k_gemm_tc's (ws_cta, DESIGN §2): warp 0 streams the A (state) and W_hh k-blocks through a ring of
// 128B-swizzled stages with TMA, warpgroups 1 and 2 each own 64 rows of the 128-row tile.  Grid = (H / 32 unit
// tiles, row tiles, 2 directions), one tile per CTA; no CTA waits on another, steps are ordered by the stream.
#include <algorithm>

#include "ops.cuh"
#include "tc_common.cuh"

namespace {
using namespace tc;

constexpr int BN = 96, UNITS = 32;                           // a tile: 128 rows x 32 hidden units (96 gate columns)
using Cfg = StageLayout<BN, 4>;                              // 56 KB stages (tc_common.cuh)

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
    const float* g = a.gi + ((int64_t)m * a.L + t) * (a.dirs * 3 * H) + dir * 3 * H;
    const float* b = a.b_hh + dir * 3 * H;
    hn = gru_cell(g[u], g[H + u], g[2 * H + u], hh_r + b[u], hh_z + b[H + u], hh_n + b[2 * H + u], hp);
    if (a.seq_out.hi) {
      const int64_t so = ((int64_t)m * a.L + t) * H + u;
      __half hi, lo;
      split_f32(hn, hi, lo);
      a.seq_out.hi[so] = hi;
      a.seq_out.lo()[so] = lo;
    }
  }
  a.hf_out[o] = hn;
  __half hi, lo;
  split_f32(hn, hi, lo);
  a.h_out.hi[o] = hi;
  a.h_out.lo()[o] = lo;
}

// One tile per CTA: unit tile nt, rows m0.., direction dir; arow / wrow: its first row of A (the state of both
// directions) and of W_hh.
struct GruTile { int nt, m0, dir, arow, wrow; };
__global__ void __launch_bounds__(WS_THREADS, 1)
k_gru_step_tc(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
              const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const GruStepArgs a) {
  // one tile per CTA: nothing more goes through the ring, so its last position is not released
  ws_cta<Cfg, false>(
      tmAh, tmAl, tmWh, tmWl, nullptr, a.H / BK, [] { return 1; },
      [&](int) {
        GruTile t;
        t.nt = (int)blockIdx.x; t.m0 = (int)blockIdx.y * BM; t.dir = (int)blockIdx.z;
        t.arow = t.dir * a.rows_pad + t.m0; t.wrow = t.dir * 3 * a.H + t.nt * BN;
        return t;
      },
      [&](const GruTile& t, int kb, const auto& s, uint32_t full) {
        tma_load_2d(s.ah, &tmAh, full, kb * BK, t.arow);
        tma_load_2d(s.al, &tmAl, full, kb * BK, t.arow);
        tma_load_2d(s.wh, &tmWh, full, kb * BK, t.wrow);
        tma_load_2d(s.wl, &tmWl, full, kb * BK, t.wrow);
      },
      [&](const GruTile& t, const float (&d)[BN / 2], const TileThread& th) {
        // gate epilogue.  Every load of a row (state, gi, biases) is issued before any store, so the loads of the 8
        // (unit, row) pairs overlap instead of each waiting behind the previous pair's stores.
        const int dir = t.dir, r_lo = t.m0 + th.row();
        const int H = a.H, u0 = t.nt * UNITS + th.cp;
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
      });
}

// CUDA-core gate step (gemm=simt): gh [2 * rows_pad, 3H] fp32 in the packed column order, from k_gemm_simt
__global__ void __launch_bounds__(256) k_gru_gate_simt(const GruStepArgs a) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)a.dirs * a.rows * a.H) return;
  const int u = (int)(idx % a.H);
  const int m = (int)((idx / a.H) % a.rows);
  const int dir = (int)(idx / ((int64_t)a.H * a.rows));
  const float* g = a.gh + ((int64_t)dir * a.rows_pad + m) * (3 * a.H);
  gru_update(a, dir, m, u, g[gru_packed_col(0, u)], g[gru_packed_col(1, u)], g[gru_packed_col(2, u)]);
}

__global__ void k_gru_init(GruStepArgs a, const float* __restrict__ h0) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)a.dirs * a.rows * a.H) return;
  const int u = (int)(idx % a.H);
  const int m = (int)((idx / a.H) % a.rows);
  const int dir = (int)(idx / ((int64_t)a.H * a.rows));
  const int64_t o = ((int64_t)dir * a.rows_pad + m) * a.H + u;
  const float v = h0[dir * a.H + m * a.h0_ld + u];
  a.hf_out[o] = v;
  __half hi, lo;
  split_f32(v, hi, lo);
  a.h_out.hi[o] = hi;
  a.h_out.lo()[o] = lo;
}

// ----------------------------------------------------------------------------- one whole layer per launch
// k_gru_seq_tc: one unidirectional layer (the action classifier's nn.GRU, H = 64 or 128) over all L steps.
//  - The packed split16 W_hh of the layer (3H x H x 2 planes: 192 KB at H = 128) is loaded into shared memory by one
//    TMA burst and read from there by every step: the CTA is persistent over the sequence.
//  - Each warpgroup owns a 64-row tile for the whole sequence, so no CTA or warpgroup ever waits on another.  Two
//    warpgroups per CTA share W_hh: the grid is min(tiles, SMs) CTAs, and the second warpgroup of a CTA takes tiles
//    past the first round (it has nothing to do when the tiles fit on the SMs).
//  - The state never leaves the registers.  The packed order (gru_packed_col) puts gate r, z and n of units
//    16 kk + cp + {0, 1, 8, 9} into the thread that holds exactly those columns of k-slice kk's register A fragment,
//    so the new h is split into the next step's A operand in place.  The fp32 state (the z * h term) stays beside it.
//  - A step runs 16 units (48 gate columns, half a unit tile) at a time: gi of those units is loaded, their gate
//    columns are accumulated over all K (A_lo W_hi + A_hi W_lo + A_hi W_hi per 16-wide k-slice, as kblock_ss), and
//    the gates are applied, with the gi loads in flight under the MMAs.  The new A fragments are built at the end of
//    the step.  Half a unit tile rather than a whole one: with 96 columns the accumulators and the gi prefetch do not
//    fit beside the 64 A-fragment and 64 fp32 state registers of H = 128 (ptxas spills).
constexpr int SEQ_ROWS = 64, SEQ_WG = 2, SEQ_THREADS = 128 * SEQ_WG;
__host__ __device__ constexpr int seq_smem_bytes(int H) { return 2 * 3 * H * H * 2 + 3 * H * 4 + 64 + 1024; }
static_assert(seq_smem_bytes(128) <= 232448, "shared memory budget");

template <int H>
__global__ void __launch_bounds__(SEQ_THREADS, 1)
k_gru_seq_tc(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const GruSeqArgs a) {
  constexpr int NT = H / 32, KS = H / 16;                 // unit tiles (96 packed rows each), 16-wide k-slices
  constexpr int TILE_BYTES = 96 * 128;                     // one unit tile x one 64-wide k-block of one plane
  constexpr int PLANE_BYTES = 3 * H * H * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
  float* sb = reinterpret_cast<float*>(smem + 2 * PLANE_BYTES);          // b_hh [3H]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sb + 3 * H);
  int* smax = reinterpret_cast<int*>(bar + 1);                            // [SEQ_WG][4] per-warp max length
  const uint32_t sW = smem_u32(smem);

  if (threadIdx.x == 0) {
    mbar_init(smem_u32(bar), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
    mbar_expect_tx(smem_u32(bar), 2 * PLANE_BYTES);                      // W_hh is a weight: no need to wait for
    for (int p = 0; p < 2; ++p)                                          // the previous kernel before loading it
      for (int kb = 0; kb < H / 64; ++kb)
        for (int t = 0; t < NT; ++t)
          tma_load_2d(sW + p * PLANE_BYTES + (kb * NT + t) * TILE_BYTES, p ? &tmWl : &tmWh, smem_u32(bar), kb * 64, t * 96);
  }
  for (int i = threadIdx.x; i < 3 * H; i += SEQ_THREADS) sb[i] = __ldg(a.b_hh + i);
  __syncthreads();
  pdl_wait();                  // gi, h0 and the lengths come from (or are reused behind) earlier kernels
  mbar_wait(smem_u32(bar), 0);

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int cp = 2 * (lane & 3);
  const int ntiles = (a.rows + SEQ_ROWS - 1) / SEQ_ROWS;
  const float sc = a.w_inv_scale;
  for (int tile = blockIdx.x + wg * gridDim.x; tile < ntiles; tile += SEQ_WG * gridDim.x) {
    int len[2], row[2];
    float hf[NT][4][2][2];                                 // [unit tile][jj][row h][e]: unit 32 c + 8 jj + cp + e
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = tile * SEQ_ROWS + warp * 16 + (lane >> 2) + 8 * h;
      row[h] = m;
      int l = m < a.rows ? __ldg(a.lengths + m) : 0;
      len[h] = l < 0 ? 0 : (l > a.L ? a.L : l);
#pragma unroll
      for (int c = 0; c < NT; ++c)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const float2 v = m < a.rows ? __ldg(reinterpret_cast<const float2*>(a.h0 + (int64_t)m * H + 32 * c + 8 * jj + cp))
                                      : make_float2(0.0f, 0.0f);
          hf[c][jj][h][0] = v.x;
          hf[c][jj][h][1] = v.y;
        }
    }
    // the tile runs until its longest row is done
    int lmax = __reduce_max_sync(0xffffffffu, max(len[0], len[1]));
    if (lane == 0) smax[wg * 4 + warp] = lmax;
    named_bar_sync(1 + wg, 128);
    lmax = max(max(smax[wg * 4], smax[wg * 4 + 1]), max(smax[wg * 4 + 2], smax[wg * 4 + 3]));
    named_bar_sync(1 + wg, 128);                           // smax is reused by the next tile

    uint32_t ah[KS][4], al[KS][4];                         // A fragment of k-slice kk: units 16 kk + cp + {0,1,8,9}
#pragma unroll
    for (int kk = 0; kk < KS; ++kk)
#pragma unroll
      for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          split2(hf[kk / 2][2 * (kk % 2) + q][h][0], hf[kk / 2][2 * (kk % 2) + q][h][1], ah[kk][2 * q + h], al[kk][2 * q + h]);

    for (int s = 0; s < lmax; ++s) {
#pragma unroll
      for (int c = 0; c < NT; ++c)
#pragma unroll
        for (int half = 0; half < 2; ++half) {                    // units 32 c + 16 half .. + 15: 48 gate columns
          float2 gv[2][2][3];                                     // their gi, loaded under the MMAs
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float* gr = a.gi + ((int64_t)row[h] * a.L + s) * (3 * H) + 32 * c + 16 * half + cp;
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
              for (int g = 0; g < 3; ++g)
                gv[h][j][g] = s < len[h] ? __ldg(reinterpret_cast<const float2*>(gr + g * H + 8 * j)) : make_float2(0.0f, 0.0f);
          }
          float d[24];
          wg_fence();
#pragma unroll
          for (int kk = 0; kk < KS; ++kk) {
            const uint32_t w = sW + ((kk / 4) * NT + c) * TILE_BYTES + half * (48 * 128) + (kk % 4) * 32;
            const uint64_t wh = make_desc(w), wl = make_desc(w + PLANE_BYTES);
            wgmma_rs_n48(d, al[kk], wh, kk == 0 ? 0u : 1u);
            wgmma_rs_n48(d, ah[kk], wl, 1u);
            wgmma_rs_n48(d, ah[kk], wh, 1u);
          }
          wg_commit();
          wg_wait<0>();
          acc_fence(d);
#pragma unroll
          for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (s >= len[h]) continue;
                const int jj = 2 * half + j, u = 32 * c + 8 * jj + cp + e, k = 2 * h + e;
                const float gr = e ? gv[h][j][0].y : gv[h][j][0].x;
                const float gz = e ? gv[h][j][1].y : gv[h][j][1].x;
                const float gn = e ? gv[h][j][2].y : gv[h][j][2].x;
                hf[c][jj][h][e] = gru_cell(gr, gz, gn, d[4 * (3 * j) + k] * sc + sb[u], d[4 * (3 * j + 1) + k] * sc + sb[H + u],
                                           d[4 * (3 * j + 2) + k] * sc + sb[2 * H + u], hf[c][jj][h][e]);
              }
        }
      // the next step's A operand; a layer that feeds another writes h_s as the next input GEMM's split16 row
#pragma unroll
      for (int kk = 0; kk < KS; ++kk)
#pragma unroll
        for (int q = 0; q < 2; ++q)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            split2(hf[kk / 2][2 * (kk % 2) + q][h][0], hf[kk / 2][2 * (kk % 2) + q][h][1], ah[kk][2 * q + h], al[kk][2 * q + h]);
            if (a.seq_out.hi && s < len[h]) {
              const int64_t o = ((int64_t)row[h] * a.L + s) * H + 16 * kk + 8 * q + cp;
              *reinterpret_cast<uint32_t*>(a.seq_out.hi + o) = ah[kk][2 * q + h];
              *reinterpret_cast<uint32_t*>(a.seq_out.lo() + o) = al[kk][2 * q + h];
            }
          }
    }
    if (a.h_last) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (row[h] >= a.rows) continue;
#pragma unroll
        for (int c = 0; c < NT; ++c)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
            *reinterpret_cast<float2*>(a.h_last + (int64_t)row[h] * H + 32 * c + 8 * jj + cp) = make_float2(hf[c][jj][h][0], hf[c][jj][h][1]);
      }
    }
  }
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
  return smem_opt_in(k_gru_step_tc, Cfg::SMEM_BYTES, "k_gru_step_tc") &&
         smem_opt_in(k_gru_seq_tc<64>, seq_smem_bytes(64), "k_gru_seq_tc<64>") &&
         smem_opt_in(k_gru_seq_tc<128>, seq_smem_bytes(128), "k_gru_seq_tc<128>");
}

bool gru_shape_supported(int H) { return H >= 64 && H <= 1024 && H % 64 == 0; }

bool gru_step_tc(const GruStepArgs& a, cudaStream_t st) {
  CUtensorMap mAh, mAl, mWh, mWl;
  const bool ok = make_map(&mAh, a.h_in.hi, 2 * a.rows_pad, a.H, BM) && make_map(&mAl, a.h_in.lo(), 2 * a.rows_pad, a.H, BM) &&
                  make_map(&mWh, a.w_hh, 6 * a.H, a.H, BN) && make_map(&mWl, a.w_hh + a.w_plane_stride, 6 * a.H, a.H, BN);
  if (!ok) return false;
  const dim3 grid((unsigned)(a.H / UNITS), (unsigned)((a.rows + BM - 1) / BM), 2);
  launch_pdl(k_gru_step_tc, grid, dim3(WS_THREADS), Cfg::SMEM_BYTES, st, mAh, mAl, mWh, mWl, a);
  return true;
}

bool gru_seq_supported(int H) { return H == 64 || H == 128; }

bool gru_seq_tc(const GruSeqArgs& a, int sm_count, cudaStream_t st) {
  CUtensorMap mWh, mWl;
  if (!make_map(&mWh, a.w_hh, 3 * a.H, a.H, 96) || !make_map(&mWl, a.w_hh + a.w_plane_stride, 3 * a.H, a.H, 96))
    return false;
  const int ntiles = (a.rows + SEQ_ROWS - 1) / SEQ_ROWS;
  const dim3 grid((unsigned)std::min(ntiles, std::max(sm_count, 1)));
  if (a.H == 64) launch_pdl(k_gru_seq_tc<64>, grid, dim3(SEQ_THREADS), seq_smem_bytes(64), st, mWh, mWl, a);
  else launch_pdl(k_gru_seq_tc<128>, grid, dim3(SEQ_THREADS), seq_smem_bytes(128), st, mWh, mWl, a);
  return true;
}

void gru_gate_simt(const GruStepArgs& a, cudaStream_t st) {
  const int64_t n = (int64_t)a.dirs * a.rows * a.H;
  k_gru_gate_simt<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a);
}

void gru_init_state(const GruStepArgs& a, const float* h0, cudaStream_t st) {
  const int64_t n = (int64_t)a.dirs * a.rows * a.H;
  k_gru_init<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, h0);
}

void im2col_k4s2(ActBuf X, const float* src, int64_t ld, int T_in, int C, int Cp, int T_out, int rows, cudaStream_t st) {
  const int64_t n = (int64_t)rows * 4 * Cp;
  k_im2col_k4s2<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(X, src, ld, T_in, C, Cp, T_out, rows);
}
