// The SMPL layer of the action model's evaluation (Rotation2xyz with SMPL, mld/transforms/rotation2xyz.py): rot6d
// features to the 24 SMPL joints ('smpl') or to the skinned mesh ('vertices'), with zero betas, as smplx 0.1.28's
// SMPLLayer -> lbs(..., pose2rot=False) computes them.
//
//   k_smpl_fk   (CUDA cores, one warp per frame): rot6d -> R_j (Gram-Schmidt), the kinematic chain along `parents`
//               from the rest joints J (J_regressor v_template, in double at load).  'smpl' writes the joints with
//               the root and translation handling straight into [B, 24, 3, T].  'vertices' writes each frame's
//               relative transforms A_j (24 x 3 x 4) plus (valid, translation offset), and its pose feature
//               (R_1..23 - I, 207 values, zero padded to 256) as a split16 A-operand row.  A masked-out frame's
//               features are never read: it gets identity transforms and a zero feature row.
//   k_smpl_lbs  (wgmma + CUDA cores, one launch): the pose-blend GEMM [frames x 256] . [256 x 3 V'] in split16 with
//               skinning fused into the epilogue, so v_posed and T_v never reach global memory.
//
// LBS tile: 64 frames (one consumer warpgroup) x 96 columns = 32 vertices in coordinate-planar order (column
// c * 32 + i of vertex tile n is coordinate c of vertex 32 n + i), so a thread's accumulator holds x, y and z of the
// same 8 vertices for its 2 frames.  The CTA keeps its 64 frames' features (64 KB) and transforms (73 KB) in shared
// memory and streams the packed posedirs tiles of its range of vertex tiles through a 2-stage TMA ring fed by one
// producer warp.  Skinning per (frame, vertex): T_v = sum_j w[v, j] A_j over the joints that weigh on some vertex of
// the tile (a per-tile mask built at load; a tile with one dense row runs all 24), in joint order, then
// T_v[:, :3] v_posed + T_v[:, 3].  The result is staged in shared memory and stored along t, the innermost
// dimension of [B, V, 3, T].
#include "engine.h"

#include <math.h>
#include <string.h>

#include <algorithm>

#include "tc_common.cuh"

static const char* const kSmpl = "smpl.";
static constexpr int kJ = 24, kFeat = 150, kPoseK = 207, kPoseKpad = 256;
static constexpr int kXf = kJ * 12 + 4;             // per-frame floats: A_j rows (3 x 4 each), valid, translation offset

namespace {
using namespace tc;

// ---------------------------------------------------------------------------------------------------- FK
struct FkParams {
  const float* feats;          // [frames, 150]
  const uint8_t* mask;         // [frames] or null (every frame)
  int frames, T, vertstrans;
  float* joints;               // 'smpl': [nseq, 24, 3, T] (null: the vertex path)
  float* xf;                   // 'vertices': [frames][kXf]
  ActBuf feat;                 // 'vertices': split16 [frames, 256]
  float J[kJ * 3];             // rest joints
  int parents[kJ];
};

__global__ void __launch_bounds__(128) k_smpl_fk(const FkParams p) {
  __shared__ float sJ[kJ * 3];
  __shared__ int sPar[kJ];
  __shared__ float sLoc[4][kJ][12], sWld[4][kJ][12];
  for (int i = threadIdx.x; i < kJ * 3; i += blockDim.x) sJ[i] = p.J[i];
  if (threadIdx.x < kJ) sPar[threadIdx.x] = p.parents[threadIdx.x];
  __syncthreads();
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float (*L)[12] = sLoc[w];
  float (*W)[12] = sWld[w];
  for (int f = blockIdx.x * 4 + w; f < p.frames; f += gridDim.x * 4) {
    const int b = f / p.T, t = f - b * p.T;
    const bool valid = !p.mask || p.mask[f] != 0;
    const float* x = p.feats + (int64_t)f * kFeat;
    if (lane < kJ) {
      const int j = lane;
      float R[9] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f};
      if (valid) {                                   // rotation_6d_to_matrix, F.normalize's max(norm, 1e-12)
        const float a0 = x[j], a1 = x[25 + j], a2 = x[50 + j];
        const float c0 = x[75 + j], c1 = x[100 + j], c2 = x[125 + j];
        const float n1 = fmaxf(sqrtf(a0 * a0 + a1 * a1 + a2 * a2), 1e-12f);
        const float b0 = a0 / n1, b1 = a1 / n1, b2 = a2 / n1;
        const float d = b0 * c0 + b1 * c1 + b2 * c2;
        float e0 = c0 - d * b0, e1 = c1 - d * b1, e2 = c2 - d * b2;
        const float n2 = fmaxf(sqrtf(e0 * e0 + e1 * e1 + e2 * e2), 1e-12f);
        e0 /= n2; e1 /= n2; e2 /= n2;
        R[0] = b0; R[1] = b1; R[2] = b2;
        R[3] = e0; R[4] = e1; R[5] = e2;
        R[6] = b1 * e2 - b2 * e1; R[7] = b2 * e0 - b0 * e2; R[8] = b0 * e1 - b1 * e0;
      }
      const int pj = sPar[j];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        L[j][r * 4 + 0] = R[r * 3 + 0]; L[j][r * 4 + 1] = R[r * 3 + 1]; L[j][r * 4 + 2] = R[r * 3 + 2];
        L[j][r * 4 + 3] = j ? sJ[j * 3 + r] - sJ[pj * 3 + r] : sJ[r];
      }
      if (p.feat.hi && j > 0) {                      // pose feature (R_j - I).flatten(), columns 9 (j - 1) ..
        const int64_t o = (int64_t)f * kPoseKpad + 9 * (j - 1);
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          __half hi, lo;
          split_f32(R[k] - ((k % 4) == 0 ? 1.0f : 0.0f), hi, lo);
          p.feat.hi[o + k] = hi;
          p.feat.lo()[o + k] = lo;
        }
      }
    } else if (p.feat.hi) {                          // lanes 24..31: the K padding 207 .. 255
      for (int k = kPoseK + lane - kJ; k < kPoseKpad; k += 32 - kJ) {
        const int64_t o = (int64_t)f * kPoseKpad + k;
        p.feat.hi[o] = __float2half_rn(0.0f);
        p.feat.lo()[o] = __float2half_rn(0.0f);
      }
    }
    __syncwarp();
    // the chain: world_i = world_parent(i) . local_i (3 x 4, implicit last row 0 0 0 1), one entry per lane
    const int r = lane >> 2, c = lane & 3;
    if (lane < 12) W[0][lane] = L[0][lane];
    __syncwarp();
    for (int i = 1; i < kJ; ++i) {
      if (lane < 12) {
        const float* P = W[sPar[i]];
        float v = P[r * 4 + 0] * L[i][c] + P[r * 4 + 1] * L[i][4 + c] + P[r * 4 + 2] * L[i][8 + c];
        if (c == 3) v += P[r * 4 + 3];
        W[i][lane] = v;
      }
      __syncwarp();
    }
    // translation: trans[t] - trans[0] of this sequence, on every frame (masked or not), as Rotation2xyz adds it
    float toff[3] = {0.f, 0.f, 0.f};
    if (p.vertstrans) {
      const float* x0 = p.feats + (int64_t)b * p.T * kFeat;
#pragma unroll
      for (int k = 0; k < 3; ++k) toff[k] = x[k * 25 + 24] - x0[k * 25 + 24];
    }
    if (p.joints) {
      if (lane < kJ) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float v = valid ? W[lane][k * 4 + 3] - W[0][k * 4 + 3] : 0.0f;
          p.joints[(((int64_t)b * kJ + lane) * 3 + k) * p.T + t] = v + toff[k];
        }
      }
    } else {
      float* xf = p.xf + (int64_t)f * kXf;
      if (lane < kJ) {                               // A_j = [R | t - R J_j]
        const float* G = W[lane];
        const float* Jj = sJ + lane * 3;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          xf[lane * 12 + k * 4 + 0] = G[k * 4 + 0];
          xf[lane * 12 + k * 4 + 1] = G[k * 4 + 1];
          xf[lane * 12 + k * 4 + 2] = G[k * 4 + 2];
          xf[lane * 12 + k * 4 + 3] = G[k * 4 + 3] - (G[k * 4 + 0] * Jj[0] + G[k * 4 + 1] * Jj[1] + G[k * 4 + 2] * Jj[2]);
        }
      } else if (lane == kJ) {
        xf[kJ * 12 + 0] = valid ? 1.0f : 0.0f;
        xf[kJ * 12 + 1] = toff[0]; xf[kJ * 12 + 2] = toff[1]; xf[kJ * 12 + 3] = toff[2];
      }
    }
    __syncwarp();                                    // L / W are rewritten by the next frame
  }
}

// ---------------------------------------------------------------------------------------------------- LBS
constexpr int LBS_BM = 64, BN = 96, VT = 32, BK = 64, KB = kPoseKpad / BK, STAGES = 2;
constexpr int LBS_THREADS = 160;                      // one consumer warpgroup + one TMA producer warp
constexpr int OUT_LD = 68;                            // staging row (frames) stride: conflict-free epilogue writes
constexpr int A_PLANE = LBS_BM * BK * 2, A_BYTES = KB * 2 * A_PLANE;      // 8 KB, 64 KB
constexpr int W_PLANE = BN * BK * 2, W_STAGE = 2 * W_PLANE;                // 12 KB, 24 KB
constexpr int OFF_W = A_BYTES, OFF_X = OFF_W + STAGES * W_STAGE;
constexpr int OFF_O = OFF_X + LBS_BM * kXf * 4, OFF_LW = OFF_O + BN * OUT_LD * 4;
constexpr int OFF_BAR = OFF_LW + kJ * VT * 4;
constexpr int LBS_SMEM = OFF_BAR + 64 + 1024;
static_assert(LBS_SMEM <= 232448, "shared memory budget");
static_assert(OFF_W % 1024 == 0 && W_STAGE % 1024 == 0 && OFF_X % 16 == 0 && OFF_BAR % 8 == 0, "alignment");

struct LbsParams {
  int frames, T, V, vtiles_per_cta, vtiles;
  float inv_scale;
  const float* xf;             // [frames][kXf]
  const float* vt;             // [vtiles * 32][3] v_template, zero past V
  const float* lbsw;           // [vtiles][24][32] skinning weights, zero past V
  const uint32_t* jmask;       // [vtiles] joints with a non-zero weight in the tile
  float* out;                  // [nseq, V, 3, T]
};

__global__ void __launch_bounds__(LBS_THREADS, 1)
k_smpl_lbs(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
           const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, const LbsParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
  float* sX = reinterpret_cast<float*>(smem + OFF_X);
  float* sO = reinterpret_cast<float*>(smem + OFF_O);
  float* sLw = reinterpret_cast<float*>(smem + OFF_LW);
  uint64_t* bar_a = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  // the W stream.  Its loops stay written out: through ring_feed / ring_mma nvcc folds the stage addresses
  // differently and the kernel's code changes
  const Ring<STAGES> ring{bar_a + 1, bar_a + 1 + STAGES};

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int nsplit = (p.vtiles + p.vtiles_per_cta - 1) / p.vtiles_per_cta;
  const int mt = blockIdx.x / nsplit, n0 = (blockIdx.x % nsplit) * p.vtiles_per_cta;
  const int n1 = min(p.vtiles, n0 + p.vtiles_per_cta);
  const int m0 = mt * LBS_BM;

  if (threadIdx.x == 0) {
    mbar_init(smem_u32(bar_a), 1);
    ring.init(4);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 4) {
    // ---------------------------------------------------------------- TMA producer
    if (elect_one()) {
      const uint32_t ba = smem_u32(bar_a);
      mbar_expect_tx(ba, A_BYTES);
      for (int kb = 0; kb < KB; ++kb) {
        const uint32_t s = smem_u32(smem + kb * 2 * A_PLANE);
        tma_load_2d(s, &tmAh, ba, kb * BK, m0);
        tma_load_2d(s + A_PLANE, &tmAl, ba, kb * BK, m0);
      }
    }
    __syncwarp();
    int kbg = 0;
    for (int nt = n0; nt < n1; ++nt)
      for (int kb = 0; kb < KB; ++kb, ++kbg) {
        const int s = kbg % STAGES;
        ring.wait_empty(kbg);
        if (elect_one()) {
          const uint32_t full = ring.full_bar(kbg);
          const uint32_t sw = smem_u32(smem + OFF_W + s * W_STAGE);
          mbar_expect_tx(full, W_STAGE);
          tma_load_2d(sw, &tmWh, full, kb * BK, nt * BN);
          tma_load_2d(sw + W_PLANE, &tmWl, full, kb * BK, nt * BN);
        }
        __syncwarp();
      }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroup
  const int tid = threadIdx.x;
  // this CTA's frames' transforms (rows past the last frame: zero, never stored)
  for (int i = tid; i < LBS_BM * (kXf / 4); i += 128) {
    const int r = i / (kXf / 4), q = i - r * (kXf / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m0 + r < p.frames) v = __ldg(reinterpret_cast<const float4*>(p.xf + (int64_t)(m0 + r) * kXf) + q);
    reinterpret_cast<float4*>(sX)[i] = v;
  }
  mbar_wait(smem_u32(bar_a), 0);

  const int q = lane & 3;
  const int r0 = 16 * warp + (lane >> 2);              // this thread's frames: tile rows r0 and r0 + 8
  float d[BN / 2];
  int kbg = 0;
  for (int nt = n0; nt < n1; ++nt) {
    for (int kb = 0; kb < KB; ++kb, ++kbg) {
      const int s = kbg % STAGES;
      ring.wait_full(kbg);
      const uint32_t sAh = smem_u32(smem + kb * 2 * A_PLANE), sWh = smem_u32(smem + OFF_W + s * W_STAGE);
      wg_fence();
      kblock_ss<BN>(d, sAh, sAh + A_PLANE, sWh, sWh + W_PLANE, kb == 0);
      wg_commit();
      if (kb > 0) {                                   // the previous k-block's MMAs have retired: free its stage
        wg_wait<1>();
        if (lane == 0) ring.release(kbg - 1);
      }
    }
    wg_wait<0>();
    acc_fence(d);
    if (lane == 0) ring.release(kbg - 1);

    for (int i = tid; i < kJ * VT; i += 128) sLw[i] = __ldg(p.lbsw + (int64_t)nt * kJ * VT + i);
    named_bar_sync(1, 128);                           // sLw and sX ready; the previous tile's staging is stored
    // v_posed = v_template + pose offsets, in place: column group 4 c + jj holds coordinate c of vertices 8 jj ..
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int v = nt * VT + 8 * jj + 2 * q + e;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float t0 = __ldg(p.vt + (int64_t)v * 3 + c);
          float& lo = d[4 * (4 * c + jj) + e];
          float& hi = d[4 * (4 * c + jj) + 2 + e];
          lo = fmaf(lo, p.inv_scale, t0);
          hi = fmaf(hi, p.inv_scale, t0);
        }
      }
    const uint32_t jm = __ldg(p.jmask + nt);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + 8 * h;
      const float* X = sX + r * kXf;
#pragma unroll
      for (int half = 0; half < 2; ++half) {          // vertices 8 jj + 2 q + e for jj in {2 half, 2 half + 1}
        float acc[4][12];
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int k = 0; k < 12; ++k) acc[u][k] = 0.0f;
        for (uint32_t m = jm; m; m &= m - 1) {
          const int j = __ffs(m) - 1;
          const float4* Aj = reinterpret_cast<const float4*>(X + j * 12);
          const float4 a0 = Aj[0], a1 = Aj[1], a2 = Aj[2];
          const float a[12] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w};
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int vl = 8 * (2 * half + (u >> 1)) + 2 * q + (u & 1);
            const float wv = sLw[j * VT + vl];
#pragma unroll
            for (int k = 0; k < 12; ++k) acc[u][k] = fmaf(wv, a[k], acc[u][k]);
          }
        }
        const float valid = X[kJ * 12];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int jj = 2 * half + (u >> 1), e = u & 1, vl = 8 * jj + 2 * q + e;
          const float px = d[4 * (0 + jj) + 2 * h + e], py = d[4 * (4 + jj) + 2 * h + e], pz = d[4 * (8 + jj) + 2 * h + e];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const float* T4 = acc[u] + 4 * c;
            const float v = fmaf(T4[0], px, fmaf(T4[1], py, fmaf(T4[2], pz, T4[3])));
            sO[(c * VT + vl) * OUT_LD + r] = (valid != 0.0f ? v : 0.0f) + X[kJ * 12 + 1 + c];
          }
        }
      }
    }
    named_bar_sync(1, 128);                           // the tile is staged
    // store along t: consecutive threads take consecutive frames of one (vertex, coordinate)
    for (int i = tid; i < BN * LBS_BM; i += 128) {
      const int col = i / LBS_BM, r = i - col * LBS_BM;
      const int row = m0 + r, c = col / VT, v = nt * VT + (col - c * VT);
      if (row >= p.frames || v >= p.V) continue;
      const int b = row / p.T, t = row - b * p.T;
      p.out[(((int64_t)b * p.V + v) * 3 + c) * p.T + t] = sO[col * OUT_LD + r];
    }
  }
}

}  // namespace

bool smpl_tc_init() { return smem_opt_in(k_smpl_lbs, LBS_SMEM, "k_smpl_lbs"); }

// ---------------------------------------------------------------------------------------------------- engine
extern "C" void mldb_default_smpl_config(mldb_smpl_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = MLDB_SMPL_ABI_VERSION;
  c->num_vertices = 6890;
}

extern "C" int mldb_smpl_configure(mldb_handle* h, const mldb_smpl_config* cfg) {
  if (!h || !cfg) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(may_configure(h, cfg->abi_version, MLDB_SMPL_ABI_VERSION, h->smpl.on, "smpl", "the SMPL layer"));
  const int V = cfg->num_vertices;
  if (V < 1 || V > (1 << 20)) FAIL(MLDB_ERR_INVALID, "num_vertices must be in [1, 2^20], got %d", V);
  const std::string p = kSmpl;
  spec_add(h, p + "v_template", {V, 3});
  spec_add(h, p + "posedirs", {kPoseK, 3 * (int64_t)V});
  spec_add(h, p + "J_regressor", {kJ, V});
  spec_add(h, p + "lbs_weights", {V, kJ});
  spec_add(h, p + "parents", {kJ});
  h->smpl.cfg = *cfg;
  h->smpl.on = true;
  return MLDB_OK;
}

int pack_smpl(mldb_handle* h) {
  SmplW& s = h->smpl;
  const int V = s.cfg.num_vertices, nt = (V + VT - 1) / VT, Vp = nt * VT;
  const std::string p = kSmpl;
  const float* par = rt(h, p + "parents").host.data();
  for (int j = 0; j < kJ; ++j) {
    const int pj = (int)par[j];
    if ((float)pj != par[j] || (j == 0 ? pj != -1 : (pj < 0 || pj >= j)))
      FAIL(MLDB_ERR_INVALID, "key '%sparents': parents[0] must be -1 and 0 <= parents[j] < j (topological order), "
           "got parents[%d] = %g", kSmpl, j, (double)par[j]);
    s.parents[j] = pj;
  }
  const float* vt = rt(h, p + "v_template").host.data();
  const float* jr = rt(h, p + "J_regressor").host.data();
  for (int j = 0; j < kJ; ++j)                       // J = J_regressor v_template, in double
    for (int c = 0; c < 3; ++c) {
      double acc = 0.0;
      for (int v = 0; v < V; ++v) acc += (double)jr[(size_t)j * V + v] * (double)vt[(size_t)v * 3 + c];
      s.J[j * 3 + c] = (float)acc;
    }
  // posedirs [207, 3 V] -> W [3 Vp, 207] with vertex tile n's columns coordinate-planar
  const float* pd = rt(h, p + "posedirs").host.data();
  std::vector<float> W((size_t)3 * Vp * kPoseK, 0.0f);
  for (int v = 0; v < V; ++v)
    for (int c = 0; c < 3; ++c) {
      const size_t n = (size_t)(v / VT) * BN + c * VT + v % VT;
      for (int k = 0; k < kPoseK; ++k) W[n * kPoseK + k] = pd[(size_t)k * 3 * V + 3 * v + c];
    }
  TRY(pack_linear(h, W.data(), 3 * Vp, kPoseK, nullptr, &s.posedirs, kPoseKpad));
  std::vector<float> vtp((size_t)Vp * 3, 0.0f), lw((size_t)nt * kJ * VT, 0.0f);
  std::copy(vt, vt + (size_t)V * 3, vtp.begin());
  std::vector<uint32_t> jm(nt, 0u);
  const float* w = rt(h, p + "lbs_weights").host.data();
  for (int v = 0; v < V; ++v)
    for (int j = 0; j < kJ; ++j) {
      const float x = w[(size_t)v * kJ + j];
      lw[((size_t)(v / VT) * kJ + j) * VT + v % VT] = x;
      if (x != 0.0f) jm[v / VT] |= 1u << j;        // a zero weight adds nothing to T_v; a NaN one is kept
    }
  TRY(upload_f32(h, vtp.data(), vtp.size(), &s.v_template));
  TRY(upload_f32(h, lw.data(), lw.size(), &s.lbsw));
  TRY(dev_alloc(h, (void**)&s.jmask, nt * sizeof(uint32_t)));
  CK(cudaMemcpy(s.jmask, jm.data(), nt * sizeof(uint32_t), cudaMemcpyHostToDevice));
  return MLDB_OK;
}

extern "C" int mldb_smpl_forward(mldb_handle* h, const float* feats, const uint8_t* mask, int32_t B, int32_t T,
                                 int32_t jointstype, int32_t vertstrans, float* out, void* stream) {
  if (!h || !feats || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(check_configured(h, h->smpl.on, "smpl", "the SMPL layer"));
  SmplW& s = h->smpl;
  const int V = s.cfg.num_vertices;
  if (B < 1 || T < 1 || (int64_t)B * T > (1 << 24))
    FAIL(MLDB_ERR_INVALID, "features must be [B >= 1, T >= 1, 150] with B * T <= 2^24, got B=%d T=%d", B, T);
  if (jointstype != MLDB_SMPL_JOINTS && jointstype != MLDB_SMPL_VERTICES)
    FAIL(MLDB_ERR_INVALID, "jointstype must be MLDB_SMPL_JOINTS or MLDB_SMPL_VERTICES, got %d", jointstype);
  if (vertstrans != 0 && vertstrans != 1) FAIL(MLDB_ERR_INVALID, "vertstrans must be 0 or 1, got %d", vertstrans);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const bool verts = jointstype == MLDB_SMPL_VERTICES;
  const size_t per_frame = split16_bytes(1, kPoseKpad) / 128 + kXf * sizeof(float);
  const int Bc = eval_chunk(s.chunk, B, verts ? (size_t)T * per_frame : 1, 1);   // joints: no workspace
  const int nout = verts ? V : kJ;
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0), frames = n * T;
    FkParams fp{};
    fp.feats = feats + (int64_t)b0 * T * kFeat;
    fp.mask = mask ? mask + (int64_t)b0 * T : nullptr;
    fp.frames = frames; fp.T = T; fp.vertstrans = vertstrans;
    memcpy(fp.J, s.J, sizeof fp.J);
    memcpy(fp.parents, s.parents, sizeof fp.parents);
    float* o = out + (int64_t)b0 * nout * 3 * T;
    ActBuf A{};
    if (verts) {
      TRY(grow_act(s.feat, frames, kPoseKpad, &A));
      TRY(grow(s.xf, (size_t)frames * kXf * sizeof(float)));
      fp.xf = (float*)s.xf.p; fp.feat = A;
    } else {
      fp.joints = o;
    }
    k_smpl_fk<<<(unsigned)std::min((frames + 3) / 4, 16 * h->sm_count), 128, 0, st>>>(fp);
    kcount(h, MLDB_KSTAT_MISC);
    if (!verts) continue;
    const LinW& w = s.posedirs;
    CUtensorMap mAh, mAl, mWh, mWl;
    if (!make_map(&mAh, A.hi, frames, kPoseKpad, LBS_BM) || !make_map(&mAl, A.lo(), frames, kPoseKpad, LBS_BM) ||
        !make_map(&mWh, w.w, w.N, w.K, BN) || !make_map(&mWl, w.w + w.plane_stride, w.N, w.K, BN)) {
      h->op_failed = true;
      break;
    }
    LbsParams lp{};
    lp.frames = frames; lp.T = T; lp.V = V; lp.vtiles = (V + VT - 1) / VT;
    lp.inv_scale = w.inv_scale; lp.xf = (const float*)s.xf.p; lp.vt = s.v_template; lp.lbsw = s.lbsw;
    lp.jmask = s.jmask; lp.out = o;
    // split the vertex tiles over CTAs until the grid covers the SMs (each CTA loads its 64 frames once)
    const int mtiles = (frames + LBS_BM - 1) / LBS_BM;
    const int nsplit = std::max(1, std::min(lp.vtiles, (h->sm_count + mtiles - 1) / mtiles));
    lp.vtiles_per_cta = (lp.vtiles + nsplit - 1) / nsplit;
    const int grid = mtiles * ((lp.vtiles + lp.vtiles_per_cta - 1) / lp.vtiles_per_cta);
    k_smpl_lbs<<<(unsigned)grid, LBS_THREADS, LBS_SMEM, st>>>(mAh, mAl, mWh, mWl, lp);
    kcount(h, MLDB_KSTAT_GEMM_TC);
  }
  return ops_done(h);
}
