// APE and AVE of the text-to-motion test (TemosMetric = ComputeMetrics.update, mld/models/metrics/compute.py): both
// joint tensors through the Rifke feature round trip (transforms/joints2jfeats/rifke.py), then per sequence the
// position errors summed over the valid frames and the distance between the per-coordinate variances.
//
//   k_ape_ave         one CTA per sequence (a grid of at most kApeCtas CTAs walks b, b + grid, ...), both inputs
//                     in the same CTA since every term compares text and ref at the same frame.  All arithmetic is
//                     in double.  (1) a min/max reduction over all T frames of the lowest foot height gives each
//                     input's floor (padding included, as the reference computes it before remove_padding).  (2) per
//                     tile of 128 valid frames, one thread per frame computes the forward direction, the relative
//                     angle and the frame's trajectory step, and a block scan integrates the trajectory; (3) each
//                     warp then takes every 4th frame of the tile with one lane per joint and sums the L2 errors and
//                     the shifted first and second moments of each coordinate.  The warps' sums are added in a fixed
//                     order and the CTA's sequences into one partial row, also in order.
//   k_ape_ave_reduce  one CTA: the partial rows summed in order into the [4 J + 2] fp32 output, so that the result
//                     is the same bits from run to run.
#include "engine.h"

#include <math.h>

namespace {

constexpr int kThreads = 128, kWarps = kThreads / 32;
constexpr int kMaxJ = 22;
constexpr int kApeCtas = 1024;
constexpr int kMaxRow = 4 * kMaxJ + 2;
constexpr int kQ = 27;          // per-joint sums: APE joint, APE pose, APE traj, 12 joint moments, 12 pose moments

// The joint tables of mld/utils/joints.py.  The forward direction reads the shoulders and hips from the array with
// the root removed but looks them up in the full table, so it reads the joints one index further (rifke.py:43,55);
// the indices below are those original joints.  The feet of the floor are not shifted.
struct JointTable {
  int J;
  int feet[4];
  int ls, rs, lh, rh;
  double factor;                // to meters
};
constexpr JointTable kHumanml3d{22, {8, 11, 7, 10}, 18, 17, 3, 2, 1000.0 * 0.75 / 480.0};
constexpr JointTable kMmm{21, {14, 15, 19, 20}, 6, 9, 12, 17, 1000.0};

struct ApeArgs {
  const float* x[2];            // text, ref [B, T, J, 3]
  const int32_t* lengths;       // [B]
  int B, T, J;
  int feet[4], ls, rs, lh, rh;
  double factor;
  double* part;                 // [gridDim.x, 4 J + 2]
  float* out;                   // [4 J + 2]
};

// One frame's rotation state: the raw root (x, z), the normalised forward (sin, cos) of the inverse rotation, the
// (cos, sin) of the angle relative to frame 0, and the integrated trajectory.
struct FrameSm {
  double rx[2][kThreads], rz[2][kThreads], fs[2][kThreads], fc[2][kThreads];
  double C[2][kThreads], S[2][kThreads], tx[2][kThreads], tz[2][kThreads];
};

__device__ __forceinline__ void forward_dir(const float* x, int t, const ApeArgs& a, double& fs, double& fc) {
  const float* f = x + (int64_t)t * a.J * 3;
  const double rx = f[0], rz = f[2];
  // across = P[RH] - P[LH] + P[RS] - P[LS] on the root-relative poses, evaluated left to right as torch does
  const double ax = (((double)f[a.rh * 3] - rx) - ((double)f[a.lh * 3] - rx) + ((double)f[a.rs * 3] - rx)) -
                    ((double)f[a.ls * 3] - rx);
  const double az = (((double)f[a.rh * 3 + 2] - rz) - ((double)f[a.lh * 3 + 2] - rz) +
                     ((double)f[a.rs * 3 + 2] - rz)) - ((double)f[a.ls * 3 + 2] - rz);
  // F.normalize: x / max(|x|, 1e-12), so a zero `across` gives forward (0, 0): angle atan2(0, 0) = 0 and a zero
  // inverse rotation
  const double s = -az, c = ax;
  const double n = fmax(sqrt(s * s + c * c), 1e-12);
  fs = s / n;
  fc = c / n;
}

// Joint j of frame t of one input, in the output units: the reconstructed joint (jts) and the local pose (pose,
// joints >= 1).  The angle relative to frame 0 is (C, S); the trajectory (tx, tz).
__device__ __forceinline__ void joint_vals(const float* p, int j, double floor, double factor, double rx, double rz,
                                           double fs, double fc, double C, double S, double tx, double tz,
                                           double jts[3], double pose[3]) {
  const double y = ((double)p[1] - floor) / factor;
  if (j == 0) {
    jts[0] = tx / factor; jts[1] = y; jts[2] = tz / factor;
    pose[0] = pose[1] = pose[2] = 0.0;
    return;
  }
  const double dx = (double)p[0] - rx, dz = (double)p[2] - rz;
  const double lx = dx * fc - dz * fs, lz = dx * fs + dz * fc;        // [x, z] . R_inv, R_inv = [[c, s], [-s, c]]
  const double px = lx * C + lz * S, pz = -lx * S + lz * C;          // [x, z] . R,     R     = [[C, -S], [S, C]]
  jts[0] = (px + tx) / factor; jts[1] = y; jts[2] = (pz + tz) / factor;
  pose[0] = lx / factor; pose[1] = y; pose[2] = lz / factor;
}

__device__ __forceinline__ double norm3(const double a[3], const double b[3]) {
  const double x = a[0] - b[0], y = a[1] - b[1], z = a[2] - b[2];
  return sqrt(x * x + y * y + z * z);
}

__device__ __forceinline__ double var_of(double s1, double s2, double n) { return (s2 - s1 * s1 / n) / (n - 1.0); }

__global__ void __launch_bounds__(kThreads) k_ape_ave(ApeArgs a) {
  __shared__ union {
    FrameSm fr;
    double red[kWarps][kQ][32];
  } sm;
  __shared__ double s_mm[kWarps][4], s_scan[kWarps][4], s_carry[4];
  __shared__ double s_floor[2], s_f0[2][2];           // floor; frame 0's (fs, fc) and the angle a_0 come from it
  __shared__ double s_a0[2], s_r0[2][2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int J = a.J, T = a.T, row = 4 * J + 2;
  const int64_t seq = (int64_t)T * J * 3;
  // the CTA's row: thread j < J owns APE_pose[j - 1], APE_joints[j], AVE_pose[j - 1], AVE_joints[j]; thread 0 also
  // APE_root, APE_traj, AVE_root, AVE_traj
  double r_ape_j = 0.0, r_ape_p = 0.0, r_ave_j = 0.0, r_ave_p = 0.0, r_ape_tr = 0.0, r_ave_tr = 0.0;

  for (int b = blockIdx.x; b < a.B; b += gridDim.x) {
    const int L = a.lengths[b];
    if (L < 2 || L > T) {                             // the host refuses these; a bad device copy shows as NaN
      r_ape_j = r_ape_p = r_ave_j = r_ave_p = r_ape_tr = r_ave_tr = nan("");
      continue;
    }
    const float* xs[2] = {a.x[0] + b * seq, a.x[1] + b * seq};

    // (1) floor = softmin(h, 0.5) = min h - log(0.5 + exp(min h - max h)) over every frame of the padded tensor
    double mn[2] = {INFINITY, INFINITY}, mx[2] = {-INFINITY, -INFINITY};
    for (int t = tid; t < T; t += kThreads)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const float* f = xs[k] + (int64_t)t * J * 3;
        double h = f[a.feet[0] * 3 + 1];
#pragma unroll
        for (int i = 1; i < 4; ++i) h = fmin(h, (double)f[a.feet[i] * 3 + 1]);
        mn[k] = fmin(mn[k], h);
        mx[k] = fmax(mx[k], h);
      }
#pragma unroll
    for (int o = 16; o; o >>= 1)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        mn[k] = fmin(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
        mx[k] = fmax(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
      }
    if (lane == 0) {
      s_mm[warp][0] = mn[0]; s_mm[warp][1] = mn[1]; s_mm[warp][2] = mx[0]; s_mm[warp][3] = mx[1];
    }
    __syncthreads();
    if (tid < 2) {
      double lo = s_mm[0][tid], hi = s_mm[0][2 + tid];
      for (int w = 1; w < kWarps; ++w) { lo = fmin(lo, s_mm[w][tid]); hi = fmax(hi, s_mm[w][2 + tid]); }
      s_floor[tid] = lo - log(0.5 + exp(lo - hi));
      double fs, fc;
      forward_dir(xs[tid], 0, a, fs, fc);
      s_f0[tid][0] = fs; s_f0[tid][1] = fc;
      s_a0[tid] = atan2(fs, fc);
      s_r0[tid][0] = xs[tid][0]; s_r0[tid][1] = xs[tid][2];
    }
    if (tid < 4) s_carry[tid] = 0.0;
    __syncthreads();
    const double flo[2] = {s_floor[0], s_floor[1]};

    // the moments are shifted by frame 0's values (C = 1, S = 0 and a zero trajectory there)
    double sh_j[2][3], sh_p[2][3];
    if (lane < J) {
#pragma unroll
      for (int k = 0; k < 2; ++k)
        joint_vals(xs[k] + lane * 3, lane, flo[k], a.factor, s_r0[k][0], s_r0[k][1], s_f0[k][0], s_f0[k][1],
                   1.0, 0.0, 0.0, 0.0, sh_j[k], sh_p[k]);
    }
    double acc[kQ];
#pragma unroll
    for (int q = 0; q < kQ; ++q) acc[q] = 0.0;

    for (int t0 = 0; t0 < L; t0 += kThreads) {
      // (2) one thread per frame: rotation state and trajectory step, then the block scan of the steps
      const int t = t0 + tid;
      double v[4] = {0.0, 0.0, 0.0, 0.0};
      if (t < L) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          double fs, fc;
          forward_dir(xs[k], t, a, fs, fc);
          const double th = atan2(fs, fc) - s_a0[k];   // the cumsum of the angle's diff, minus its first value
          double S, C;
          sincos(th, &S, &C);
          const float* r = xs[k] + (int64_t)t * J * 3;
          const float* rp = t ? r - J * 3 : r;
          const double dx = (double)r[0] - rp[0], dz = (double)r[2] - rp[2];
          const double lx = dx * fc - dz * fs, lz = dx * fs + dz * fc;
          v[2 * k] = lx * C + lz * S;
          v[2 * k + 1] = -lx * S + lz * C;
          sm.fr.rx[k][tid] = r[0]; sm.fr.rz[k][tid] = r[2];
          sm.fr.fs[k][tid] = fs; sm.fr.fc[k][tid] = fc;
          sm.fr.C[k][tid] = C; sm.fr.S[k][tid] = S;
        }
      }
#pragma unroll
      for (int o = 1; o < 32; o <<= 1)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const double u = __shfl_up_sync(0xffffffffu, v[q], o);
          if (lane >= o) v[q] += u;
        }
      if (lane == 31)
#pragma unroll
        for (int q = 0; q < 4; ++q) s_scan[warp][q] = v[q];
      __syncthreads();
      double carry[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        double pre = s_carry[q];
        carry[q] = s_carry[q];
        for (int w = 0; w < kWarps; ++w) {
          if (w < warp) pre += s_scan[w][q];
          carry[q] += s_scan[w][q];
        }
        v[q] += pre;
      }
#pragma unroll
      for (int k = 0; k < 2; ++k) { sm.fr.tx[k][tid] = v[2 * k]; sm.fr.tz[k][tid] = v[2 * k + 1]; }
      __syncthreads();
      if (tid == 0)                                   // every thread has read s_carry; the next tile reads it
#pragma unroll                                        // after its scan barrier
        for (int q = 0; q < 4; ++q) s_carry[q] = carry[q];

      // (3) lane = joint, warp = every 4th frame of the tile
      const int nt = min(kThreads, L - t0);
      if (lane < J) {
        for (int i = warp; i < nt; i += kWarps) {
          double jt[2][3], ps[2][3];
#pragma unroll
          for (int k = 0; k < 2; ++k)
            joint_vals(xs[k] + ((int64_t)(t0 + i) * J + lane) * 3, lane, flo[k], a.factor, sm.fr.rx[k][i],
                       sm.fr.rz[k][i], sm.fr.fs[k][i], sm.fr.fc[k][i], sm.fr.C[k][i], sm.fr.S[k][i],
                       sm.fr.tx[k][i], sm.fr.tz[k][i], jt[k], ps[k]);
          acc[0] += norm3(jt[0], jt[1]);
          acc[1] += norm3(ps[0], ps[1]);
          const double ex = jt[0][0] - jt[1][0], ez = jt[0][2] - jt[1][2];
          acc[2] += sqrt(ex * ex + ez * ez);
#pragma unroll
          for (int k = 0; k < 2; ++k)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const double dj = jt[k][c] - sh_j[k][c], dp = ps[k][c] - sh_p[k][c];
              acc[3 + (k * 3 + c) * 2] += dj;
              acc[4 + (k * 3 + c) * 2] += dj * dj;
              acc[15 + (k * 3 + c) * 2] += dp;
              acc[16 + (k * 3 + c) * 2] += dp * dp;
            }
        }
      }
      __syncthreads();
    }

    // the warps' sums in a fixed order; thread j < J finishes joint j
#pragma unroll
    for (int q = 0; q < kQ; ++q) sm.red[warp][q][lane] = acc[q];
    __syncthreads();
    if (tid < J) {
      double tot[kQ];
#pragma unroll
      for (int q = 0; q < kQ; ++q) {
        tot[q] = sm.red[0][q][tid];
#pragma unroll
        for (int w = 1; w < kWarps; ++w) tot[q] += sm.red[w][q][tid];
      }
      const double n = L;
      double ej = 0.0, ep = 0.0, vj[3], vp[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        vj[c] = var_of(tot[3 + c * 2], tot[4 + c * 2], n) - var_of(tot[9 + c * 2], tot[10 + c * 2], n);
        vp[c] = var_of(tot[15 + c * 2], tot[16 + c * 2], n) - var_of(tot[21 + c * 2], tot[22 + c * 2], n);
        ej += vj[c] * vj[c];
        ep += vp[c] * vp[c];
      }
      r_ape_j += tot[0];
      r_ape_p += tot[1];
      r_ave_j += sqrt(ej);
      r_ave_p += sqrt(ep);
      if (tid == 0) {
        r_ape_tr += tot[2];
        r_ave_tr += sqrt(vj[0] * vj[0] + vj[2] * vj[2]);
      }
    }
    __syncthreads();
  }

  double* p = a.part + (int64_t)blockIdx.x * row;
  if (tid < J) {
    p[J + 1 + tid] = r_ape_j;
    p[3 * J + 2 + tid] = r_ave_j;
    if (tid) {
      p[1 + tid] = r_ape_p;
      p[2 * J + 2 + tid] = r_ave_p;
    } else {
      p[0] = r_ape_j;                                 // the root is joint 0 of the reconstructed joints
      p[1] = r_ape_tr;
      p[2 * J + 1] = r_ave_j;
      p[2 * J + 2] = r_ave_tr;
    }
  }
}

__global__ void __launch_bounds__(kThreads) k_ape_ave_reduce(const double* part, int nrows, int row, float* out) {
  for (int q = threadIdx.x; q < row; q += kThreads) {
    double s = 0.0;
    for (int r = 0; r < nrows; ++r) s += part[(int64_t)r * row + q];
    out[q] = (float)s;
  }
}

}  // namespace

extern "C" int mldb_ape_ave(mldb_handle* h, const float* jts_text, const float* jts_ref, const int32_t* lengths,
                            int32_t B, int32_t T, int32_t J, int32_t jointstype, int32_t force_in_meter, float* out,
                            void* stream) {
  if (!h || !jts_text || !jts_ref || !lengths || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  const JointTable* tab = jointstype == MLDB_JOINTS_HUMANML3D ? &kHumanml3d
                        : jointstype == MLDB_JOINTS_MMM       ? &kMmm
                                                              : nullptr;
  if (!tab) FAIL(MLDB_ERR_INVALID, "jointstype must be MLDB_JOINTS_HUMANML3D or MLDB_JOINTS_MMM, got %d", jointstype);
  if (J != tab->J) FAIL(MLDB_ERR_INVALID, "this jointstype has %d joints, got J=%d", tab->J, J);
  if (B < 1 || T < 2 || (int64_t)B * T * J * 3 >= ((int64_t)1 << 40))
    FAIL(MLDB_ERR_INVALID, "joints must be [B >= 1, T >= 2, J, 3], got B=%d T=%d", B, T);
  if (force_in_meter != 0 && force_in_meter != 1)
    FAIL(MLDB_ERR_INVALID, "force_in_meter must be 0 or 1, got %d", force_in_meter);
  DeviceGuard guard(h->device);
  if (!h->ape_part) TRY(dev_alloc(h, (void**)&h->ape_part, sizeof(double) * kApeCtas * kMaxRow));
  cudaStream_t st = (cudaStream_t)stream;
  ApeArgs a{};
  a.x[0] = jts_text; a.x[1] = jts_ref; a.lengths = lengths;
  a.B = B; a.T = T; a.J = J;
  for (int i = 0; i < 4; ++i) a.feet[i] = tab->feet[i];
  a.ls = tab->ls; a.rs = tab->rs; a.lh = tab->lh; a.rh = tab->rh;
  a.factor = force_in_meter ? tab->factor : 1.0;
  a.part = h->ape_part; a.out = out;
  const int grid = B < kApeCtas ? B : kApeCtas;
  k_ape_ave<<<grid, kThreads, 0, st>>>(a);
  kcount(h, MLDB_KSTAT_MISC);
  k_ape_ave_reduce<<<1, kThreads, 0, st>>>(h->ape_part, grid, 4 * J + 2, out);
  kcount(h, MLDB_KSTAT_MISC);
  return ops_done(h);
}
