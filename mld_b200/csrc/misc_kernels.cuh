// Small elementwise / scan kernels of the sampling path (token assembly, timestep features,
// classifier-free guidance + scheduler update, feats2joints).
#pragma once
#include "ops.cuh"

// get_timestep_embedding (mld/models/architectures/tools/embeddings.py:245-285) for a list of
// integer timesteps: out[i, :] = [cos | sin] (flip_sin_to_cos) of t_i * exp(-ln(1e4) k/(half-shift)).
static __global__ void k_timestep_features(const int64_t* __restrict__ ts, int64_t t_scalar, int n, int dim, int flip,
                                    float freq_shift, float* __restrict__ out) {
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half) return;
  const int i = idx / half, k = idx - i * half;
  float exponent = -9.210340371976184f * (float)k;  // -ln(10000) * k in fp32 like torch
  exponent = exponent / ((float)half - freq_shift);
  const float arg = (float)(ts ? ts[i] : t_scalar) * expf(exponent);
  const float sn = sinf(arg), cs = cosf(arg);
  float* o = out + (int64_t)i * dim;
  if (flip) { o[k] = cs; o[half + k] = sn; }
  else      { o[k] = sn; o[half + k] = cs; }
  if ((dim & 1) && k == 0) o[dim - 1] = 0.0f;
}

// Token assembly for the trans_enc denoiser (mld_denoiser.py:171,187,196):
//   X[s, j]      = latent[(s % lat_mod), j] + pe[j]            j < n_lat
//   X[s, n_lat]  = tt[:]  (time token, pe already added)
// The condition tokens X[s, n_lat+1 ...] are written once per batch by the ctx GEMM.
static __global__ void k_assemble_tokens(ActBuf X, int Ntok, int Bx, int lat_mod, int n_lat, int d,
                                  const float* __restrict__ latents, const float* __restrict__ pe,
                                  const float* __restrict__ tt) {
  pdl_trigger();
  pdl_wait();
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)Bx * (n_lat + 1) * d;
  if (idx >= total) return;
  const int n = (int)(idx % d);
  const int j = (int)((idx / d) % (n_lat + 1));
  const int s = (int)(idx / ((int64_t)d * (n_lat + 1)));
  float v;
  if (j < n_lat) v = latents[((int64_t)(s % lat_mod) * n_lat + j) * d + n] + pe[(int64_t)j * d + n];
  else v = tt[n];
  __half h, l;
  split_f32(v, h, l);
  const int64_t o = ((int64_t)s * Ntok + j) * X.cols + n;
  X.hi[o] = h;
  X.lo()[o] = l;
}

// Rows of a split buffer <- fp32 rows (+ optional table row), with the (seq, pos) row mapping.
//   X[(r / in_group) * out_group + out_off + r % in_group, :] = src[src_row(r), :] + tab[out_off + r % in_group, :]
// src_row(r) = r (src_bcast == 0) or r % in_group (broadcast one group to every sequence).
// idx_ptr != null: src is offset by *idx_ptr * idx_stride floats (the step counter of a replayed step graph).
static __global__ void k_rows_to_split(ActBuf X, const float* __restrict__ src, int ld_src, int M, int d,
                                int in_group, int out_group, int out_off, int src_bcast,
                                const float* __restrict__ tab, int relu = 0, const int* __restrict__ idx_ptr = nullptr,
                                int64_t idx_stride = 0) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)M * d) return;
  if (idx_ptr) src += (int64_t)(*idx_ptr) * idx_stride;
  const int n = (int)(idx % d);
  const int r = (int)(idx / d);
  const int seq = r / in_group, pos = r - seq * in_group;
  float v = 0.0f;
  if (src) v = src[(int64_t)(src_bcast ? pos : r) * ld_src + n];
  if (relu) v = fmaxf(v, 0.0f);
  if (tab) v += tab[(int64_t)(out_off + pos) * d + n];
  __half h, l;
  split_f32(v, h, l);
  const int64_t o = ((int64_t)seq * out_group + out_off + pos) * X.cols + n;
  X.hi[o] = h;
  X.lo()[o] = l;
}

// The same mapping, eight columns per thread: two 128-bit loads of the fp32 source (the CLIP context:
// coalesced 128-bit HBM loads), one 128-bit store per fp16 plane.  Needs d % 8 == 0, ld_src % 4 == 0,
// X.cols % 8 == 0 and 16-byte aligned bases (checked by the caller).
static __global__ void k_rows_to_split8(ActBuf X, const float* __restrict__ src, int ld_src, int M, int d,
                                 int in_group, int out_group, int out_off, int src_bcast,
                                 const float* __restrict__ tab, int relu) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int d8 = d >> 3;
  if (idx >= (int64_t)M * d8) return;
  const int n = (int)(idx % d8) * 8;
  const int r = (int)(idx / d8);
  const int seq = r / in_group, pos = r - seq * in_group;
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (src) {
    const float4* s4 = reinterpret_cast<const float4*>(src + (int64_t)(src_bcast ? pos : r) * ld_src + n);
    const float4 a = __ldg(s4), b = __ldg(s4 + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  if (relu) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = fmaxf(v[i], 0.0f);
  }
  if (tab) {
    const float4* t4 = reinterpret_cast<const float4*>(tab + (int64_t)(out_off + pos) * d + n);
    const float4 a = __ldg(t4), b = __ldg(t4 + 1);
    v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
  }
  uint32_t ph[4], pl[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2 h2 = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    const float2 hf = __half22float2(h2);
    const __half2 l2 = __floats2half2_rn(v[2 * i] - hf.x, v[2 * i + 1] - hf.y);
    ph[i] = *reinterpret_cast<const uint32_t*>(&h2);
    pl[i] = *reinterpret_cast<const uint32_t*>(&l2);
  }
  const int64_t o = ((int64_t)seq * out_group + out_off + pos) * X.cols + n;
  *reinterpret_cast<uint4*>(X.hi + o) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
  *reinterpret_cast<uint4*>(X.lo() + o) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
}

// fp32 [rows, cols] -> split16 [rep * rows, X.cols] with the columns zero-padded to X.cols (a multiple
// of 64: the K extent of a tensor-core GEMM whose true K is odd, e.g. the 263 motion features) and the
// rows written `rep` times (torch.cat([latents] * 2), mld.py:325: both guidance halves see the same input).
static __global__ void k_f32_to_split_pad(ActBuf X, const float* __restrict__ src, int ld_src, int rows, int cols, int rep) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)rows * X.cols) return;
  const int n = (int)(idx % X.cols);
  const int r = (int)(idx / X.cols);
  const float v = n < cols ? src[(int64_t)r * ld_src + n] : 0.0f;
  __half h, l;
  split_f32(v, h, l);
  for (int k = 0; k < rep; ++k) {
    const int64_t o = ((int64_t)k * rows + r) * X.cols + n;
    X.hi[o] = h;
    X.lo()[o] = l;
  }
}

// the first n elements of a split16 buffer whose rows are contiguous (cols == leading dimension), widened to fp32
static __global__ void k_split_to_f32(ActBuf X, float* __restrict__ out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = join_f32(X.hi[i], X.lo()[i]);
}

// device-side step counter of a replayed single-step graph (the 1000-step DDPM loop of the no-VAE model)
static __global__ void k_step_set(int* step, int v) { *step = v; }
static __global__ void k_step_inc(int* step) { *step += 1; }

// [A, B, d] -> [B, A, d] fp32 (latents [B,n_lat,d] <-> [n_lat,B,d], mld.py:359; mld_vae.py:247)
static __global__ void k_permute_01(const float* __restrict__ src, float* __restrict__ dst, int A, int B, int d) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)A * B * d) return;
  const int n = (int)(idx % d);
  const int b = (int)((idx / d) % B);
  const int a = (int)(idx / ((int64_t)d * B));
  dst[((int64_t)b * A + a) * d + n] = src[idx];
}

__device__ __forceinline__ float sched_update(const StepCoef& k, float x, float e, float nz) {
  // pred_original_sample = (sample - beta_prod_t ** 0.5 * model_output) / alpha_prod_t ** 0.5
  float x0 = __fdiv_rn(__fsub_rn(x, __fmul_rn(k.c1, e)), k.c0);
  if (k.clip) x0 = x0 < -1.0f ? -1.0f : (x0 > 1.0f ? 1.0f : x0);   // torch.clamp: a NaN stays NaN
  // DDIM: prev = alpha_prod_t_prev ** 0.5 * x0 + (1 - alpha_prod_t_prev - std_dev_t ** 2) ** 0.5 * model_output
  // DDPM: prev = x0 coeff * x0 + sample coeff * sample
  float p = __fadd_rn(__fmul_rn(k.c2, x0), __fmul_rn(k.c3, k.kind == 0 ? e : x));
  // + std_dev_t * variance_noise (DDIM, eta > 0) / + variance ** 0.5 * variance_noise (DDPM, t > 0)
  if (k.sigma != 0.0f) p = __fadd_rn(p, __fmul_rn(k.sigma, nz));
  return p;
}

// Classifier-free guidance (mld.py:339-342) + scheduler.step (mld.py:345), in place on latents.
//   eps: [Bx, per] with the uncond half first when cfg_on; latents: [B, per];
//   noise_base: [n_steps, B, per] injected N(0,1) or null, read only by steps with a non-zero sigma;
//   step_ptr != null overrides `step` (device-side counter of a replayed step graph).
static __global__ void k_cfg_sched(const float* __restrict__ eps, float* __restrict__ latents,
                            const float* __restrict__ noise_base, int64_t n_per_half, int cfg_on,
                            float guidance, const StepCoef* __restrict__ coefs, int step,
                            const int* __restrict__ step_ptr) {
  pdl_trigger();
  pdl_wait();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_per_half) return;
  if (step_ptr) step = *step_ptr;
  float e = eps[i];
  if (cfg_on) {
    const float c = eps[n_per_half + i];
    e = __fadd_rn(e, __fmul_rn(guidance, __fsub_rn(c, e)));
  }
  const StepCoef k = coefs[step];
  const float nz = noise_base && k.sigma != 0.0f ? noise_base[(int64_t)step * n_per_half + i] : 0.0f;
  latents[i] = sched_update(k, latents[i], e, nz);
}

static __global__ void k_sched_step(const float* __restrict__ eps, const float* __restrict__ sample,
                             const float* __restrict__ noise, float* __restrict__ out, int64_t n,
                             StepCoef k) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = sched_update(k, sample[i], eps[i], noise && k.sigma != 0.0f ? noise[i] : 0.0f);
}

// feats2joints (mld/data/HumanML3D.py:41-45 -> motion_process.py:415-431, 362-381;
// quaternion.py:16-20, 54-73).  One block per motion, frames in chunks of F2J_CHUNK.  Per chunk,
// thread 0 continues the two sequential fp32 prefix sums in the reference's order (torch.cumsum on CPU
// is a serial sum), then all threads rotate the chunk's rotation-invariant joint coordinates into the
// global frame.  The chunking bounds the shared memory at any motion length.
//   feats [B, T, F] normalised; joints [B, T, J, 3]
constexpr int F2J_CHUNK = 1024;
static __global__ void __launch_bounds__(256) k_feats2joints(const float* __restrict__ feats,
                                                      const float* __restrict__ mean,
                                                      const float* __restrict__ stdv, int T, int F,
                                                      int J, float* __restrict__ joints) {
  __shared__ float cs[F2J_CHUNK];   // cos(angle)
  __shared__ float sn[F2J_CHUNK];   // sin(angle)
  __shared__ float px[F2J_CHUNK];   // root x
  __shared__ float pz[F2J_CHUNK];   // root z
  const int b = blockIdx.x;
  const float* f = feats + (int64_t)b * T * F;
  float* out = joints + (int64_t)b * T * J * 3;
  float ang = 0.0f, ax = 0.0f, az = 0.0f;   // thread 0's running sums across chunks
  for (int t0 = 0; t0 < T; t0 += F2J_CHUNK) {
    const int n = min(F2J_CHUNK, T - t0);
    if (threadIdx.x == 0) {
      // r_rot_ang[t] = sum_{u<t} rot_vel[u]; quaternion q = (cos, 0, sin, 0); r_pos accumulates
      // qrot(qinv(q[t]), (vx[t-1], 0, vz[t-1])).
      for (int u = 0; u < n; ++u) {
        const int t = t0 + u;
        float vx = 0.0f, vz = 0.0f;
        if (t > 0) {
          const float* fp = f + (int64_t)(t - 1) * F;
          ang = __fadd_rn(ang, __fadd_rn(__fmul_rn(fp[0], stdv[0]), mean[0]));
          vx = __fadd_rn(__fmul_rn(fp[1], stdv[1]), mean[1]);
          vz = __fadd_rn(__fmul_rn(fp[2], stdv[2]), mean[2]);
        }
        const float c = cosf(ang), s = sinf(ang);
        cs[u] = c;
        sn[u] = s;
        // qrot with q = (w=c, x=0, y=-s, z=0) on v=(vx,0,vz):
        //   uv = cross(qvec, v) = (-s*vz, 0, s*vx); uuv = cross(qvec, uv) = (-s*s*vx, 0, -s*s*vz)
        //   out = v + 2*(w*uv + uuv)
        const float uvx = -s * vz, uvz = s * vx;
        const float uuvx = -s * uvz, uuvz = s * uvx;
        const float rx = vx + 2.0f * (c * uvx + uuvx);
        const float rz = vz + 2.0f * (c * uvz + uuvz);
        ax = __fadd_rn(ax, rx);
        az = __fadd_rn(az, rz);
        px[u] = ax;
        pz[u] = az;
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n * J; i += blockDim.x) {
      const int u = i / J, j = i - u * J;
      const float* fp = f + (int64_t)(t0 + u) * F;
      float x, y, z;
      if (j == 0) {
        x = px[u];
        y = fp[3] * stdv[3] + mean[3];
        z = pz[u];
      } else {
        const int o = 4 + (j - 1) * 3;
        const float vx = fp[o] * stdv[o] + mean[o];
        const float vy = fp[o + 1] * stdv[o + 1] + mean[o + 1];
        const float vz = fp[o + 2] * stdv[o + 2] + mean[o + 2];
        const float c = cs[u], s = sn[u];
        // qvec = (0, -s, 0): uv = cross(qvec, v) = (-s*vz, 0, s*vx)
        const float uvx = -s * vz, uvz = s * vx;
        const float uuvx = -s * uvz, uuvz = s * uvx;
        x = vx + 2.0f * (c * uvx + uuvx) + px[u];
        y = vy;
        z = vz + 2.0f * (c * uvz + uuvz) + pz[u];
      }
      const int64_t oi = (int64_t)t0 * J + i;
      out[oi * 3 + 0] = x;
      out[oi * 3 + 1] = y;
      out[oi * 3 + 2] = z;
    }
    __syncthreads();                        // the next chunk overwrites the tables
  }
}
