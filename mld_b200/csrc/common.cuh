// Shared device/host helpers for libmldb200 (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

void mldb_set_err(const std::string& s);   // engine.cu: the message mldb_last_error() returns

// ---------------------------------------------------------------------------------------
// "split16" activation format.  Every activation tensor that feeds a GEMM is stored as two
// fp16 planes hi = fp16(x), lo = fp16(x - hi); hi + lo carries ~22 significant bits.  The
// tensor-core GEMMs compute A_hi*W_hi + A_lo*W_hi + A_hi*W_lo with fp32 accumulation, which
// reproduces the reference's fp32 GEMMs to ~1e-6 relative (a single fp16/tf32 pass is ~5e-4
// and does not survive 50 guided DDIM steps within the 1e-3 joint-position gate).
// Planes are row-major [rows, cols]; lo plane = hi plane + plane_stride elements.
// ---------------------------------------------------------------------------------------
struct ActBuf {
  __half* hi;            // plane 0
  int64_t plane_stride;  // elements between the hi and lo planes
  int rows, cols;        // logical shape (cols == leading dimension)
  __host__ __device__ __half* lo() const { return hi + plane_stride; }
};

__device__ __forceinline__ void split_f32(float x, __half& hi, __half& lo) {
  hi = __float2half_rn(x);
  lo = __float2half_rn(x - __half2float(hi));
}
__device__ __forceinline__ float join_f32(__half hi, __half lo) {
  return __half2float(hi) + __half2float(lo);
}

__device__ __forceinline__ float gelu_erf(float x) {
  // F.gelu default (exact erf form), cross_attention.py:408-409
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
// GELU with erf from Abramowitz-Stegun 7.1.26 (|erf error| < 1.5e-7, i.e. at the level of the fp32
// rounding of the exact-erf form): one rcp, one ex2, six FMAs - about half the instructions of erff.
// Used by the tensor-core GEMM epilogue, where the FFN up-projection is epilogue-bound.
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z * z));
  const float erf_abs = fmaf(-poly * t, e, 1.0f);
  return 0.5f * x * (1.0f + copysignf(erf_abs, x));
}
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
// CLIP's quick-GELU x * sigmoid(1.702 x) (transformers ACT2FN["quick_gelu"])
__device__ __forceinline__ float quick_gelu_f(float x) { return x / (1.0f + expf(-1.702f * x)); }

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-serialization
// attribute may begin (prologue: barrier init, descriptor prefetch) while its predecessor
// drains; it must execute pdl_wait() before touching anything the predecessor produced or reads.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

#ifdef __CUDACC__
extern int g_mldb_pdl;   // 1 = launch the step-loop kernels with the PDL attribute (MLDB_PDL=0 disables)
template <typename... KArgs, typename... Args>
static inline void launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                      int cluster, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (g_mldb_pdl) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster > 1) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = (unsigned)cluster; at[n].val.clusterDim.y = 1; at[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = at; cfg.numAttrs = n;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
static inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
  launch_pdl_cluster(kernel, grid, block, smem, st, 1, static_cast<Args&&>(args)...);
}
// Opt `kernel` in to `bytes` of dynamic shared memory (outside stream capture).  false: the attribute was refused
// and mldb_last_error() says so.
template <typename... KArgs>
static inline bool smem_opt_in(void (*kernel)(KArgs...), int bytes, const char* name) {
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) mldb_set_err(std::string("cudaFuncSetAttribute(") + name + "): " + cudaGetErrorString(e));
  return e == cudaSuccess;
}
#endif

enum ActKind { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2, ACT_SILU = 3, ACT_QUICKGELU = 4, ACT_LEAKY = 5 };

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case ACT_GELU: return gelu_erf(v);
    case ACT_RELU: return fmaxf(v, 0.0f);
    case ACT_SILU: return silu_f(v);
    case ACT_QUICKGELU: return quick_gelu_f(v);
    case ACT_LEAKY: return v > 0.0f ? v : v * 0.2f;   // nn.LeakyReLU(0.2) (the T2M evaluator)
    default: return v;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
