// PTX wrappers shared by the warpgroup-MMA kernels (gemm_tc.cu, attn_tc.cu, gru_tc.cu, tconv_tc.cu, smpl.cu):
// mbarriers, TMA (bulk tensor copies), wgmma.mma_async and its shared-memory matrix descriptors, the split16
// k-block, the TMA rings and the 128-row warp-specialised CTA; on the host, the tensor maps of split16 planes.
// sm_90a only.
#pragma once
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>

#include "common.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// Bytes from the dynamic shared-memory window `raw` up to the next 1024-B boundary: a 128B-swizzled tile (TMA box
// and wgmma descriptor, make_desc) must start on one, so every kernel reserves 1024 B of slack and takes its tiles
// from raw + smem_pad1024(raw) (pointer arithmetic: an integer round trip would lose the shared address space).
// An offset rather than the aligned pointer: nvcc folds a returned pointer into k_ffn_tc's and k_proj_tc's ring
// addresses differently.
__device__ __forceinline__ uint32_t smem_pad1024(const void* raw) { return (1024u - (smem_u32(raw) & 1023u)) & 1023u; }

// ---------------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_cnt(uint32_t bar, uint32_t n) {   // n arrivals at once
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(n) : "memory");
}
// A lost arrival must not hang the GPU: after ~2 s of spinning the kernel traps (the host sees a
// launch failure instead of a dead box).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0, spins = 0;
  long long t0 = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (!done && (++spins & 1023u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ll) __trap();
    }
  } while (!done);
}
// non-blocking: has the phase of this parity completed?
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}

// ---------------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// pull one box of a tensor into L2 (no shared-memory destination, no barrier): issued one tile ahead so that
// the real TMA loads of a shallow ring hit L2 instead of paying the HBM latency
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// Store one box from shared memory into a tensor (elements outside the tensor are not written), as part of the
// issuing thread's current bulk group.  The shared-memory source is reused only after bulk_wait_read.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1) : "memory");
}
// close the issuing thread's bulk group / wait until at most N of its groups still read their shared memory
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// make this thread's shared-memory writes (generic proxy) visible to later TMA stores and wgmma operand reads
// (async proxy); a barrier between the writers and the issuing thread follows
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// one lane of a fully converged warp (elect.sync): lets ptxas keep the TMA operands in uniform
// registers instead of emitting a per-instruction ELECT loop for a lane-id branch
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------- warpgroups
// Register re-allocation between the producer warpgroup (which only issues TMA) and the consumer
// warpgroups (which hold the accumulators): executed by every warp of a warpgroup.
template <int N> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// named barrier over `threads` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---------------------------------------------------------------------------------- wgmma
// fence: registers written by this warpgroup (accumulators, A fragments) are ordered before the next
// wgmma.mma_async; commit closes a group of MMAs, wait<N> leaves at most N groups in flight.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// The accumulators of an asynchronous MMA are only valid after wg_wait: pinning them here keeps the compiler from
// moving reads of `d` above the wait (or writes below the next MMA).
template <int N> __device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor, SWIZZLE_128B, 8-row groups 1024 B apart: start address >> 4 |
// LBO << 16 | SBO = 1024 B << 32 | swizzle mode 1 (128 B) << 62.  The tile base is 1024-B aligned.
//   K-major operand : rows = M/N index, 64 K-elements (128 B) per row; next 16-wide k-step = +32 B.
//   MN-major operand: rows = K index, 64 MN-elements (128 B) per row, ONE 64-wide MN block (LBO
//                     unused); next 16-deep k-step = +2048 B.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// Accumulator fragment of a [64 x N] tile (one warpgroup): thread t holds, for every 8-column group j,
// d[4j], d[4j+1] = row 16*(t/32) + (t%32)/4, columns 8j + 2*(t%4), +1 and d[4j+2], d[4j+3] = the same columns
// of row + 8.  Two adjacent groups (16 columns) are exactly the A fragment of a [64 x 16] register operand.
// D[64 x 256] (+)= A[64 x 16] . B[16 x 256], both K-major in shared memory
__device__ __forceinline__ void wgmma_ss_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(acc)
      : "memory");
}
// D[64 x 128] (+)= A[64 x 16] . B[16 x 128], both K-major in shared memory
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(acc)
      : "memory");
}
// D[64 x 96] (+)= A[64 x 16] . B[16 x 96], both K-major in shared memory
__device__ __forceinline__ void wgmma_ss_n96(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
      "%48, %49, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(adesc), "l"(bdesc), "r"(acc)
      : "memory");
}
// D[64 x 64] (+)= A[64 x 16] . B[16 x 64], both K-major in shared memory
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(acc)
      : "memory");
}
// D[64 x 256] (+)= A[64 x 16] (registers) . B[16 x 256] (shared memory, K-major)
__device__ __forceinline__ void wgmma_rs_n256(float (&d)[128], const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %133, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "{%128, %129, %130, %131}, %132, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc)
      : "memory");
}
// D[64 x 48] (+)= A[64 x 16] (registers) . B[16 x 48] (shared memory, K-major)
__device__ __forceinline__ void wgmma_rs_n48(float (&d)[24], const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %29, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
      "{%24, %25, %26, %27}, %28, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc)
      : "memory");
}
// D[64 x 64] (+)= A[64 x 16] (registers) . B[16 x 64] (shared memory, MN-major)
__device__ __forceinline__ void wgmma_rs_n64_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc)
      : "memory");
}

template <int N>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc) {
  static_assert(N == 256 || N == 128 || N == 96 || N == 64, "wgmma_ss width");
  if constexpr (N == 256) wgmma_ss_n256(d, a, b, acc);
  else if constexpr (N == 128) wgmma_ss_n128(d, a, b, acc);
  else if constexpr (N == 96) wgmma_ss_n96(d, a, b, acc);
  else wgmma_ss_n64(d, a, b, acc);
}
// The split16 product of one k-block into a warpgroup's [64 x N] tile: four 16-deep steps of
// A_lo.W_hi + A_hi.W_lo + A_hi.W_hi, in that order, both operands K-major and 64 deep (one 128B swizzle row).
// `first` makes the first MMA overwrite the accumulator.  Every shared-memory-operand kernel goes through here:
// this order fixes the bits of its results.
template <int N>
__device__ __forceinline__ void kblock_ss(float (&d)[N / 2], uint32_t sAh, uint32_t sAl, uint32_t sWh, uint32_t sWl, bool first) {
  uint64_t ah = make_desc(sAh), al = make_desc(sAl), wh = make_desc(sWh), wl = make_desc(sWl);
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    wgmma_ss<N>(d, al, wh, (first && kk == 0) ? 0u : 1u);
    wgmma_ss<N>(d, ah, wl, 1u);
    wgmma_ss<N>(d, ah, wh, 1u);
    ah += 2; al += 2; wh += 2; wl += 2;                // next 16-wide slice: +32 B (>> 4)
  }
}

// ---------------------------------------------------------------------------------- TMA rings
// A ring of S shared-memory slots that TMA fills and MMA warps drain.  Ring position q (a running count of the
// loads that went through the ring) lives in slot q % S, in phase (q / S) & 1 of that slot's two barriers: full[s]
// (one arrival, the producer's expect_tx, plus the TMA bytes) and empty[s] (one arrival per consumer warp once
// its MMAs on the slot have retired).  The producer of position q waits for empty's previous phase, so its first S
// waits return at once on fresh barriers.  init runs on one thread, before fence.mbarrier_init.
template <int S>
struct Ring {
  uint64_t* full;
  uint64_t* empty;
  __device__ __forceinline__ void init(uint32_t consumers) const {
    for (int s = 0; s < S; ++s) {
      mbar_init(smem_u32(&full[s]), 1);
      mbar_init(smem_u32(&empty[s]), consumers);
    }
  }
  __device__ __forceinline__ static uint32_t phase(int q) { return ((uint32_t)(q / S)) & 1u; }
  __device__ __forceinline__ uint32_t full_bar(int q) const { return smem_u32(&full[q % S]); }
  __device__ __forceinline__ void wait_full(int q) const { mbar_wait(full_bar(q), phase(q)); }
  __device__ __forceinline__ void wait_empty(int q) const { mbar_wait(smem_u32(&empty[q % S]), phase(q) ^ 1u); }
  __device__ __forceinline__ bool test_empty(int q) const { return mbar_test(smem_u32(&empty[q % S]), phase(q) ^ 1u); }
  __device__ __forceinline__ void release(int q) const { mbar_arrive(smem_u32(&empty[q % S])); }
};

// The producer warp's loop over n k-blocks, from ring position q on (q is advanced past them).  The whole warp
// walks it (uniform control flow); one elected lane calls before(kb) (k_gemm_tc's L2 prefetch), arms full with
// `bytes` and issues load(kb, slot, full).
struct NoOp { template <class... A> __device__ __forceinline__ void operator()(A&&...) const {} };
template <int S, class Load, class Before = NoOp>
__device__ __forceinline__ void ring_feed(const Ring<S>& ring, int& q, int n, uint32_t bytes, Load&& load,
                                          Before&& before = {}) {
  for (int kb = 0; kb < n; ++kb, ++q) {
    ring.wait_empty(q);
    if (elect_one()) {
      before(kb);
      const uint32_t full = ring.full_bar(q);
      mbar_expect_tx(full, bytes);
      load(kb, q % S, full);
    }
    __syncwarp();
  }
}

// A consumer warpgroup's loop over n k-blocks from ring position q on (q is advanced past them): d = the sum of
// kblock_ss<BN> over them, with stage(kb, slot, ah, al, wh, wl) giving the operand addresses.  Each position is
// released (lane 0 of every warp) once the next one's MMAs are issued and its own have retired, the last one after
// the drain - unless RELEASE_LAST is false: a CTA that loads nothing more leaves it.
template <int BN, bool RELEASE_LAST = true, int S, class Stage>
__device__ __forceinline__ void ring_mma(float (&d)[BN / 2], const Ring<S>& ring, int& q, int n, int lane, Stage&& stage) {
  for (int kb = 0; kb < n; ++kb, ++q) {
    ring.wait_full(q);
    uint32_t ah, al, wh, wl;
    stage(kb, q % S, ah, al, wh, wl);
    wg_fence();
    kblock_ss<BN>(d, ah, al, wh, wl, kb == 0);
    wg_commit();
    if (kb > 0) {
      wg_wait<1>();
      if (lane == 0) ring.release(q - 1);
    }
  }
  wg_wait<0>();
  acc_fence(d);
  if (RELEASE_LAST && lane == 0) ring.release(q - 1);
}

// ---------------------------------------------------------------------------------- the 128-row CTA
// The CTA shape of k_gemm_tc, k_tconv_tc and k_gru_step_tc (ws_cta below) and of k_attn_tc (DESIGN §2): a producer
// warpgroup that gives its registers away and two consumer warpgroups of 64 rows each.  At 384 threads ptxas
// compiles the consumers under 168 registers, whatever setmaxnreg raises them to at run time.
constexpr int BM = 128, BK = 64;                       // tile rows; k-block depth (one 128B swizzle row of fp16)
constexpr int WS_THREADS = 384;
constexpr int CONSUMER_WARPS = 8;
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;

// One ring stage of a 128 x BN split16 tile: [A hi | A lo | W hi | W lo], each plane a 64-deep k-block (one 128B
// swizzle row per tile row), A 128 rows and W BN rows; two consumer warpgroups take 64 A rows each.  STAGES stages
// followed by the ring's barriers, plus the alignment slack of smem_pad1024.
template <int BN_, int STAGES_>
struct StageLayout {
  static constexpr int BN = BN_, STAGES = STAGES_;
  static constexpr int A_BYTES = BM * BK * 2;         // one plane of the A tile (16 KB)
  static constexpr int W_BYTES = BN * BK * 2;         // one plane of the W tile
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * W_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256 + 1024;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget");
  // the shared-memory addresses of slot s's planes, the A planes from byte a_off of the tile on; smem: the first stage
  struct Planes { uint32_t ah, al, wh, wl; };
  __device__ __forceinline__ static Planes planes(const uint8_t* smem, int s, uint32_t a_off = 0) {
    const uint32_t ah = smem_u32(smem + s * STAGE_BYTES) + a_off, al = ah + A_BYTES;
    const uint32_t wh = smem_u32(smem + s * STAGE_BYTES) + 2 * A_BYTES, wl = wh + W_BYTES;
    return {ah, al, wh, wl};
  }
};

// sum over the 4 lanes of a quad (the lanes that hold one accumulator row)
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// fp32 pair -> packed fp16 hi pair and lo pair (x = hi + lo to ~22 bits)
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h2 = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h2);
  const __half2 l2 = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h2);
  lo = *reinterpret_cast<const uint32_t*>(&l2);
}
// split2 into element pair o of two fp16 planes (o even)
__device__ __forceinline__ void store_split2(__half* hi, __half* lo, int64_t o, float x0, float x1) {
  uint32_t h, l;
  split2(x0, x1, h, l);
  *reinterpret_cast<uint32_t*>(hi + o) = h;
  *reinterpret_cast<uint32_t*>(lo + o) = l;
}

// Debug timeline (mldb_debug_timeline): when `tl` is non-null, lane 0 of the calling warp of CTA 0 stores
// (tag | aux << 24, SM clock) into its warp's private slot array (plain stores, no atomics: ~10 cycles per
// event).  Layout: [32 warps][TL_CAPW events][2]; `n` is the warp's own event counter (a register).
constexpr int TL_CAPW = 512;
__device__ __forceinline__ void tl_event(long long* tl, int& n, int tag, int aux = 0) {
  if (tl != nullptr && blockIdx.x == 0 && (threadIdx.x & 31) == 0 && n < TL_CAPW) {
    long long* e = tl + ((size_t)(threadIdx.x >> 5) * TL_CAPW + n) * 2;
    e[0] = (long long)tag | ((long long)aux << 24);
    e[1] = clock64();
    ++n;
  }
}
long long* mldb_timeline_buffer();   // debug.cu: the device buffer while a timeline is being recorded, else nullptr

// A consumer thread of ws_cta: its warp and lane, its warpgroup's 64 rows of the tile (cw) and its column offset
// inside an 8-column group (cp).  Its accumulator fragment holds tile rows row() and row() + 8.
struct TileThread {
  int warp, lane, cw, cp;
  __device__ __forceinline__ int row() const { return cw * 64 + (warp & 3) * 16 + (lane >> 2); }
};

// The tiles this CTA runs of a persistent grid over ntiles tiles: CTA c takes tiles c, c + #CTAs, ...
__device__ __forceinline__ int persistent_count(int ntiles) {
  return (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
}

// The whole body of a kernel launched with WS_THREADS threads and L::SMEM_BYTES of dynamic shared memory: L::STAGES
// stages of the StageLayout L, then the ring's barriers.  Thread 0 sets up the ring and prefetches the tensor maps
// m0..m3.  After the PDL wait, warpgroup 0 drops to PRODUCER_REGS registers and its warp 0 feeds the ring
// (ring_feed); warpgroups 1 and 2 raise themselves to CONSUMER_REGS and each multiply 64 rows of every tile
// (ring_mma).  Every tile is kblocks k-blocks deep.  The kernel supplies
//   count()                   how many tiles this CTA runs (called once, in the prologue);
//   tile(j)                   the j-th of them, in whatever form load, epilogue and before take it;
//   load(t, kb, planes, full) tile t's loads of k-block kb into the stage at `planes` (one elected lane);
//   epilogue(t, d, th)        the consumers' epilogue on their [64 x L::BN] accumulator fragment d;
//   before(t, j, ntiles, kb)  run by the producer's elected lane before it arms k-block kb of t, the j-th of the
//                             CTA's ntiles tiles.
// RELEASE_LAST as in ring_mma.  tl: the debug timeline (nullptr: none), with tags 40 at entry, 41 after the PDL
// wait, 1 as the producer starts a tile, 2 / 4 / 5 as the consumers start its MMAs, have its accumulator and have
// run its epilogue, and 42 at the consumers' exit.  tl and kblocks are taken by reference, so that a kernel
// parameter is read where it is used: a copy made at the call is computed ahead of the prologue, and nvcc then
// schedules the whole kernel differently.
template <class L, bool RELEASE_LAST = true, class Count, class Tile, class Load, class Epilogue, class Before = NoOp>
__device__ __forceinline__ void ws_cta(const CUtensorMap& m0, const CUtensorMap& m1, const CUtensorMap& m2,
                                       const CUtensorMap& m3, long long* const& tl, const int& kblocks, Count&& count, Tile&& tile,
                                       Load&& load, Epilogue&& epilogue, Before&& before = {}) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem + L::STAGES * L::STAGE_BYTES);
  const Ring<L::STAGES> ring{bar_full, bar_full + L::STAGES};
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // provably warp-uniform
  int tl_n = 0;                                     // debug-timeline event counter of this warp
  tl_event(tl, tl_n, 40);
  const int ntiles = count();
  if (threadIdx.x == 0) {
    ring.init(CONSUMER_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&m0); tma_prefetch_desc(&m1); tma_prefetch_desc(&m2); tma_prefetch_desc(&m3);
  }
  pdl_trigger();               // let the next kernel's prologue overlap our tail
  __syncthreads();
  pdl_wait();                  // everything below touches the previous kernel's outputs
  tl_event(tl, tl_n, 41);

  if (warp < 4) {
    reg_dec<PRODUCER_REGS>();
    if (warp != 0) return;
    int q = 0;                 // ring position, across tiles
    for (int j = 0; j < ntiles; ++j) {
      const auto t = tile(j);
      tl_event(tl, tl_n, 1, j);
      ring_feed(ring, q, kblocks, L::STAGE_BYTES,
                [&](int kb, int s, uint32_t full) { load(t, kb, L::planes(smem, s), full); },
                [&](int kb) { before(t, j, ntiles, kb); });
    }
    return;
  }
  reg_inc<CONSUMER_REGS>();
  const TileThread th{warp, lane, (warp >> 2) - 1, 2 * (lane & 3)};
  float d[L::BN / 2];
  int q = 0;
  for (int j = 0; j < ntiles; ++j) {
    const auto t = tile(j);
    tl_event(tl, tl_n, 2, j);
    ring_mma<L::BN, RELEASE_LAST>(d, ring, q, kblocks, lane, [&](int, int s, uint32_t& ah, uint32_t& al, uint32_t& wh, uint32_t& wl) {
      const auto pl = L::planes(smem, s, th.cw * (64 * 128));             // the warpgroup's 64 A rows
      ah = pl.ah; al = pl.al; wh = pl.wh; wl = pl.wl;
    });
    tl_event(tl, tl_n, 4, j);
    epilogue(t, d, th);
    tl_event(tl, tl_n, 5, j);
  }
  tl_event(tl, tl_n, 42);
}

// ---------------------------------------------------------------------------------- host: tensor maps
// both planes of a split16 buffer 16-byte aligned (TMA base addresses, 16-byte accesses)
inline bool planes_aligned16(const ActBuf& b) { return ((uintptr_t)b.hi & 15) == 0 && ((uintptr_t)b.lo() & 15) == 0; }

typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                        CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                        CUtensorMapFloatOOBfill);

// The driver's cuTensorMapEncodeTiled, looked up once per process.  nullptr (and mldb_last_error() set) when the
// driver does not provide it.
inline PFN_tmapEncodeTiled tmap_encoder() {
  static const PFN_tmapEncodeTiled fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    const cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    return e == cudaSuccess && q == cudaDriverEntryPointSuccess ? (PFN_tmapEncodeTiled)p : nullptr;
  }();
  if (!fn) mldb_set_err("cuTensorMapEncodeTiled is not available from the driver");
  return fn;
}

// A tensor map of one split16 plane (fp16, columns contiguous): boxes of 64 columns (one 128B swizzle row) x
// box[1] rows, SWIZZLE_128B, L2 256B promotion, and elements outside the plane zero-filled - so M and N need not
// be tile multiples, and a box never brings in rows of another sequence (DESIGN §2).  dims / strides / box are
// innermost first; rank <= 5.  estr: the traversal stride of each dimension (nullptr: all 1); a box then holds
// ceil(box[i] / estr[i]) elements along dimension i, every estr[i]-th one from the load's start coordinate.
// false: encoding failed and mldb_last_error() names the plane.
inline bool encode_plane_map(CUtensorMap* m, const __half* base, int rank, const cuuint64_t* dims,
                             const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t* estr = nullptr) {
  const PFN_tmapEncodeTiled encode = tmap_encoder();
  if (!encode) return false;
  const cuuint32_t ones[5] = {1, 1, 1, 1, 1};
  const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, (void*)base, dims, strides, box,
                            estr ? estr : ones, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    std::string shape;
    for (int i = rank - 1; i >= 0; --i) shape += std::to_string(dims[i]) + (i ? " x " : "");
    char buf[96];
    snprintf(buf, sizeof buf, "(CUresult %d): fp16 plane at %p", (int)r, (const void*)base);
    mldb_set_err("cuTensorMapEncodeTiled failed " + std::string(buf) + ", [" + shape + "], box " +
                 std::to_string(box[1]) + " rows");
  }
  return r == CUDA_SUCCESS;
}
// a [rows, cols] plane
inline bool make_map(CUtensorMap* m, const __half* base, int rows, int cols, int box_rows) {
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)cols * sizeof(__half)};
  const cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  return encode_plane_map(m, base, 2, dims, strides, box);
}
// the same plane seen as [nseq, L, cols]: a box never reaches past its own sequence, rows >= L are zero-filled
inline bool make_seq_map(CUtensorMap* m, const __half* base, int nseq, int L, int cols, int box_rows) {
  const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)L, (cuuint64_t)nseq};
  const cuuint64_t strides[2] = {(cuuint64_t)cols * sizeof(__half), (cuuint64_t)L * cols * sizeof(__half)};
  const cuuint32_t box[3] = {64u, (cuuint32_t)box_rows, 1u};
  return encode_plane_map(m, base, 3, dims, strides, box);
}

// Snake order across the per-layer kernels: the GEMMs walk the token tiles upwards, attention and the fused FFN
// downwards, so every kernel starts on the rows its producer wrote LAST - those are the ones most likely to be
// still in L2.  MLDB_SNAKE=0 turns it off (A/B); read once per process.
inline int snake_order() {
  static const int on = [] { const char* e = getenv("MLDB_SNAKE"); return (e && !strcmp(e, "0")) ? 0 : 1; }();
  return on;
}

}  // namespace tc
