// Row LayerNorm of the text towers on the fp32 residual stream: CLIP's pre-norm LN1 / LN2 and final LN, fused with the
// token + position embedding for layer 0 and with the eos-row gather of pooled mode; BERT's post-norm LNs (written
// back into the stream) and its embedding LN.
// One warp per row, the row in registers (d / 32 floats per lane, float4 loads), exact two-pass statistics with
// warp shuffles and no shared memory; the output is the split16 A operand of the next GEMM and/or fp32.
#include "ops.cuh"

namespace {

// position of the pooled token of sequence s: HF CLIPTextTransformer (first id == eos_id, or 0 when absent;
// argmax(ids) under the legacy eos_token_id == 2, first maximum on ties)
__device__ __forceinline__ int eos_position(const int64_t* ids, int L, int eos_id, int lane) {
  if (eos_id == 2) {
    int64_t best = INT64_MIN;
    int at = 0;
    for (int t = lane; t < L; t += 32) {
      const int64_t v = (int64_t)(int32_t)ids[t];         // HF casts the ids to int32 before argmax
      if (v > best) { best = v; at = t; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const int64_t ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oa = __shfl_xor_sync(0xffffffffu, at, o);
      if (ob > best || (ob == best && oa < at)) { best = ob; at = oa; }
    }
    return at;
  }
  for (int t0 = 0; t0 < L; t0 += 32) {
    const int t = t0 + lane;
    const unsigned m = __ballot_sync(0xffffffffu, t < L && (int32_t)ids[t] == eos_id);
    if (m) return t0 + __ffs(m) - 1;
  }
  return 0;
}

template <int NV>   // float4 vectors per lane: d = 128 * NV
__global__ void __launch_bounds__(256) k_text_ln(const TextLnArgs a) {
  const int r = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= a.M) return;
  constexpr int D = 128 * NV;
  float v[NV][4];
  int64_t irow = r;
  if (a.mode == TEXT_LN_EOS) irow = (int64_t)r * a.L + eos_position(a.ids + (int64_t)r * a.L, a.L, a.eos_id, lane);
  if (a.mode == TEXT_LN_EMBED || a.mode == TEXT_LN_EMBED_LN) {
    const int64_t id = a.ids[r];
    const bool ok = id >= 0 && id < a.vocab;            // never read outside the table: a bad id is a NaN row
    const float* te = a.tok + (ok ? id : 0) * D;
    const float* pe = a.pos + (int64_t)(r % a.L) * D;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int n = 4 * (lane + 32 * i);
      float4 t = __ldg(reinterpret_cast<const float4*>(te + n));
      const float4 p = __ldg(reinterpret_cast<const float4*>(pe + n));
      if (a.type0) {                                     // BERT: (word + token_type) + position, torch's order
        const float4 y = __ldg(reinterpret_cast<const float4*>(a.type0 + n));
        t.x += y.x; t.y += y.y; t.z += y.z; t.w += y.w;
      }
      v[i][0] = t.x + p.x; v[i][1] = t.y + p.y; v[i][2] = t.z + p.z; v[i][3] = t.w + p.w;
      if (!ok) v[i][0] = v[i][1] = v[i][2] = v[i][3] = __int_as_float(0x7fc00000);
      if (a.mode == TEXT_LN_EMBED)
        *reinterpret_cast<float4*>(a.x + (int64_t)r * D + n) = make_float4(v[i][0], v[i][1], v[i][2], v[i][3]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 t = *reinterpret_cast<const float4*>(a.x + irow * D + 4 * (lane + 32 * i));
      v[i][0] = t.x; v[i][1] = t.y; v[i][2] = t.z; v[i][3] = t.w;
    }
  }
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += (v[i][0] + v[i][1]) + (v[i][2] + v[i][3]);
  const float mean = warp_sum(s) * (1.0f / D);
  float q = 0.0f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float t = v[i][k] - mean; q = fmaf(t, t, q); }
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + a.eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int n = 4 * (lane + 32 * i);
    const float4 g = __ldg(reinterpret_cast<const float4*>(a.gamma + n)), b = __ldg(reinterpret_cast<const float4*>(a.beta + n));
    const float y0 = fmaf((v[i][0] - mean) * rstd, g.x, b.x), y1 = fmaf((v[i][1] - mean) * rstd, g.y, b.y);
    const float y2 = fmaf((v[i][2] - mean) * rstd, g.z, b.z), y3 = fmaf((v[i][3] - mean) * rstd, g.w, b.w);
    if (a.out.hi) {
      __half h0, l0, h1, l1, h2, l2, h3, l3;
      split_f32(y0, h0, l0); split_f32(y1, h1, l1); split_f32(y2, h2, l2); split_f32(y3, h3, l3);
      const __half2 hh[2] = {__halves2half2(h0, h1), __halves2half2(h2, h3)};
      const __half2 ll[2] = {__halves2half2(l0, l1), __halves2half2(l2, l3)};
      const int64_t o = (int64_t)r * a.out.cols + n;
      *reinterpret_cast<uint2*>(a.out.hi + o) = *reinterpret_cast<const uint2*>(hh);
      *reinterpret_cast<uint2*>(a.out.lo() + o) = *reinterpret_cast<const uint2*>(ll);
    }
    if (a.out_f32) *reinterpret_cast<float4*>(a.out_f32 + (int64_t)r * D + n) = make_float4(y0, y1, y2, y3);
  }
}

}  // namespace

bool text_ln_supported(int d) { return d > 0 && d % 128 == 0 && d <= 1024; }

void text_ln(const TextLnArgs& a, cudaStream_t st) {
  const dim3 grid((unsigned)((a.M + 7) / 8));           // 8 warps (rows) per block
  switch (a.d / 128) {
    case 1: k_text_ln<1><<<grid, 256, 0, st>>>(a); break;
    case 2: k_text_ln<2><<<grid, 256, 0, st>>>(a); break;
    case 3: k_text_ln<3><<<grid, 256, 0, st>>>(a); break;
    case 4: k_text_ln<4><<<grid, 256, 0, st>>>(a); break;
    case 5: k_text_ln<5><<<grid, 256, 0, st>>>(a); break;
    case 6: k_text_ln<6><<<grid, 256, 0, st>>>(a); break;
    case 7: k_text_ln<7><<<grid, 256, 0, st>>>(a); break;
    default: k_text_ln<8><<<grid, 256, 0, st>>>(a); break;
  }
}
