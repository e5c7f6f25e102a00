// Tensor-core multi-head attention for short sequences (L <= ~200 tokens, head_dim 64/128) in the
// split16 format.  One CTA per (sequence, head); Q, K, V head slices (hi and lo planes) are staged
// in shared memory, each warp owns 16-query-row tiles and walks the keys in chunks of 64 with an
// online (flash-style) fp32 softmax.  Both contractions use mma.sync.m16n8k16 (fp16 x fp16 -> fp32)
// with the same three-product scheme as the GEMMs:
//     S = Qh Kh^T + Ql Kh^T + Qh Kl^T,      O = Ph Vh + Pl Vh + Ph Vl
// (P = exp(S - max) is re-split into hi/lo fp16 in registers).  The sequences here are far too
// short for a wgmma tile per head (a 128-row MMA would be >35 % padding at L = 79 and the PV
// operand would need an MN-major descriptor per 64-wide head slice); legacy mma.sync tiles of
// 16 x 8 fit them exactly and attention is ~5 % of the path's FLOPs.
// Replaces the attention core of nn.MultiheadAttention (cross_attention.py:264-266, 330-338):
// scores scaled by 1/sqrt(head_dim), padded keys masked (-inf), softmax over keys, P @ V.
#include "ops.cuh"

namespace {

constexpr int AW_MAX = 8;        // warps per CTA: one per 16-row query tile, at most 8
constexpr int KCHUNK = 64;       // keys per online-softmax chunk

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  __half2 h = __halves2half2(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int HD>
__global__ void __launch_bounds__(AW_MAX * 32) k_attn_mma(const AttnArgs a) {
  constexpr int PITCH = HD + 8;              // halves per smem row (144 B / 272 B: conflict-free ldmatrix)
  constexpr int NT_D = HD / 8;               // n8 tiles across the head dimension
  constexpr int KS = HD / 16;                // k16 steps across the head dimension
  extern __shared__ __align__(16) uint8_t sm_raw[];
  const int s = blockIdx.x / a.heads, h = blockIdx.x % a.heads;
  const int Lq = a.Lq, Lk = a.Lk;
  const int LqP = (Lq + 15) & ~15, LkP = (Lk + 15) & ~15;
  int nk = Lk;
  if (a.lengths) nk = min(Lk, a.kv_prefix + a.lengths[a.len_mod > 0 ? (a.seq0 + s) % a.len_mod : s]);
  __half* Qh = reinterpret_cast<__half*>(sm_raw);
  __half* Ql = Qh + (size_t)LqP * PITCH;
  __half* Kh = Ql + (size_t)LqP * PITCH;
  __half* Kl = Kh + (size_t)LkP * PITCH;
  __half* Vh = Kl + (size_t)LkP * PITCH;
  __half* Vl = Vh + (size_t)LkP * PITCH;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nthreads = blockDim.x, AW = blockDim.x >> 5;
  pdl_trigger();
  pdl_wait();

  // ---- stage the head slices with cp.async (16-byte LDGSTS, no register staging): every copy of
  // the CTA is in flight at once, so the whole 46-69 KB working set costs about one L2 round trip.
  // Rows beyond L are zero-filled (src-size 0).
  constexpr int VPR = HD / 8;                // 16-byte vectors per row
  {
    const uint32_t sQh = (uint32_t)__cvta_generic_to_shared(Qh), sQl = (uint32_t)__cvta_generic_to_shared(Ql);
    for (int i = tid; i < LqP * VPR; i += nthreads) {
      const int r = i / VPR, c = i - r * VPR;
      const int rc = r < Lq ? r : Lq - 1;
      const int64_t o = ((int64_t)s * Lq + rc) * a.q.cols + a.q_col0 + h * HD + c * 8;
      const uint32_t so = (uint32_t)(r * PITCH + c * 8) * 2, nb = r < Lq ? 16u : 0u;
      cp_async16(sQh + so, a.q.hi + o, nb);
      cp_async16(sQl + so, a.q.lo() + o, nb);
    }
    const uint32_t sKh = (uint32_t)__cvta_generic_to_shared(Kh), sKl = (uint32_t)__cvta_generic_to_shared(Kl);
    const uint32_t sVh = (uint32_t)__cvta_generic_to_shared(Vh), sVl = (uint32_t)__cvta_generic_to_shared(Vl);
    for (int i = tid; i < LkP * VPR; i += nthreads) {
      const int r = i / VPR, c = i - r * VPR;
      const int rc = r < Lk ? r : Lk - 1;
      const int64_t base = ((int64_t)s * Lk + rc) * a.kv.cols + h * HD + c * 8;
      const uint32_t so = (uint32_t)(r * PITCH + c * 8) * 2, nb = r < Lk ? 16u : 0u;
      cp_async16(sKh + so, a.kv.hi + base + a.k_col0, nb);
      cp_async16(sKl + so, a.kv.lo() + base + a.k_col0, nb);
      cp_async16(sVh + so, a.kv.hi + base + a.v_col0, nb);
      cp_async16(sVl + so, a.kv.lo() + base + a.v_col0, nb);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
  }
  __syncthreads();

  const float scale = rsqrtf((float)HD);
  const int g = lane >> 2, t = lane & 3;
  // ldmatrix row/col offsets: x4 = four 8x8 tiles; lane l supplies the row address of tile l/8
  const int lrow = (lane & 7) + ((lane >> 3) & 1) * 8;   // A operand / V^T: rows 0..15
  const int lcol = (lane >> 4) * 8;                       // second pair of tiles: +8 columns

  for (int qt = warp; qt * 16 < Lq; qt += AW) {
    const int q0 = qt * 16;
    float o_acc[NT_D][4];
#pragma unroll
    for (int j = 0; j < NT_D; ++j) { o_acc[j][0] = o_acc[j][1] = o_acc[j][2] = o_acc[j][3] = 0.0f; }
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.0f, 0.0f};

    for (int kc = 0; kc < nk; kc += KCHUNK) {
      // ---------------- S = Q K^T for up to 64 keys (8 n8 tiles)
      float sc[8][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) { sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.0f; }
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        uint32_t qh[4], ql[4];
        const uint32_t qoff = (uint32_t)((q0 + lrow) * PITCH + ks * 16 + lcol) * 2;
        ldsm_x4(qh, (uint32_t)__cvta_generic_to_shared(Qh) + qoff);
        ldsm_x4(ql, (uint32_t)__cvta_generic_to_shared(Ql) + qoff);
#pragma unroll
        for (int jp = 0; jp < 4; ++jp) {              // pairs of key tiles (16 keys)
          if (kc + jp * 16 < nk) {
            // K tile rows = keys, cols = d: non-transposed ldmatrix gives the col-major B fragment.
            // tiles: (keys 0-7, d 0-7), (keys 0-7, d 8-15), (keys 8-15, d 0-7), (keys 8-15, d 8-15)
            const int krow = kc + jp * 16 + (lane & 7) + (lane >> 4) * 8;
            const int kcol = ks * 16 + ((lane >> 3) & 1) * 8;
            const uint32_t koff = (uint32_t)(krow * PITCH + kcol) * 2;
            uint32_t kh[4], kl[4];
            ldsm_x4(kh, (uint32_t)__cvta_generic_to_shared(Kh) + koff);
            ldsm_x4(kl, (uint32_t)__cvta_generic_to_shared(Kl) + koff);
            mma16816(sc[2 * jp], ql, kh[0], kh[1]);
            mma16816(sc[2 * jp], qh, kl[0], kl[1]);
            mma16816(sc[2 * jp], qh, kh[0], kh[1]);
            mma16816(sc[2 * jp + 1], ql, kh[2], kh[3]);
            mma16816(sc[2 * jp + 1], qh, kl[2], kl[3]);
            mma16816(sc[2 * jp + 1], qh, kh[2], kh[3]);
          }
        }
      }
      // ---------------- online softmax (rows g and g+8 of the tile)
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = kc + j * 8 + 2 * t + (e & 1);
          const float v = key < nk ? sc[j][e] * scale : -INFINITY;
          sc[j][e] = v;
          mx[e >> 1] = fmaxf(mx[e >> 1], v);
        }
      }
      float corr[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float m_new = fmaxf(m_run[r], mx[r]);
        corr[r] = (m_run[r] == -INFINITY) ? 0.0f : expf(m_run[r] - m_new);
        m_run[r] = m_new;
        l_run[r] *= corr[r];
      }
#pragma unroll
      for (int j = 0; j < NT_D; ++j) {
        o_acc[j][0] *= corr[0]; o_acc[j][1] *= corr[0];
        o_acc[j][2] *= corr[1]; o_acc[j][3] *= corr[1];
      }
      float ls[2] = {0.0f, 0.0f};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float p = (sc[j][e] == -INFINITY) ? 0.0f : expf(sc[j][e] - m_run[e >> 1]);
          sc[j][e] = p;
          ls[e >> 1] += p;
        }
      }
      l_run[0] += ls[0];
      l_run[1] += ls[1];
      // ---------------- O += P V   (16 keys per k16 step)
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        if (kc + jp * 16 < nk) {
          uint32_t ph[4], pl[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            // A fragment regs: a0 (row g, k 2t..), a1 (row g+8), a2 (row g, k 8+2t..), a3 (row g+8)
            const float x0 = sc[2 * jp + (e >> 1)][(e & 1) * 2], x1 = sc[2 * jp + (e >> 1)][(e & 1) * 2 + 1];
            __half h0, l0, h1, l1;
            split_f32(x0, h0, l0);
            split_f32(x1, h1, l1);
            ph[e] = pack_h2(h0, h1);
            pl[e] = pack_h2(l0, l1);
          }
#pragma unroll
          for (int dp = 0; dp < NT_D / 2; ++dp) {     // pairs of d tiles (16 columns)
            // V rows = keys (k), cols = d (n): transposed ldmatrix gives the col-major B fragment.
            // tiles: (keys 0-7, d 0-7), (keys 8-15, d 0-7), (keys 0-7, d 8-15), (keys 8-15, d 8-15)
            const uint32_t voff = (uint32_t)((kc + jp * 16 + lrow) * PITCH + dp * 16 + lcol) * 2;
            uint32_t vh[4], vl[4];
            ldsm_x4_t(vh, (uint32_t)__cvta_generic_to_shared(Vh) + voff);
            ldsm_x4_t(vl, (uint32_t)__cvta_generic_to_shared(Vl) + voff);
            mma16816(o_acc[2 * dp], pl, vh[0], vh[1]);
            mma16816(o_acc[2 * dp], ph, vl[0], vl[1]);
            mma16816(o_acc[2 * dp], ph, vh[0], vh[1]);
            mma16816(o_acc[2 * dp + 1], pl, vh[2], vh[3]);
            mma16816(o_acc[2 * dp + 1], ph, vl[2], vl[3]);
            mma16816(o_acc[2 * dp + 1], ph, vh[2], vh[3]);
          }
        }
      }
    }
    // ---------------- normalise and store (split16)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float inv[2] = {1.0f / l_run[0], 1.0f / l_run[1]};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int qi = q0 + g + r * 8;
      if (qi < Lq) {
        const int64_t ob = ((int64_t)s * Lq + qi) * a.out.cols + h * HD + 2 * t;
#pragma unroll
        for (int j = 0; j < NT_D; ++j) {
          __half h0, l0, h1, l1;
          split_f32(o_acc[j][2 * r] * inv[r], h0, l0);
          split_f32(o_acc[j][2 * r + 1] * inv[r], h1, l1);
          *reinterpret_cast<uint32_t*>(a.out.hi + ob + j * 8) = pack_h2(h0, h1);
          *reinterpret_cast<uint32_t*>(a.out.lo() + ob + j * 8) = pack_h2(l0, l1);
        }
      }
    }
  }
}

template <int HD>
size_t attn_smem(const AttnArgs& a) {
  const int LqP = (a.Lq + 15) & ~15, LkP = (a.Lk + 15) & ~15;
  return (size_t)(2 * LqP + 4 * LkP) * (HD + 8) * sizeof(__half);
}

}  // namespace

bool mma_attention_supported(const AttnArgs& a) {
  if (a.hd != 64 && a.hd != 128) return false;
  if (a.Lk < 8) return false;                                  // 1-2 memory tokens: CUDA-core kernel
  if ((a.q.cols % 8) || (a.kv.cols % 8) || (a.q_col0 % 8) || (a.k_col0 % 8) || (a.v_col0 % 8)) return false;
  const size_t smem = a.hd == 64 ? attn_smem<64>(a) : attn_smem<128>(a);
  return smem <= 227 * 1024;
}

void mma_attention_init() {
  cudaFuncSetAttribute(k_attn_mma<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  cudaFuncSetAttribute(k_attn_mma<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
}

void mma_attention(const AttnArgs& a, cudaStream_t st) {
  const int qtiles = (a.Lq + 15) / 16;
  const int nw = qtiles < AW_MAX ? qtiles : AW_MAX;     // L = 79 -> 5 warps, one tile each
  if (a.hd == 64) launch_pdl(k_attn_mma<64>, dim3(a.nseq * a.heads), dim3(nw * 32), attn_smem<64>(a), st, a);
  else launch_pdl(k_attn_mma<128>, dim3(a.nseq * a.heads), dim3(nw * 32), attn_smem<128>(a), st, a);
}
