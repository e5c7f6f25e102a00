// Multi-head attention core on wgmma / TMA for the split16 activation format.
// Replaces the attention core of nn.MultiheadAttention (cross_attention.py:264-266, 330-338):
// scores scaled by 1/sqrt(head_dim), padded keys masked (-inf), softmax over keys, P @ V - for
// every shape the sampling path uses: Lq in 1.., Lk in 1..256 (denoiser 79 / 3 tokens, VAE 196 / 198
// frames, 1-2 memory tokens), head_dim 64 or 128.  Causal self-attention (the CLIP text tower): query i sees
// keys j <= i; the key blocks that lie wholly above a query tile's diagonal are neither loaded nor multiplied.
//
// Work item = (sequence, head, 64-row query tile) = one warpgroup's MMA height.  A CTA (one per SM,
// persistent) runs TWO independent pipelines, each a consumer warpgroup with its own Q buffer and
// K / V ring and its own TMA warp in the producer warpgroup; while one warpgroup is in its softmax the
// other one's MMAs keep the tensor cores busy.  Keys are processed in blocks of 64 (the last block
// padded to a multiple of 16 with zero rows, never with the next sequence's keys):
//   S[:, kb]  = Q K_kb^T            M = 64, N = 64, K = head_dim            (A, B K-major in shared memory)
//   P         = exp2(scale*(S - max))  two exact passes over the WHOLE score row, which lives in
//                                   registers (<= 256 columns) - no online rescaling
//   O        += P[:, kb] V_kb       M = 64, N = 64 per 64-wide slice of the head, K = 64 | rem
//                                   (A = P from registers: the accumulator layout of 16 score columns IS
//                                   the register-operand layout of a 16-deep k-step; B = V_kb exactly as
//                                   TMA delivers the [keys x d] box: an MN-major operand, no transpose)
// every product in the 3-term split-fp16 form (hi.hi + lo.hi + hi.lo, fp32 accumulation).
#include "ops.cuh"
#include "tc_common.cuh"

namespace {
using namespace tc;

constexpr int KBLK = 64;                  // keys per block
constexpr int QROWS = 64;                 // query rows per item
constexpr int MAX_KB = 4;                 // key blocks of the longest score row (256 keys)
constexpr int PIPE_BYTES = 96 * 1024;     // shared memory of one pipeline: Q tile + K / V ring
constexpr int MAX_RS = 5;                 // ring slots (head_dim 64: 5 x 16 KB, head_dim 128: 2 x 32 KB)
constexpr int SMEM_BYTES = 2 * PIPE_BYTES + 256 + 1024;   // + barriers + alignment slack

struct AtcParams {
  int nseq, heads, Lq, Lk;
  int n_qt;                // 64-row query tiles per (sequence, head)
  int nkb, rem;            // key blocks; keys (multiple of 16) in the last block
  int q_col0, k_col0, v_col0;
  const int32_t* lengths; int kv_prefix, len_mod, seq0;
  __half* out_hi; __half* out_lo; int ld_out;
  float scale_log2e;       // log2(e) / sqrt(head_dim)
  long long* tl;           // debug timeline (nullptr normally)
  int reverse;             // walk the items from the last one down (see tc_attention)
  int items, heads_log2;   // nseq * heads * n_qt; log2(heads) or -1
};

struct Item { int s, h, qt; };
// key blocks item `it` needs: all of them, or (causal) the blocks up to its query tile's diagonal (KBLK == QROWS)
template <bool CAUSAL>
__device__ __forceinline__ int item_kblocks(const Item& it, int nkb) {
  return CAUSAL ? min(nkb, it.qt + 1) : nkb;
}
__device__ __forceinline__ Item decode_item(int item, const AtcParams& p) {
  Item it;
  if (p.reverse) item = p.items - 1 - item;
  // one query tile and a power-of-two head count (every shipped config) need no runtime division
  int sh = item;
  it.qt = 0;
  if (p.n_qt > 1) { sh = item / p.n_qt; it.qt = item - sh * p.n_qt; }
  if (p.heads_log2 >= 0) { it.s = sh >> p.heads_log2; it.h = sh & (p.heads - 1); }
  else { it.s = sh / p.heads; it.h = sh - it.s * p.heads; }
  return it;
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// CAUSAL is a template parameter so that the non-causal instantiations (the sampling path) carry no mask state.
// KB (2 or 4) sizes the score row held in registers: S[KB][32] is 32 * KB registers per thread, and the consumer
// warpgroup has 168 (three warpgroups per CTA), so the <= 128-key shapes (the denoiser's 79 tokens, the text
// tower's 77) compile without spills or serialised MMAs only when the row is sized for them.
template <int HD, bool CAUSAL, int KB>
__global__ void __launch_bounds__(WS_THREADS, 1)        // warps 0 / 1 of the producer warpgroup feed pipelines 0 / 1
k_attn_tc(const __grid_constant__ CUtensorMap tmQh, const __grid_constant__ CUtensorMap tmQl,
          const __grid_constant__ CUtensorMap tmKh, const __grid_constant__ CUtensorMap tmKl,    // 64-row boxes
          const __grid_constant__ CUtensorMap tmRh, const __grid_constant__ CUtensorMap tmRl,    // rem-row boxes
          const AtcParams p) {
  constexpr int NS = HD / 64;                         // 64-wide slices of the head dimension
  constexpr int TILE = KBLK * 128;                    // one [64 rows x 64 columns] swizzled tile (8 KB)
  constexpr int SLOT_BYTES = 2 * NS * TILE;           // [plane][slice] tiles of one key block; the Q tile has the same shape
  constexpr int SL_PLANE = NS * TILE;                 // plane stride inside a slot
  constexpr int RS = PIPE_BYTES / SLOT_BYTES - 1;     // ring slots next to the Q tile
  static_assert(KB >= 1 && KB <= MAX_KB, "score row");
  static_assert(RS >= 2 && RS <= MAX_RS, "ring depth");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * PIPE_BYTES);
  // pipeline g's barriers: its Q buffer's full and empty, then its K / V ring's RS full and RS empty.  Every empty
  // barrier takes one arrival per warp of the pipeline's consumer warpgroup.
  auto q_ring = [&](int g) { uint64_t* b = bars + g * (2 + 2 * RS); return Ring<1>{b, b + 1}; };
  auto kv_ring = [&](int g) { uint64_t* b = bars + g * (2 + 2 * RS) + 2; return Ring<RS>{b, b + RS}; };

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  int tl_n = 0;                                       // debug-timeline event counter of this warp
  tl_event(p.tl, tl_n, 40);                       // kernel entry
  const int nkb = p.nkb;
  if (threadIdx.x == 0) {
    for (int g = 0; g < 2; ++g) {
      q_ring(g).init(4);
      kv_ring(g).init(4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmQh); tma_prefetch_desc(&tmQl); tma_prefetch_desc(&tmKh); tma_prefetch_desc(&tmKl);
  }
  pdl_trigger();
  __syncthreads();
  pdl_wait();                                         // q|k|v come from the previous kernel
  tl_event(p.tl, tl_n, 41);                       // the previous kernel has completed

  const bool producer = warp < 4;
  const int g = producer ? (warp & 1) : (warp >> 2) - 1;    // pipeline of this warp
  uint8_t* const sQ = smem + g * PIPE_BYTES;
  uint8_t* const sR = sQ + SLOT_BYTES;
  const Ring<1> qr = q_ring(g);
  const Ring<RS> kvr = kv_ring(g);
  const int pid = (int)blockIdx.x * 2 + g, npipes = (int)gridDim.x * 2;
  const int nlocal = (p.items - pid + npipes - 1) / npipes;

  if (producer) {
    reg_dec<PRODUCER_REGS>();
    if (warp >= 2) return;
    // ------------------------------------------------------------------ TMA producer of pipeline g:
    // Q(j), the K blocks of item j, its V blocks - exactly the order the consumer takes them
    int rc = 0;                                       // ring position (K and V blocks, all items)
    for (int j = 0; j < nlocal; ++j) {
      const Item it = decode_item(pid + j * npipes, p);
      const int nkb_i = item_kblocks<CAUSAL>(it, nkb);
      qr.wait_empty(j);
      tl_event(p.tl, tl_n, 20, j);                                     // producer: Q buffer free, loads issued
      if (elect_one()) {
        const uint32_t full = qr.full_bar(j);
        mbar_expect_tx(full, (uint32_t)SLOT_BYTES);
        const uint32_t base = smem_u32(sQ);
        const int r0 = it.s * p.Lq + it.qt * QROWS;
#pragma unroll
        for (int sl = 0; sl < NS; ++sl) {
          tma_load_2d(base + sl * TILE, &tmQh, full, p.q_col0 + it.h * HD + sl * 64, r0);
          tma_load_2d(base + SL_PLANE + sl * TILE, &tmQl, full, p.q_col0 + it.h * HD + sl * 64, r0);
        }
      }
      __syncwarp();
      for (int kv = 0; kv < 2; ++kv) {
        const int col0 = (kv ? p.v_col0 : p.k_col0) + it.h * HD;
        for (int kb = 0; kb < nkb_i; ++kb, ++rc) {
          kvr.wait_empty(rc);
          if (elect_one()) {
            const bool last = kb == nkb - 1;
            const int rows = last ? p.rem : KBLK;
            const uint32_t full = kvr.full_bar(rc);
            mbar_expect_tx(full, (uint32_t)(2 * NS * rows * 128));
            const uint32_t base = smem_u32(sR + (rc % RS) * SLOT_BYTES);
            // the last block's rows past Lk would be the next sequence's first keys: its [seq, key, col] map
            // zero-fills them, since P = 0 times a non-finite V is NaN
#pragma unroll
            for (int sl = 0; sl < NS; ++sl) {
              if (last) {
                tma_load_3d(base + sl * TILE, &tmRh, full, col0 + sl * 64, kb * KBLK, it.s);
                tma_load_3d(base + SL_PLANE + sl * TILE, &tmRl, full, col0 + sl * 64, kb * KBLK, it.s);
              } else {
                tma_load_2d(base + sl * TILE, &tmKh, full, col0 + sl * 64, it.s * p.Lk + kb * KBLK);
                tma_load_2d(base + SL_PLANE + sl * TILE, &tmKl, full, col0 + sl * 64, it.s * p.Lk + kb * KBLK);
              }
            }
          }
          __syncwarp();
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumer warpgroup of pipeline g
  reg_inc<CONSUMER_REGS>();
  const int cp = 2 * (lane & 3);                      // column offset inside an 8-column group
  const int row = (warp & 3) * 16 + (lane >> 2);      // this thread's first query row (the second is row + 8)
  const float sc = p.scale_log2e;
  float S[KB][32];                                    // the score row: [key block][accumulator fragment of 64 keys]
  float O[NS][32];
  int rc = 0;
  for (int j = 0; j < nlocal; ++j) {
    const Item it = decode_item(pid + j * npipes, p);
    const int nkb_i = item_kblocks<CAUSAL>(it, nkb);
    int nk = p.Lk;
    if (p.lengths) nk = min(p.Lk, p.kv_prefix + p.lengths[p.len_mod > 0 ? (p.seq0 + it.s) % p.len_mod : it.s]);
    // valid keys of this thread's two query rows (causal: keys j <= i)
    const int q0 = it.qt * QROWS + row;
    const int nk0 = CAUSAL ? min(nk, q0 + 1) : nk, nk1 = CAUSAL ? min(nk, q0 + 9) : nk;
    qr.wait_full(j);
    tl_event(p.tl, tl_n, 22, j);                                       // Q(j) landed
    // ---- S = Q K^T, block by block; a block's ring slot is freed when the NEXT block's MMAs have been issued
    const uint32_t qbase = smem_u32(sQ);
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      if (kb < nkb_i) {
        kvr.wait_full(rc + kb);
        const uint32_t kbase = smem_u32(sR + ((rc + kb) % RS) * SLOT_BYTES);
        wg_fence();
#pragma unroll
        for (int sl = 0; sl < NS; ++sl)               // one k-block per 64-wide slice of the head dimension
          kblock_ss<64>(S[kb], qbase + sl * TILE, qbase + SL_PLANE + sl * TILE, kbase + sl * TILE,
                        kbase + SL_PLANE + sl * TILE, sl == 0);
        wg_commit();
        if (kb > 0) {
          wg_wait<1>();
          if (lane == 0) kvr.release(rc + kb - 1);
        }
      }
    }
    wg_wait<0>();
    if (lane == 0) {
      kvr.release(rc + nkb_i - 1);
      qr.release(j);                                  // Q only feeds the scores
    }
    rc += nkb_i;
#pragma unroll
    for (int kb = 0; kb < KB; ++kb)
      if (kb < nkb_i) acc_fence(S[kb]);
    tl_event(p.tl, tl_n, 31, j);                                       // softmax: S(j) ready
    // ---- pass 1: row maxima over the valid keys (a row is spread over the 4 lanes of a quad)
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      if (kb < nkb_i) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = kb * KBLK + 8 * jj + cp + e;
            mx0 = fmaxf(mx0, key < nk0 ? S[kb][4 * jj + e] : -INFINITY);
            mx1 = fmaxf(mx1, key < nk1 ? S[kb][4 * jj + 2 + e] : -INFINITY);
          }
        }
      }
    }
    mx0 = quad_max(mx0); mx1 = quad_max(mx1);
    const float mc0 = (mx0 == -INFINITY) ? 0.0f : mx0 * sc, mc1 = (mx1 == -INFINITY) ? 0.0f : mx1 * sc;
    // ---- pass 2: P = exp2(sc * s - sc * max) (unnormalised, in place), fp32 row sums
    float sum0 = 0.0f, sum1 = 0.0f;
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      if (kb < nkb_i) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int key = kb * KBLK + 8 * jj + cp + e;
            float e0, e1;
            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(fmaf(S[kb][4 * jj + e], sc, -mc0)));
            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(fmaf(S[kb][4 * jj + 2 + e], sc, -mc1)));
            e0 = key < nk0 ? e0 : 0.0f;
            e1 = key < nk1 ? e1 : 0.0f;
            S[kb][4 * jj + e] = e0; S[kb][4 * jj + 2 + e] = e1;
            sum0 += e0; sum1 += e1;
          }
        }
      }
    }
    sum0 = quad_sum(sum0); sum1 = quad_sum(sum1);
    tl_event(p.tl, tl_n, 33, j);                                       // softmax: pass 2 done
    // ---- O = P V, block by block: P re-split to hi / lo fp16 A fragments, 16 keys per k-step.  Each block waits for
    // its MMAs before the next block's split: keeping a block in flight holds its A fragments live across the next
    // split, which at 168 registers makes ptxas serialise every wgmma of the kernel.
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      if (kb < nkb_i) {
        uint32_t ph[4][4], pl[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
#pragma unroll
          for (int i = 0; i < 4; ++i) split2(S[kb][8 * ks + 2 * i], S[kb][8 * ks + 2 * i + 1], ph[ks][i], pl[ks][i]);
        kvr.wait_full(rc + kb);
        const uint32_t vbase = smem_u32(sR + ((rc + kb) % RS) * SLOT_BYTES);
        const int nks = (kb == nkb - 1 ? p.rem : KBLK) / 16;           // rows beyond `rem` of the slot are stale
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          if (ks < nks) {
#pragma unroll
            for (int sl = 0; sl < NS; ++sl) {
              // next 16 keys of the MN-major V tile: +2048 B
              const uint64_t vh = make_desc(vbase + sl * TILE) + ks * 128, vl = make_desc(vbase + SL_PLANE + sl * TILE) + ks * 128;
              wgmma_rs_n64_tb(O[sl], pl[ks], vh, (kb | ks) != 0 ? 1u : 0u);
              wgmma_rs_n64_tb(O[sl], ph[ks], vl, 1u);
              wgmma_rs_n64_tb(O[sl], ph[ks], vh, 1u);
            }
          }
        }
        wg_commit();
        wg_wait<0>();
        if (lane == 0) kvr.release(rc + kb);
      }
    }
    rc += nkb_i;
#pragma unroll
    for (int sl = 0; sl < NS; ++sl) acc_fence(O[sl]);
    tl_event(p.tl, tl_n, 34, j);                                       // O(j) ready
    // ---- epilogue: O / sum -> split16 -> global
    const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
    const int qrow = it.qt * QROWS + row;
    const int64_t o0 = ((int64_t)it.s * p.Lq + qrow) * p.ld_out + it.h * HD + cp, o1 = o0 + (int64_t)8 * p.ld_out;
#pragma unroll
    for (int sl = 0; sl < NS; ++sl) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        uint32_t h, l;
        if (qrow < p.Lq) {
          split2(O[sl][4 * jj] * inv0, O[sl][4 * jj + 1] * inv0, h, l);
          *reinterpret_cast<uint32_t*>(p.out_hi + o0 + sl * 64 + 8 * jj) = h;
          *reinterpret_cast<uint32_t*>(p.out_lo + o0 + sl * 64 + 8 * jj) = l;
        }
        if (qrow + 8 < p.Lq) {
          split2(O[sl][4 * jj + 2] * inv1, O[sl][4 * jj + 3] * inv1, h, l);
          *reinterpret_cast<uint32_t*>(p.out_hi + o1 + sl * 64 + 8 * jj) = h;
          *reinterpret_cast<uint32_t*>(p.out_lo + o1 + sl * 64 + 8 * jj) = l;
        }
      }
    }
    tl_event(p.tl, tl_n, 35, j);                                       // epilogue done
  }
  tl_event(p.tl, tl_n, 42);                       // kernel exit
}

// launch geometry for a shape; false when it does not fit
bool plan_shape(const AttnArgs& a, AtcParams* p) {
  const int npad = (a.Lk + 15) & ~15;
  p->nkb = (npad + KBLK - 1) / KBLK;
  p->rem = npad - (p->nkb - 1) * KBLK;
  p->n_qt = (a.Lq + QROWS - 1) / QROWS;
  return p->nkb <= MAX_KB;
}

// the score row sized for the shape: up to 128 keys (the denoiser, the text tower) in KB = 2, longer rows in KB = 4
template <int HD, bool CAUSAL>
auto pick_kernel(int nkb) { return nkb <= 2 ? k_attn_tc<HD, CAUSAL, 2> : k_attn_tc<HD, CAUSAL, MAX_KB>; }

}  // namespace

bool tc_attention_init() {
  using Kernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, AtcParams);
  const Kernel kernels[] = {k_attn_tc<64, false, 2>, k_attn_tc<64, false, 4>, k_attn_tc<64, true, 2>, k_attn_tc<64, true, 4>,
                            k_attn_tc<128, false, 2>, k_attn_tc<128, false, 4>, k_attn_tc<128, true, 2>, k_attn_tc<128, true, 4>};
  for (Kernel k : kernels)
    if (!smem_opt_in(k, SMEM_BYTES, "k_attn_tc")) return false;
  return true;
}

bool tc_attention_supported(const AttnArgs& a) {
  if ((a.hd != 64 && a.hd != 128) || a.Lq < 1 || a.Lk < 1 || a.Lk > 256 || a.nseq < 1) return false;
  if (a.causal && a.Lq != a.Lk) return false;
  if ((a.q.cols % 8) || (a.kv.cols % 8) || (a.q_col0 % 8) || (a.k_col0 % 8) || (a.v_col0 % 8)) return false;
  if ((a.out.cols % 8) || ((uintptr_t)a.q.hi & 15) || ((uintptr_t)a.kv.hi & 15) || ((uintptr_t)a.out.hi & 15)) return false;
  if ((a.q.plane_stride % 8) || (a.kv.plane_stride % 8) || (a.out.plane_stride % 8)) return false;
  AtcParams p{};
  return plan_shape(a, &p);
}

bool tc_attention(const AttnArgs& a, int sm_count, cudaStream_t st) {
  AtcParams p{};
  if (!plan_shape(a, &p)) return false;
  CUtensorMap mQh, mQl, mKh, mKl, mRh, mRl;
  const bool ok = make_map(&mQh, a.q.hi, a.q.rows, a.q.cols, QROWS) && make_map(&mQl, a.q.lo(), a.q.rows, a.q.cols, QROWS) &&
                  make_map(&mKh, a.kv.hi, a.kv.rows, a.kv.cols, KBLK) && make_map(&mKl, a.kv.lo(), a.kv.rows, a.kv.cols, KBLK) &&
                  make_seq_map(&mRh, a.kv.hi, a.nseq, a.Lk, a.kv.cols, p.rem) &&
                  make_seq_map(&mRl, a.kv.lo(), a.nseq, a.Lk, a.kv.cols, p.rem);
  if (!ok) return false;
  p.nseq = a.nseq; p.heads = a.heads; p.Lq = a.Lq; p.Lk = a.Lk;
  p.q_col0 = a.q_col0; p.k_col0 = a.k_col0; p.v_col0 = a.v_col0;
  p.lengths = a.lengths; p.kv_prefix = a.kv_prefix; p.len_mod = a.len_mod; p.seq0 = a.seq0;
  p.out_hi = a.out.hi; p.out_lo = a.out.lo(); p.ld_out = a.out.cols;
  p.scale_log2e = 1.4426950408889634f / sqrtf((float)a.hd);
  p.tl = tc::mldb_timeline_buffer();
  p.reverse = tc::snake_order();
  p.items = p.nseq * p.heads * p.n_qt;
  p.heads_log2 = -1;
  for (int k = 0; k < 8; ++k) if ((1 << k) == p.heads) p.heads_log2 = k;
  const int pairs = (p.items + 1) / 2;                 // two pipelines per CTA
  const int grid = pairs < sm_count ? pairs : sm_count;
  auto kernel = a.hd == 64 ? (a.causal ? pick_kernel<64, true>(p.nkb) : pick_kernel<64, false>(p.nkb))
                           : (a.causal ? pick_kernel<128, true>(p.nkb) : pick_kernel<128, false>(p.nkb));
  launch_pdl(kernel, dim3(grid), dim3(WS_THREADS), (size_t)SMEM_BYTES, st, mQh, mQl, mKh, mKl, mRh, mRl, p);
  return true;
}
