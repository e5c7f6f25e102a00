// Operator argument blocks shared by the tensor-core (wgmma) and SIMT implementations.
#pragma once
#include "common.cuh"

// Packed nn.Linear weights: W [N, K] (PyTorch [out, in] layout == K-major B operand) stored as
// two fp16 planes of W * 2^scale_log2 (power-of-two scale keeps the lo plane out of the fp16
// subnormal range; exact, undone in the epilogue).
struct LinW {
  __half* w = nullptr;        // [2][N][K]: hi plane then lo plane
  int64_t plane_stride = 0;   // N*K
  float* bias = nullptr;      // [N] fp32 or null
  int N = 0, K = 0;
  float inv_scale = 1.0f;     // 2^-scale_log2
  int id = -1;                // index into the engine's tensor-map cache
};

enum AKind { A_SPLIT = 0, A_F32 = 1, A_F32_RELU = 2 };

// out[map(r), n] = act( (sum_k A[r,k] W[n,k]) * inv_scale + bias[n] + addtab[pos(r), n] )
// with A = [a1 | a2] concatenated along K (torch.cat(..., dim=-1) of the skip connections,
// cross_attention.py:56-58) or an fp32 matrix (external inputs: CLIP context, motion feats).
struct GemmArgs {
  int a_kind = A_SPLIT;
  ActBuf a1{}; int K1 = 0;
  ActBuf a2{}; int K2 = 0;
  const float* a_f32 = nullptr; int lda = 0;
  int M = 0;
  LinW w{};
  int act = ACT_NONE;
  ActBuf out{};               // split output when out.hi != nullptr (ld = out.cols)
  int out_col0 = 0;           // column offset inside out
  float* out_f32 = nullptr; int ldc = 0;
  // row r -> out row (r / in_group) * out_group + out_off + r % in_group (identity when in_group >= M)
  int in_group = 1 << 30, out_group = 0, out_off = 0;
  const float* addtab = nullptr;        // [*, N]: row (out_off + r % in_group)
  const int32_t* zero_lengths = nullptr;  // zero rows with (r % in_group) >= zero_lengths[r / in_group]
};

// y = LayerNorm(c + res + rowvec[r / rv_group]) * gamma + beta, eps 1e-5; optional second LN
// (gamma2/beta2) applied on top (last block's norm2 followed by the stack's final norm).
struct LnArgs {
  const float* c = nullptr; int ldc = 0;   // fp32 GEMM result incl. bias (nullable)
  ActBuf res{};                              // residual (nullable: res.hi == nullptr)
  const float* rowvec = nullptr; int rv_group = 1;
  const float* gamma = nullptr; const float* beta = nullptr;
  const float* gamma2 = nullptr; const float* beta2 = nullptr;
  int M = 0, d = 0;
  // input row selection: in_row = (r / sel_group) * in_group + r % sel_group (identity default)
  int sel_group = 1 << 30, in_group = 0;
  ActBuf out{}; float* out_f32 = nullptr; int ld_out = 0;
};

// Multi-head attention over per-sequence token groups.  Row of (seq s, token t) = s*L + t.
// Q from `q` at column q_col0 + h*hd, K/V from `kv` at k_col0/v_col0 + h*hd.
struct AttnArgs {
  ActBuf q{}; int q_col0 = 0; int Lq = 0;
  ActBuf kv{}; int k_col0 = 0, v_col0 = 0; int Lk = 0;
  int nseq = 0, heads = 0, hd = 0;
  const int32_t* lengths = nullptr;   // valid keys = min(Lk, kv_prefix + lengths[s]) when set
  int kv_prefix = 0;
  int len_mod = 0;                    // lengths index = (seq0 + s) % len_mod when len_mod > 0
  int seq0 = 0;                       // global index of this launch's first sequence (chunked launches)
  ActBuf out{};                       // [nseq*Lq, heads*hd]
};

// --- SIMT implementations (simt.cu) ---
void simt_gemm(const GemmArgs& a, cudaStream_t st);
void simt_ln(const LnArgs& a, cudaStream_t st);
void simt_attention(const AttnArgs& a, cudaStream_t st);
// --- mma.sync tensor-core attention (attn_mma.cu) ---
bool mma_attention_supported(const AttnArgs& a);
void mma_attention_init();
void mma_attention(const AttnArgs& a, cudaStream_t st);
// attn_tc.cu: wgmma attention core (Lk <= 256, head_dim 64 / 128)
bool tc_attention_init(int device);                       // once per process, outside stream capture
bool tc_attention_supported(const AttnArgs& a);
bool tc_attention(const AttnArgs& a, cudaStream_t st);    // false: tensor-map encoding failed, nothing launched
void simt_init();
// --- wgmma implementations (gemm_tc.cu) ---
struct TcCtx;
