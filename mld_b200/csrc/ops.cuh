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
  // row r -> out row (r / in_group) * out_group + out_off + r % in_group, on every path (so out_off + r when
  // in_group >= M; the defaults give the identity)
  int in_group = 1 << 30, out_group = 0, out_off = 0;
  const float* addtab = nullptr;        // [*, N]: row (out_off + r % in_group)
  const int32_t* zero_lengths = nullptr;  // zero rows with (r % in_group) >= zero_lengths[r / in_group]
  // residual add: out_f32[r, n] = act(...) + res_f32[r * ldc + n] (fp32 [M, N], leading dimension ldc; may alias
  // out_f32, which is how the CLIP text tower updates its fp32 residual stream in place)
  const float* res_f32 = nullptr;
  int wide_n = 0;                       // 1: the wgmma kernel may take N up to 4096 (the text tower's 2304 / 3072);
                                        // the sampling path keeps its N <= 1024 kernel selection
  int vec_f32 = 0;                      // 1: fp32 output (no residual, identity rows, N even) through the wgmma kernel's
                                        // vectorised epilogue fmaf(acc, scale, bias) (the T2M evaluator); the
                                        // sampling path keeps the generic epilogue it was validated with
};

// y = LayerNorm(c + res + rowvec[in_row / rv_group]) * gamma + beta, eps 1e-5
struct LnArgs {
  const float* c = nullptr; int ldc = 0;   // fp32 GEMM result incl. bias (nullable)
  ActBuf res{};                              // residual (nullable: res.hi == nullptr)
  const float* rowvec = nullptr; int rv_group = 1;
  const float* gamma = nullptr; const float* beta = nullptr;
  int M = 0, d = 0;                          // d <= LN_MAX_D on the CUDA cores (simt_ln)
  // input row selection: in_row = (r / sel_group) * in_group + r % sel_group (identity default)
  int sel_group = 1 << 30, in_group = 0;
  ActBuf out{}; float* out_f32 = nullptr; int ld_out = 0;
  int act = ACT_NONE;                        // activation on the normalised output (CUDA-core kernels only)
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
  int causal = 0;                     // 1: query i attends to keys j <= i only (self-attention, Lq == Lk)
  ActBuf out{};                       // [nseq*Lq, heads*hd]
};

// Scheduler coefficients for one step, computed on the host in fp32 exactly as diffusers does
// (0-d fp32 tensor arithmetic; x ** 0.5 == sqrtf).
struct StepCoef {
  float c0, c1, c2, c3;  // DDIM: sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-std^2)
                         // DDPM: sqrt(a_t), sqrt(1-a_t), x0 coeff, sample coeff
  float sigma;           // scale of the injected N(0,1) noise; 0 = the step adds none (and reads none)
                         // DDIM: std_dev_t = eta * sqrt(variance); DDPM: sqrt(clamp(var, 1e-20)) when t > 0
  int kind;              // 0 DDIM, 1 DDPM
  int clip;              // clip_sample: x0 clamped to [-1, 1] (clip_sample_range 1.0)
};

// --- SIMT implementations (simt.cu) ---
void simt_gemm(const GemmArgs& a, cudaStream_t st);
// One warp per row; the widest kernel keeps 32 columns per lane, so rows of up to LN_MAX_D columns.  Callers keep
// d within it (mldb_create's latent_dim, gru_shape_supported's H, mldb_debug_ln).
constexpr int LN_MAX_D = 1024;
void simt_ln(const LnArgs& a, cudaStream_t st);
// CUDA-core attention: any Lq / Lk (K and V stream through shared memory in key chunks).  false: the head is too
// wide for the shared memory (simt_attention_supported), nothing launched.
bool simt_attention(const AttnArgs& a, cudaStream_t st);
bool simt_attention_supported(int hd);
// --- mma.sync tensor-core attention (attn_mma.cu) ---
bool mma_attention_supported(const AttnArgs& a);
bool mma_attention_init();                                // per device, outside stream capture
void mma_attention(const AttnArgs& a, cudaStream_t st);
// attn_tc.cu: wgmma attention core (Lk <= 256, head_dim 64 / 128)
bool tc_attention_init();                                 // per device, outside stream capture
bool tc_attention_supported(const AttnArgs& a);
// at most sm_count CTAs; false: tensor-map encoding failed, nothing launched
bool tc_attention(const AttnArgs& a, int sm_count, cudaStream_t st);
bool simt_init();                                         // reads MLDB_PDL; per device, outside stream capture
// --- text tower row kernels (text_ln.cu) ---
// One warp per row, d a multiple of 128 up to 1024, exact two-pass statistics, no shared memory.
//   TEXT_LN_ROWS:     out = LN(x[r])                                   (CLIP: pre-norm LN1 / LN2, final LN of every
//                                                                      row; BERT: the post-norm LN with out_f32 = x)
//   TEXT_LN_EMBED:    x[r] = tok[ids[r]] + pos[r % L]; out = LN(x[r])  (CLIP layer 0; an id outside [0, vocab) -> NaN
//                                                                      row)
//   TEXT_LN_EOS:      out[s] = LN(x[s * L + eos_pos(ids[s, :])])       (pooled mode: only the gathered rows)
//   TEXT_LN_EMBED_LN: out = LN(tok[ids[r]] + pos[r % L] (+ type0))     (BERT embeddings; x is not written: out_f32 = x
//                                                                      makes the normalised row the residual stream)
enum TextLnMode { TEXT_LN_ROWS = 0, TEXT_LN_EMBED = 1, TEXT_LN_EOS = 2, TEXT_LN_EMBED_LN = 3 };
struct TextLnArgs {
  int mode = TEXT_LN_ROWS;
  float* x = nullptr;                 // fp32 residual stream [rows, d] (written in TEXT_LN_EMBED, read by ROWS / EOS)
  const int64_t* ids = nullptr; int L = 0;
  const float* tok = nullptr; const float* pos = nullptr; int vocab = 0;
  const float* type0 = nullptr;       // TEXT_LN_EMBED_LN: token-type row 0 added to every row (null: none)
  int eos_id = 0;                     // eos_id == 2: eos_pos = argmax(ids) (legacy configs); else first id == eos_id, or 0
  const float* gamma = nullptr; const float* beta = nullptr; float eps = 1e-5f;
  int M = 0, d = 0;                   // output rows (TEXT_LN_EOS: sequences)
  ActBuf out{};                       // split16 output (nullable)
  float* out_f32 = nullptr;           // fp32 output [M, d] (nullable)
};
bool text_ln_supported(int d);
void text_ln(const TextLnArgs& a, cudaStream_t st);
// --- the GRUs of the T2M evaluator (bidirectional) and of the action classifier (unidirectional, gru_tc.cu) ---
// State buffers are [dirs * rows_pad, H]: direction d's row m at d * rows_pad + m (rows_pad a multiple of 128).
struct GruStepArgs {
  ActBuf h_in{}, h_out{};              // split16 state h_{s-1} (the MMA operand) / h_s
  const float* hf_in = nullptr;        // fp32 state h_{s-1} (the z * h term and the copy-through)
  float* hf_out = nullptr;
  const float* gi = nullptr;           // [rows * L, dirs * 3H]: x_t W_ih^T + b_ih, forward then backward, gates r | z | n
  const float* gh = nullptr;           // CUDA-core path: [dirs * rows_pad, 3H] h W_hh^T in the packed column order
  const float* b_hh = nullptr;         // [dirs][3H] fp32, gates r | z | n
  const int32_t* lengths = nullptr;    // [rows] valid steps per sequence (clamped to [0, L])
  const __half* w_hh = nullptr;        // packed W_hh planes [2][dirs * 3H][H] (gru_packed_col order)
  int64_t w_plane_stride = 0;
  float w_inv_scale = 1.0f;
  int rows = 0, rows_pad = 0, L = 0, H = 0, step = 0;
  int dirs = 2;                        // 2: bidirectional (k_gru_step_tc's only layout); 1: forward only
  int64_t h0_ld = 0;                   // initial state of (dir, row m) at h0[dir * H + m * h0_ld]: 0 broadcasts one vector
  ActBuf seq_out{};                    // CUDA-core gates, dirs == 1: h_s also goes to split16 row m * L + t (hi null: not)
};
// One unidirectional layer of the action classifier over every step (k_gru_seq_tc).  The split16 W_hh of the layer
// stays in shared memory for the whole launch; each warpgroup carries a 64-row tile through all L steps.
struct GruSeqArgs {
  const float* gi = nullptr;           // [rows * L, 3H]: x_t W_ih^T + b_ih, gates r | z | n; only t < len is read
  const float* b_hh = nullptr;         // [3H] fp32, gates r | z | n
  const float* h0 = nullptr;           // [rows, H] fp32, each row's own initial state
  const int32_t* lengths = nullptr;    // [rows], each in [1, L] (clamped to [0, L])
  const __half* w_hh = nullptr;        // packed W_hh planes [2][3H][H] (gru_packed_col order)
  int64_t w_plane_stride = 0;
  float w_inv_scale = 1.0f;
  ActBuf seq_out{};                    // not the last layer: h_t (t < len) as split16 row m * L + t (hi null: not written)
  float* h_last = nullptr;             // the last layer: [rows, H] fp32 h at t = len - 1 (null: not written)
  int rows = 0, L = 0, H = 0;
};
// column of gate g (0 r, 1 z, 2 n) of hidden unit u inside one direction's 3H packed rows: 32-unit tiles of 96 rows,
// 8-row group 3 * jj + g holds units 8 * jj .. 8 * jj + 7 of the tile
__host__ __device__ __forceinline__ int gru_packed_col(int g, int u) {
  const int t = u >> 5, uu = u & 31;
  return t * 96 + (3 * (uu >> 3) + g) * 8 + (uu & 7);
}
bool gru_tc_init();                                              // per device, outside stream capture
bool gru_shape_supported(int H);                                 // 64 <= H <= 1024, H % 64 == 0
bool gru_step_tc(const GruStepArgs& a, cudaStream_t st);         // false: tensor-map encoding failed, nothing launched
void gru_gate_simt(const GruStepArgs& a, cudaStream_t st);       // the gate update from a.gh (CUDA cores)
void gru_init_state(const GruStepArgs& a, const float* h0, cudaStream_t st);   // h_out / hf_out = h0 (see h0_ld)
bool gru_seq_supported(int H);                                   // H = 64 or 128: W_hh fits in shared memory
// at most sm_count CTAs; false: tensor-map encoding failed, nothing launched
bool gru_seq_tc(const GruSeqArgs& a, int sm_count, cudaStream_t st);
// Conv1d(k = 4, stride 2, padding 1) im2col: src [rows / T_out sequences][T_in][ld] fp32 -> X [rows, 4 * Cp] split16
void im2col_k4s2(ActBuf X, const float* src, int64_t ld, int T_in, int C, int Cp, int T_out, int rows, cudaStream_t st);
// --- the ST-GCN's temporal convolution (tconv_tc.cu) ---
// One st_gcn block's tcn + residual + ReLU over activations laid out [nseq][T][24 joints][C] (split16 rows
// (n * T + t) * 24 + v), as an implicit GEMM with K = 9 taps x C (+ C_res for a residual convolution):
//   out[(n, t, v), c] = relu( sum_{tap, ci} x[(n, s t + tap - 4, v), ci] W[c, tap C + ci] * inv_scale
//                             (+ sum_cr res[(n, s t, v), cr] W[c, 9 C + cr] * inv_scale) + bias[c] (+ res[(n, t, v), c]) )
// Frames outside [0, T_in) read as zero (the convolution's padding).
struct TconvArgs {
  ActBuf x{};                          // split16 [nseq * T_in * 24, C]: the block's gcn output
  ActBuf res{};                        // split16 [nseq * T_in * 24, C_res]: the block input (hi null: no residual)
  int res_conv = 0;                    // 1: res goes through the 1 x 1 stride-s convolution (W's tenth K segment);
                                       // 0: res is added as it is (C_res == C, stride 1)
  LinW w{};                            // [C, 9 C (+ C_res)] tap-major, every BatchNorm folded; bias [C]
  int nseq = 0, T_in = 0, T_out = 0, C = 0, C_res = 0, stride = 1;
  ActBuf out{};                        // split16 [nseq * T_out * 24, C] (hi null: out_f32)
  float* out_f32 = nullptr;            // fp32 [nseq * T_out * 24, C]
};
bool tconv_tc_init();                                            // per device, outside stream capture
bool tconv_tc_supported(const TconvArgs& a);                     // C in {64, 128, 256}, C_res % 64 == 0, stride 1 | 2
// at most sm_count CTAs; false: tensor-map encoding failed, nothing launched
bool tconv_tc(const TconvArgs& a, int sm_count, cudaStream_t st);
// --- the SMPL layer's skinning kernel (smpl.cu) ---
bool smpl_tc_init();                                             // per device, outside stream capture
// --- wgmma implementations (gemm_tc.cu) ---
struct TcCtx;
