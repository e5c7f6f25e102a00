// Internal engine types of libmldb200 (not part of the C ABI), and what the engine sources share: the error macros,
// the operator dispatch, the workspace and plan helpers.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/mldb.h"
#include "ops.cuh"

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t e__ = (call);                                                         \
    if (e__ != cudaSuccess) {                                                         \
      char buf__[512];                                                                \
      snprintf(buf__, sizeof buf__, "%s:%d: %s failed: %s", __FILE__, __LINE__, #call, \
               cudaGetErrorString(e__));                                              \
      mldb_set_err(buf__);                                                            \
      return MLDB_ERR_CUDA;                                                           \
    }                                                                                 \
  } while (0)

#define FAIL(code, ...)                         \
  do {                                          \
    char buf__[512];                            \
    snprintf(buf__, sizeof buf__, __VA_ARGS__); \
    mldb_set_err(buf__);                        \
    return (code);                              \
  } while (0)

#define TRY(expr)                 \
  do {                            \
    int rc__ = (expr);            \
    if (rc__ != MLDB_OK) return rc__; \
  } while (0)

// Every ABI call runs on the handle's device and restores the caller's current device afterwards
// (a single-process multi-GPU program must not find torch.cuda.current_device() changed under it).
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev); else prev = -1;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// The split16 layout (common.cuh) of a [rows, cols] activation at p: each plane padded to whole 128-row tiles.
inline ActBuf split16_at(void* p, int rows, int cols) {
  const int64_t rp = ((int64_t)rows + 127) / 128 * 128;
  return ActBuf{(__half*)p, rp * cols, rows, cols};
}
inline size_t split16_bytes(int rows, int cols) { return 2 * sizeof(__half) * split16_at(nullptr, rows, cols).plane_stride; }
inline ActBuf rows_of(ActBuf b, int64_t row0, int rows) { b.hi += row0 * b.cols; b.rows = rows; return b; }
inline unsigned nblk(int64_t n, int t = 256) { return (unsigned)((n + t - 1) / t); }

// A device buffer of the eager entry points, grown on demand and freed with the handle.
struct GrowBuf {
  void* p = nullptr;
  size_t cap = 0;
  GrowBuf() = default;
  GrowBuf(const GrowBuf&) = delete;
  GrowBuf& operator=(const GrowBuf&) = delete;
  ~GrowBuf() { cudaFree(p); }
};

// op_gru's state, one per model: two models' calls may run on different streams.  h_split / h_f32: the split16 /
// fp32 state ping-pong (k_gru_seq_tc: h_f32 holds the final state); gh: h W_hh^T under gemm=simt.
struct GruState { GrowBuf h_split, h_f32, gh; };

struct LnW { float* g = nullptr; float* b = nullptr; };

struct EncW {  // TransformerEncoderLayer (cross_attention.py:236-257)
  LinW in_proj, out_proj, l1, l2;
  LnW n1, n2;
  LinW q_only, kv_only;   // row slices [0:d) / [d:3d) of in_proj, packed for the stack's last layer
};
struct DecW {  // TransformerDecoderLayer (cross_attention.py:297-321)
  LinW sa_in, sa_out, ca_q, ca_kv, ca_v, ca_out, l1, l2;   // ca_v: rows [2d,3d) for the 1-memory-token collapse
  LnW n1, n2, n3;
};
// STACK_PLAIN_ENC: torch nn.TransformerEncoder without a final norm (ActorVae's encoder); its last layer always
// runs trimmed to the n_sel distribution rows
enum StackKind { STACK_SKIP_ENC = 0, STACK_SKIP_DEC = 1, STACK_PLAIN_DEC = 2, STACK_PLAIN_ENC = 3 };
struct StackW {
  int kind = STACK_SKIP_ENC;
  int d = 0, ff = 0, heads = 0, layers = 0;
  std::vector<EncW> enc;   // input blocks, middle, output blocks (in execution order); plain: layers in order
  std::vector<DecW> dec;
  std::vector<LinW> skip;  // linear_blocks (Linear(2d -> d))
  LnW norm;                // final norm (g == nullptr: none, ActorVae)
};

// CLIP text tower (mldb_text_configure): pre-norm layers, fused q|k|v operand
struct TextLayerW {
  LinW qkv, out, fc1, fc2;
  LnW ln1, ln2;
};
struct TextW {
  bool on = false;
  mldb_text_config cfg{};
  std::vector<TextLayerW> layers;
  LnW final_ln;
  LinW proj;                      // text_projection, no bias
  float* tok = nullptr;           // token_embedding [vocab, hidden] fp32
  float* pos = nullptr;           // position_embedding [max_positions, hidden] fp32
  // workspace of mldb_text_encode
  GrowBuf x;                      // [rows, hidden] fp32 residual stream
  GrowBuf a, qkv, att, h;         // LN output, q|k|v, attention output, fc1 output (split16)
  GrowBuf pooled;                 // [seqs, hidden] final LN of the eos rows (split16, A of text_projection)
};

// T2M evaluator (mldb_t2m_configure): bidirectional GRU + BiGRUCo head, the movement convolutions
struct GruW {
  int H = 0;
  LinW w_ih[2];                   // per direction [3H, in], gates r | z | n, bias b_ih
  LinW w_hh;                      // both directions [2 * 3H, H], rows in gru_packed_col order, no bias
  float* b_hh = nullptr;          // [2][3H] fp32
  float* h0 = nullptr;            // the learned `hidden` [2][H]
  LinW head1, head2;              // output_net.0 (2H -> H), output_net.3 (H -> out)
  LnW ln;                         // output_net.1
};
struct T2mW {
  bool on = false;
  mldb_t2m_config cfg{};
  LinW pos_emb, text_in;          // text: pos_emb (K padded to 64), input_emb (K padded to 64)
  LinW conv1, conv2, move_out;    // movement: main.0 / main.3 as [out, 4 * Cp] operands, out_net
  LinW motion_in;                 // motion: input_emb
  GruW text_gru, motion_gru;
  int chunk = 0;                  // option t2m_chunk (0: from the workspace budget)
  // workspace; the encoders run one at a time, so buffers that are never live together are shared
  GrowBuf in;                     // split16 A of the first GEMM: movement im2col of the poses, motion rows, text pos_ohot
  GrowBuf f32;                    // fp32: the GRU's x W_ih^T + b_ih, movement conv1 output
  GrowBuf emb;                    // split16: the GRU input rows, movement im2col of the conv1 output
  GrowBuf mid;                    // movement conv2 output (split16), text word_embs + pos_emb (fp32)
  GrowBuf words;                  // text word_embs + pos_emb (split16, K padded)
  GruState gru;
  GrowBuf head_f32, head_ln;      // GRU head: first Linear, LayerNorm + LeakyReLU
};

// HumanAct12 action classifier (mldb_a2m_configure): nn.GRU(input, H, layers) + Linear(H, 30), tanh, Linear(30, out)
struct A2mLayerW {
  LinW w_ih;                      // [3H, in] (K padded to a multiple of 64), gates r | z | n, bias b_ih
  LinW w_hh;                      // [3H, H], rows in gru_packed_col order, no bias
  float* b_hh = nullptr;          // [3H] fp32
};
struct A2mW {
  bool on = false;
  mldb_a2m_config cfg{};
  std::vector<A2mLayerW> layers;
  float *l1w = nullptr, *l1b = nullptr, *l2w = nullptr, *l2b = nullptr;   // the fp32 head: linear1, linear2
  int chunk = 0;                  // option a2m_chunk (0: from the workspace budget)
  // workspace of mldb_a2m_classify
  GrowBuf x;                      // split16 frames [n * T, input_size padded to 64]
  GrowBuf gi;                     // fp32 [n * T, 3H]: x_t W_ih^T + b_ih of the running layer
  GrowBuf seq;                    // split16 [n * T, H]: a layer's h_t, the A operand of the next layer's input GEMM
  GruState gru;
};

// UESTC action classifier (mldb_stgcn_configure): STGCN (uestc_stgcn.py), ten st_gcn blocks
constexpr int kStgcnBlocks = 10;
struct StgcnBlockW {
  LinW gcn;                       // [C_out, 3 C_in] (K padded to 64): the 1 x 1 conv with BN1 folded, column k C_in + ci
  float* gcn_tab = nullptr;       // [24, C_out] fp32: the gcn bias through the graph, + BN1's shift, per joint
  LinW tcn;                       // [C_out, 9 C_out (+ C_in)]: the (9, 1) conv tap-major with BN2 folded (+ the
                                  // residual 1 x 1 conv with its BN folded); bias: both biases and shifts
};
struct StgcnW {
  bool on = false;
  mldb_stgcn_config cfg{};
  StgcnBlockW blocks[kStgcnBlocks];
  float* adj = nullptr;           // [10][3][24][24] fp32: A * edge_importance[i]
  float *bn_scale = nullptr, *bn_shift = nullptr;   // data_bn [24 * in_channels], channel v * in_channels + c
  float *fcn_w = nullptr, *fcn_b = nullptr;         // [num_class, 256], [num_class]
  int chunk = 0;                  // option stgcn_chunk (0: from the workspace budget)
  // workspace of mldb_stgcn_classify
  GrowBuf z;                      // split16 [n * T * 24, 3 C_in (padded to 64)]: the graph mix, the gcn GEMM's A
  GrowBuf y;                      // split16 [n * T * 24, C_out]: the gcn output, the temporal convolution's input
  GrowBuf x[2];                   // split16 block outputs (ping-pong)
  GrowBuf last;                   // fp32 [n * T_out * 24, 256]: the last block's output
  GrowBuf col, acc;               // gemm=simt: the temporal convolution's im2col (split16) and its fp32 GEMM output
};

// SMPL layer (mldb_smpl_configure): zero betas, 24 joints, V vertices
struct SmplW {
  bool on = false;
  mldb_smpl_config cfg{};
  float J[24 * 3] = {};           // rest joints J_regressor v_template (computed in double)
  int parents[24] = {};
  LinW posedirs;                  // [3 V', 256]: posedirs^T (K 207 zero padded), 32-vertex tiles coordinate-planar
  float* v_template = nullptr;    // [V', 3] fp32, V' = V rounded up to 32, zero past V
  float* lbsw = nullptr;          // [V' / 32][24][32] fp32 lbs_weights, transposed per vertex tile
  uint32_t* jmask = nullptr;      // [V' / 32] joints with a non-zero weight in the tile
  int chunk = 0;                  // option smpl_chunk (0: the vertex path's workspace budget, the joints unchunked)
  // workspace of mldb_smpl_forward (vertices)
  GrowBuf feat;                   // split16 [frames, 256]: the pose features (R_j - I), the LBS GEMM's A
  GrowBuf xf;                     // fp32 [frames][24 * 12 + 4]: A_j, valid, translation offset
};

struct RawTensor {
  std::vector<float> host;
  std::vector<int64_t> shape;
  bool loaded = false;
};

// Workspace for one transformer stack pass over nseq sequences of L tokens.
struct StackWs {
  int nseq = 0, L = 0, M = 0, d = 0, ff = 0, Lmem = 0;
  ActBuf x0, cur[2], x1, x2, att, qkv, qc, kvm, h, cat;
  // compact buffers for the trimmed last layer (rows = nseq * n_sel)
  int n_sel = 0;
  ActBuf sx, sq, satt, sx1, sh, sout;
  // single-memory-token cross-attention collapse (per-sequence vectors)
  ActBuf vrow;            // [nseq, d]  V projection of the memory token
  float* cvec = nullptr;  // [nseq, d]  out_proj(V) + bias
  std::vector<ActBuf> ys;
  float* cf32 = nullptr;  // [M, d] GEMM result staging for the unfused (SIMT) LN path
};

struct TcCtx;

// A plan's workspace serves one entry point at one shape; the kind is part of the plan key.
enum PlanKind {
  PLAN_REVERSE = 0,       // reverse diffusion, trans_enc denoiser (mldb_diffusion_reverse, mldb_sample)
  PLAN_VAE_DECODE = 1,
  PLAN_VAE_ENCODE = 2,
  PLAN_DENOISE = 3,       // one trans_enc denoiser pass (mldb_denoise)
  PLAN_DENOISE_DEC = 4,   // one trans_dec (no-VAE) denoiser pass (mldb_denoise)
  PLAN_REVERSE_DEC = 5,   // reverse diffusion, trans_dec denoiser
};

struct Plan {
  int kind = PLAN_REVERSE;
  int B = 0, S = 0, T = 0, Bx = 0, Ntok = 0;
  StackWs ws;
  ActBuf mem;         // memory tokens for decoder stacks
  float* latents = nullptr;   // [B, per]
  float* eps = nullptr;       // [Bx, per]
  float* stage_f32 = nullptr; // misc fp32 staging
  float* tt_single = nullptr; // [d] time token for mldb_denoise
  float* feats = nullptr;     // [B, T, F] decode output staging for mldb_sample
  ActBuf ctx_split;           // relu(ctx) in split16 form, A operand of the emb_proj GEMM
  float* cond_f = nullptr;    // staged condition (host entry point)
  size_t cond_cap = 0;
  int64_t* cond_i = nullptr;
  float* noise_in = nullptr;
  float* step_noise = nullptr; // plan-owned copy of the injected per-step DDPM noise (graph-stable pointer)
  size_t noise_cap = 0;
  const float* noise_ptr = nullptr;  // caller noise pointer baked into the step graph (no-VAE loop)
  int* d_step = nullptr;       // device-side step counter of the replayed step graph
  ActBuf in_split;             // model input in split16 form, K zero-padded (no-VAE pose embedding)
  int32_t* lengths = nullptr; // device lengths (plan-owned copy)
  float* joints = nullptr;
  float* joints_all = nullptr;  // gathered joints of every rank (host entry point with a communicator)
  cudaGraphExec_t exec = nullptr;
  int64_t graph_nodes = 0;
  int sched_epoch = -1;
};

struct mldb_handle {
  mldb_config cfg;
  int device = 0;
  int sm_count = 0;
  bool finalized = false;
  std::map<std::string, RawTensor> raw;      // expected tensors (spec) + loaded data
  std::vector<void*> allocs;                 // everything cudaMalloc'ed by the handle
  // packed weights
  StackW den;          // denoiser stack
  StackW vdec, venc;   // VAE decoder / encoder stacks
  LinW time_l1, time_l2, emb_proj, pose_embd, pose_proj, skel_emb, final_layer;
  float* action_emb = nullptr;       // [nclasses, d]
  float* query_pe = nullptr;         // denoiser query_pos.pe [500, d]
  float* mem_pe = nullptr;           // denoiser mem_pos.pe [500, d]
  float* vae_dec_pe = nullptr;       // [500 | 5000, d]
  int vae_dec_pe_rows = 0;
  float* vae_enc_pe = nullptr;       // MldVae [500, d] | ActorVae [5000, d]
  int vae_enc_pe_rows = 0;
  float* global_token = nullptr;     // [2*n_lat, d]; ActorVae: [mu_token; logvar_token]
  float* mean = nullptr; float* stdv = nullptr; int nstat = 0;
  TextW text;          // CLIP text tower (mldb_text_configure)
  T2mW t2m;            // T2M evaluator (mldb_t2m_configure)
  A2mW a2m;            // HumanAct12 action classifier (mldb_a2m_configure)
  StgcnW stgcn;        // UESTC action classifier (mldb_stgcn_configure)
  SmplW smpl;          // SMPL layer (mldb_smpl_configure)
  // scheduler
  std::vector<float> alphas_cumprod;
  std::vector<int64_t> timesteps;
  std::vector<StepCoef> coefs_host;
  int64_t* d_timesteps = nullptr;
  StepCoef* d_coefs = nullptr;
  float* d_tt = nullptr;             // [nsteps, d] time tokens (time MLP + PE)
  float* d_tfeats = nullptr;         // time MLP scratch (sin/cos features)
  float* d_thid = nullptr;           // time MLP scratch (hidden)
  int sched_epoch = 0;
  // execution
  cudaStream_t cap_stream = nullptr;
  std::map<std::string, Plan*> plans;
  int64_t launches = 0;
  int64_t capture_nodes = 0;
  bool capturing = false;
  bool use_tc = true;        // wgmma GEMMs (option gemm=simt switches to the CUDA-core path)
  bool use_graph = true;
  // Concurrent sub-batches: the denoiser stack runs as `branches` independent sequence ranges on
  // parallel streams (parallel chains inside the captured graph), each with its own workspace rows,
  // so one range's kernel tails (316 m-tiles on 132 SMs = 2.39 rounds) and kernel boundaries are
  // filled by the other range's kernels.  1 = off.
  int branches = 2;
  int attn_kind = 0;         // 0 = wgmma (attn_tc.cu), 1 = mma.sync (attn_mma.cu), 2 = CUDA-core; option `attn`
  // which kernel every operator of the path was ENQUEUED on (recorded launches, incl. graph capture);
  // read through mldb_kernel_stats so that tests can assert "nothing fell back to CUDA cores"
  int64_t kstat[MLDB_KSTAT_COUNT] = {};
  bool op_failed = false;    // an operator could not be enqueued (tensor-map encoding): sticky until reported
  static constexpr int MAX_BRANCHES = 4;
  cudaStream_t br_stream[MAX_BRANCHES - 1] = {};
  // partial-accumulator scratch + flags of the fused FFN's hidden-dimension split (gemm_tc.h), one per stream a
  // stack can run on: [0] the caller's stream, [k] br_stream[k - 1]
  float* ffn_scratch[MAX_BRANCHES] = {};
  int* ffn_flags[MAX_BRANCHES] = {};
  cudaEvent_t ev_fork = nullptr, ev_join[MAX_BRANCHES - 1] = {};
  TcCtx* tc = nullptr;
  // the path's one collective (comm.cu): NCCL communicator bound at run time, gathers on a side stream
  void* nccl_comm = nullptr;
  bool comm_owned = false;
  int comm_world = 1, comm_rank = 0;
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t ev_local_done = nullptr, ev_gather_done[2] = {};
  int64_t gather_count = 0;
};

struct SeqInfo {
  const int32_t* lengths = nullptr;  // key-padding: valid keys = kv_prefix + lengths[s % len_mod]
  int kv_prefix = 0;
  int len_mod = 0;
};

// engine.cu
inline void kcount(mldb_handle* h, int kind) {
  h->kstat[kind]++;
  if (h->capturing) h->capture_nodes++; else h->launches++;
}
int check_ready(mldb_handle* h, bool need_sched);
int check_ops(mldb_handle* h);
// The exit of an eager entry point that enqueued operators: a launch error or an operator that could not be
// enqueued fails the call.
inline int ops_done(mldb_handle* h) {
  CK(cudaGetLastError());
  return check_ops(h);
}
// mldb_<name>_configure after its null check: the config's abi_version, before finalize, not yet configured (`on`)
int may_configure(const mldb_handle* h, int abi_version, int expected, bool on, const char* name, const char* what);
// an entry point of a model configured by mldb_<name>_configure: configured (`on`) and finalized
int check_configured(const mldb_handle* h, bool on, const char* name, const char* what);
// sequences per chunk of an eager evaluator: the option, else what keeps the chunk's workspace near 1 GiB (whole
// `round`-row tiles when more than one)
int eval_chunk(int option, int B, size_t per_seq, int round);
int dev_alloc(mldb_handle* h, void** p, size_t bytes);
int grow(GrowBuf& b, size_t bytes);
int grow_act(GrowBuf& b, int rows, int cols, ActBuf* out);
int upload_f32(mldb_handle* h, const float* src, size_t n, float** out);
int upload_pe(mldb_handle* h, const std::string& key, float** out, int* rows = nullptr);
const RawTensor& rt(mldb_handle* h, const std::string& k);
void spec_add(mldb_handle* h, const std::string& key, std::vector<int64_t> shape);
void spec_ln(mldb_handle* h, const std::string& p, int d);
int pack_linear(mldb_handle* h, const float* W, int N, int K, const float* bias, LinW* out, int Kpad = 0);
int pack_named(mldb_handle* h, const std::string& wkey, const std::string& bkey, LinW* out, int row0 = 0,
               int nrows = -1, bool pad_k = false);
int pack_ln(mldb_handle* h, const std::string& p, int d, LnW* out);
int time_tokens(mldb_handle* h, const int64_t* d_ts, int64_t t_scalar, int n, const float* pe_row, float* out,
                float* scratch_feats, float* scratch_h, cudaStream_t st);
Plan* find_plan(mldb_handle* h, PlanKind kind, int B, int S, int T);
Plan* add_plan(mldb_handle* h, PlanKind kind, int B, int S, int T);
// Run `record` either directly on `st` or as a (cached) CUDA graph.
int run_graphed(mldb_handle* h, Plan* p, cudaStream_t st, const std::function<void(cudaStream_t)>& record);

// stack.cu: operators (each picks its kernel and counts it in kstat), workspaces, transformer stacks
void op_gemm(mldb_handle* h, const GemmArgs& g, cudaStream_t st);
void op_gemm_ln(mldb_handle* h, GemmArgs g, LnArgs l, float* cf32, cudaStream_t st);
void op_ln(mldb_handle* h, const LnArgs& l, cudaStream_t st);
void op_attn(mldb_handle* h, const AttnArgs& a, cudaStream_t st);
// One GRU layer over n sequences of L steps, x [n * L, in] split16 (row b * L + t): gi = x W_ih^T + b_ih (grown
// here), then the recurrence on k_gru_seq_tc (dirs == 1, H = 64 or 128 as mldb_a2m_configure enforces), on
// k_gru_step_tc per step (dirs == 2), or under gemm=simt on CUDA-core GEMMs and k_gru_gate_simt per step.
// w_hh: the directions' packed [3H, H] stacked; b_hh [dirs][3H]; h0 of (dir, row m) at h0[dir * H + m * h0_ld]
// (k_gru_seq_tc: h0_ld == H).  seq_out (dirs == 1; hi null: none) gets h_t as split16 row m * L + t.  The final
// states at t = len - 1 (null: not wanted), direction d's row m at row d * rows_pad + m (n rounded up to 128):
// *fin split16 (not from k_gru_seq_tc), *fin_f32 fp32 with rows H floats apart.
int op_gru(mldb_handle* h, ActBuf x, const LinW* w_ih, const LinW& w_hh, const float* b_hh, const float* h0,
           int64_t h0_ld, const int32_t* lengths, int n, int L, int H, int dirs, GrowBuf& gi, GruState& ws,
           ActBuf seq_out, ActBuf* fin, const float** fin_f32, cudaStream_t st);
void op_tail(mldb_handle* h, const LinW& wo, const LnW& n1, const LinW& l1, const LinW& l2, const LnW& n2, ActBuf att,
             ActBuf x, ActBuf x1, ActBuf hbuf, ActBuf xout, int M, int d, int ff, float* cf32, cudaStream_t st,
             int fuse = 1);
void rows_to_split(mldb_handle* h, ActBuf X, const float* src, int ld_src, int M, int d, int in_group, int out_group,
                   int out_off, int src_bcast, const float* tab, int relu, cudaStream_t st);
int alloc_act(mldb_handle* h, int rows, int cols, ActBuf* out);
int alloc_stack_ws(mldb_handle* h, const StackW& sw, int nseq, int L, int Lmem, StackWs* ws, int n_sel = 0);
StackWs ws_slice(const StackWs& ws, int s0, int n);
void out_proj_ln(mldb_handle* h, const LinW& w, const LnW& n, ActBuf att, ActBuf res, ActBuf xout, int M, int d,
                 float* cf32, cudaStream_t st);
void ffn_block(mldb_handle* h, const LinW& l1, const LinW& l2, const LnW& n, ActBuf xin, ActBuf xout, StackWs& ws,
               int act, cudaStream_t st);
void enc_layer(mldb_handle* h, const StackW& sw, const EncW& w, ActBuf xin, ActBuf xout, StackWs& ws,
               const SeqInfo& si, cudaStream_t st);
ActBuf run_stack(mldb_handle* h, const StackW& sw, ActBuf x0, ActBuf mem, StackWs& ws, const SeqInfo& si,
                 cudaStream_t st);

// denoiser.cu
int enc_plan(mldb_handle* h, PlanKind kind, int B, int Bx, int S, Plan** out);
int place_condition(mldb_handle* h, Plan* p, const void* cond, cudaStream_t st);
void denoiser_pass(mldb_handle* h, Plan* p, const float* latents, int lat_mod, const float* tt, float* eps_out,
                   cudaStream_t st);
// vae.cu
int dec_plan(mldb_handle* h, int B, int T, Plan** out);
int run_decode(mldb_handle* h, const float* z, const int32_t* lengths, int B, int T, float* feats_out, cudaStream_t st,
               Plan** plan_out);
int run_f2j(mldb_handle* h, const float* feats, int B, int T, float* joints, cudaStream_t st);
// text_tower.cu, t2m.cu, a2m.cu, stgcn.cu
int pack_text(mldb_handle* h);
int pack_t2m(mldb_handle* h);
int pack_a2m(mldb_handle* h);   // a2m.cu
int pack_stgcn(mldb_handle* h); // stgcn.cu
int pack_smpl(mldb_handle* h);  // smpl.cu

// comm.cu
void mldb_comm_release(mldb_handle* h);
int mldb_gather_begin(mldb_handle* h, cudaStream_t stream);
int mldb_gather_async(mldb_handle* h, float* global, int64_t count, cudaStream_t stream);
