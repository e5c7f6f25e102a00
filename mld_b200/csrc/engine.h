// Internal engine types of libmldb200 (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/mldb.h"
#include "misc_kernels.cuh"
#include "ops.cuh"

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
enum StackKind { STACK_SKIP_ENC = 0, STACK_SKIP_DEC = 1, STACK_PLAIN_DEC = 2 };
struct StackW {
  int kind = STACK_SKIP_ENC;
  int d = 0, ff = 0, heads = 0, layers = 0;
  std::vector<EncW> enc;   // input blocks, middle, output blocks (in execution order)
  std::vector<DecW> dec;
  std::vector<LinW> skip;  // linear_blocks (Linear(2d -> d))
  LnW norm;                // final norm (g == nullptr: none, ActorVae)
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

struct Plan {
  int kind = 0;       // 0 reverse (denoiser), 1 vae decode, 2 vae encode, 3 single denoise
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
  float* vae_enc_pe = nullptr;
  float* global_token = nullptr;     // [2*n_lat, d]
  float* mean = nullptr; float* stdv = nullptr; int nstat = 0;
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

// helpers implemented in engine.cu
void mldb_set_err(const std::string& s);
// comm.cu
void mldb_comm_release(mldb_handle* h);
int mldb_gather_begin(mldb_handle* h, cudaStream_t stream);
int mldb_gather_async(mldb_handle* h, float* global, int64_t count, cudaStream_t stream);
