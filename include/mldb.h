/*
 * mldb.h - C ABI of libmldb200.so: the B200-native MLD latent-diffusion sampling path.
 *
 * The reference (ChenFengYe/motion-latent-diffusion) is pure Python and has no FFI; its
 * extension point is the YAML `target:` factory (mld/config.py:106-121) plus
 * `load_state_dict(strict=True)` (demo.py:150).  Each entry point below replaces one
 * reference Python interface on the sampling path (file:line given per function); the
 * torch-side binding a maintainer adds is the ctypes shim shown in INTEGRATION.md
 * (mld_b200/_lib.py + mld_b200/modules.py).
 *
 * Conventions
 *  - plain C, no exceptions across the boundary; every call returns an int status
 *    (MLDB_OK == 0); the message of the last failure on the calling thread is
 *    mldb_last_error().
 *  - the caller (PyTorch) owns every tensor; the library borrows raw pointers for the
 *    duration of the enqueue and never frees them.  Unless a parameter is marked HOST, it
 *    is a device pointer on the handle's device, fp32 row-major contiguous.
 *  - all work is enqueued on the `stream` argument (a cudaStream_t passed as void*), calls
 *    are asynchronous with respect to the host unless stated otherwise.
 *  - a handle is bound to one device and is not thread-safe (one handle per GPU/stream).
 *  - there is NO CPU fallback: a device that is not sm_90 makes mldb_create fail.
 */
#ifndef MLDB_H_
#define MLDB_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MLDB_OK 0
#define MLDB_ERR_INVALID 1   /* bad argument / unknown key / shape mismatch */
#define MLDB_ERR_CUDA 2      /* a CUDA runtime/driver call failed */
#define MLDB_ERR_STATE 3     /* call out of order (weights not finalized, ...) */
#define MLDB_ERR_UNSUPPORTED 4

#define MLDB_ABI_VERSION 3

typedef struct mldb_handle mldb_handle;

/* condition kinds: MldDenoiser(condition=...) mld_denoiser.py:54-79 */
#define MLDB_COND_TEXT 0
#define MLDB_COND_ACTION 1
/* denoiser arch: mld_denoiser.py:91-131 */
#define MLDB_ARCH_TRANS_ENC 0  /* SkipTransformerEncoder over [latent, time, cond...] */
#define MLDB_ARCH_TRANS_DEC 1  /* TransformerDecoder, memory = [time, cond]; no-VAE model */
/* VAE kinds */
#define MLDB_VAE_NONE 0
#define MLDB_VAE_MLD 1    /* MldVae arch=encoder_decoder, learned PE (mld_vae.py) */
#define MLDB_VAE_ACTOR 2  /* ActorVae (actor_vae.py) */
/* scheduler kinds (diffusers; configs/modules/scheduler.yaml) */
#define MLDB_SCHED_DDIM 0
#define MLDB_SCHED_DDPM 1
/* tensor dtypes for mldb_load_tensor */
#define MLDB_DTYPE_F32 0

/* Mirrors the ctor kwargs of MldDenoiser (mld_denoiser.py:18-38), MldVae (mld_vae.py:35-47)
 * / ActorVae (actor_vae.py:13-24) and the diffusers scheduler params
 * (configs/modules/scheduler.yaml:1-14) that change the math of the sampling path. */
typedef struct mldb_config {
  int32_t abi_version;        /* must be MLDB_ABI_VERSION */
  /* denoiser */
  int32_t cond_kind;          /* MLDB_COND_* */
  int32_t arch;               /* MLDB_ARCH_* */
  int32_t latent_dim;         /* d: latent_dim[-1] (256; 512 for the no-VAE model) */
  int32_t n_lat;              /* latent_dim[0] (1) */
  int32_t num_heads;          /* 4 */
  int32_t ff_size;            /* 1024 */
  int32_t num_layers;         /* 9 (15 for the action model); odd for the skip encoder */
  int32_t text_dim;           /* text_encoded_dim, 768 */
  int32_t nclasses;           /* action classes (12) */
  int32_t nfeats;             /* motion features (263 / 150), used when diffusion_only */
  int32_t diffusion_only;     /* ablation.VAE_TYPE == "no" */
  int32_t flip_sin_to_cos;    /* 1 */
  float   freq_shift;         /* 0 */
  float   guidance_scale;     /* 7.5; > 1 enables classifier-free guidance */
  /* VAE */
  int32_t vae_kind;           /* MLDB_VAE_* */
  int32_t vae_layers;         /* 9 (MldVae) / 6 (ActorVae) */
  int32_t vae_heads;          /* 4 */
  int32_t vae_ff;             /* 1024 */
  int32_t vae_nfeats;         /* 263 / 150 */
  /* scheduler */
  int32_t sched_kind;         /* MLDB_SCHED_* */
  int32_t num_train_timesteps;/* 1000 */
  double  beta_start;         /* 0.00085 (double: diffusers takes the Python float's sqrt) */
  double  beta_end;           /* 0.012  (beta_schedule is scaled_linear) */
  int32_t steps_offset;       /* DDIM: 1 */
  int32_t set_alpha_to_one;   /* DDIM: 0 */
  float   eta;                /* DDIM: 0.0 (only eta == 0 is supported: no step noise) */
  int32_t njoints;            /* 22 (HumanML3D) for feats2joints */
} mldb_config;

/* Fill cfg with the shipped text-to-motion defaults (configs/modules/{denoiser,motion_vae,
 * scheduler}.yaml + configs/config_mld_humanml3d.yaml). */
void mldb_default_config(mldb_config* cfg);

/* Replaces: instantiate_from_config(cfg.model.{denoiser,motion_vae,scheduler})
 * (mld/models/modeltype/mld.py:56-83).  Fails unless `device` is an sm_90 GPU. */
int mldb_create(const mldb_config* cfg, int device, mldb_handle** out);
void mldb_destroy(mldb_handle* h);

/* Replaces: load_state_dict(strict=True) (demo.py:150, base.py:117-127).  `key` is the
 * reference state-dict key with its Lightning prefix ("denoiser.encoder.norm.weight",
 * "vae.final_layer.bias", ...).  `data` may be a HOST or device pointer (cudaMemcpyDefault);
 * the call copies synchronously.  Unknown keys and shape mismatches are errors. */
int mldb_load_tensor(mldb_handle* h, const char* key, const void* data,
                     const int64_t* shape, int32_t ndim, int32_t dtype);

/* Pack / split / transpose the loaded tensors into the device arena.  Every key the
 * configured modules need must have been loaded (strict).  Synchronous. */
int mldb_finalize_weights(mldb_handle* h, void* stream);

/* HumanML3D dataset statistics used by feats2joints (mld/data/HumanML3D.py:41-45);
 * HOST or device pointers, `nfeats` floats each. */
int mldb_set_mean_std(mldb_handle* h, const float* mean, const float* std, int32_t nfeats);

/* Host-only helpers (no GPU, no handle): the scheduler's tables, exposed so that the integer
 * timestep arithmetic and the alphas_cumprod table can be checked on a CPU-only machine.
 * alphas_cumprod_out: HOST float[num_train_timesteps]; out: HOST int64[n]. */
int mldb_scheduler_table(const mldb_config* cfg, float* alphas_cumprod_out);
int mldb_scheduler_timesteps(const mldb_config* cfg, int32_t n, int64_t* out);

/* Replaces: scheduler.set_timesteps(n); scheduler.timesteps (mld.py:312-314).
 * timesteps_out: HOST int64[n] (may be NULL).  Integer arithmetic is bit-exact with
 * diffusers: DDIM (arange(n)*(T/n))[::-1]+steps_offset, DDPM arange(0,T,T/n)[::-1]. */
int mldb_scheduler_set_timesteps(mldb_handle* h, int32_t n, int64_t* timesteps_out);

/* Replaces: scheduler.step(model_output, t, sample, eta=0).prev_sample (mld.py:345).
 * `noise` is the injected N(0,1) tensor for DDPM when t > 0 (NULL for DDIM).
 * count = number of floats in sample. */
int mldb_scheduler_step(mldb_handle* h, const float* model_output, int64_t timestep,
                        const float* sample, const float* noise, int64_t count,
                        float* prev_sample, void* stream);

/* Replaces: MldDenoiser.forward(sample, timestep, encoder_hidden_states, lengths)[0]
 * (mld_denoiser.py:135-228).
 *   sample  [Bx, n_lat, d]  (or [Bx, T, nfeats] when diffusion_only)
 *   cond    text: float [Bx, S_ctx, text_dim];  action: int64 [Bx, 1] (class ids, already
 *           cat(zeros, actions) as at mld.py:716-717)
 *   lengths device int32[Bx] or NULL (only read when diffusion_only)
 *   out     same shape as sample */
int mldb_denoise(mldb_handle* h, const float* sample, int64_t timestep, const void* cond,
                 const int32_t* lengths, int32_t Bx, int32_t S_ctx, int32_t T,
                 float* out, void* stream);

/* Replaces: MLD._diffusion_reverse(encoder_hidden_states, lengths) (mld.py:290-360) with the
 * initial latents passed in instead of drawn at :303-307 (the caller keeps torch's RNG).
 *   cond        [2B, S_ctx, text_dim] uncond half first (mld.py:225-230) when guidance > 1,
 *               else [B, ...]; int64 [2B,1] for the action model
 *   init_noise  [B, n_lat, d] (or [B, T, nfeats] when diffusion_only)
 *   step_noise  DDPM only (required then): the N(0,1) draws of scheduler.step, [n_steps, B, n_lat, d]
 *               (or [n_steps, B, T, nfeats] when diffusion_only); NULL for DDIM
 *   latents_out [n_lat, B, d]  (mld.py:359)  (or [T, B, nfeats])
 * The n scheduler steps are replayed from one CUDA graph per (B, S_ctx, T) shape (the no-VAE model: one
 * captured step, replayed n times with a device-side step counter). */
int mldb_diffusion_reverse(mldb_handle* h, const void* cond, const float* init_noise,
                           const float* step_noise, const int32_t* lengths, int32_t B,
                           int32_t S_ctx, int32_t T, float* latents_out, void* stream);

/* Replaces: vae.decode(z, lengths) (mld_vae.py:186-248, actor_vae.py:210-235).
 * z [n_lat, B, d]; lengths device int32[B]; feats_out [B, T, nfeats], rows >= length zero. */
int mldb_vae_decode(mldb_handle* h, const float* z, const int32_t* lengths, int32_t B,
                    int32_t T, float* feats_out, void* stream);

/* Replaces: vae.encode(features, lengths) up to the distribution parameters
 * (mld_vae.py:124-178): mu, logvar [n_lat, B, d]; the rsample() at :181-183 stays in torch. */
int mldb_vae_encode(mldb_handle* h, const float* feats, const int32_t* lengths, int32_t B,
                    int32_t T, float* mu, float* logvar, void* stream);

/* Replaces: datamodule.feats2joints(feats) (mld/data/HumanML3D.py:41-45 ->
 * motion_process.py:415-431, 362-381; quaternion.py:16-20,54-73).
 * feats [B, T, 263] -> joints [B, T, njoints, 3]; uses the mean/std set above. */
int mldb_feats2joints(mldb_handle* h, const float* feats, int32_t B, int32_t T,
                      float* joints_out, void* stream);

/* Replaces: MLD.forward(batch) after the text encoder (mld.py:232-264): reverse diffusion ->
 * vae.decode -> feats2joints, replayed as one CUDA graph.  Buffers as above; feats_out and
 * joints_out may each be NULL when not wanted. */
int mldb_sample(mldb_handle* h, const void* cond, const float* init_noise,
                const int32_t* lengths, int32_t B, int32_t S_ctx, int32_t T,
                float* latents_out, float* feats_out, float* joints_out, void* stream);

/* Same as mldb_sample but through HOST buffers (pinned or pageable): copies cond/noise/
 * lengths host->device, runs, copies joints device->host, all on `stream`; returns after
 * enqueue (synchronise the stream before reading joints_host).  This is the call the
 * end-to-end benchmark times.  With a communicator attached joints_host receives the GATHERED motions
 * [nranks * B, T, njoints, 3]. */
int mldb_sample_host(mldb_handle* h, const void* cond_host, const float* init_noise_host,
                     const int32_t* lengths_host, int32_t B, int32_t S_ctx, int32_t T,
                     float* joints_host, void* stream);

/* ---- multi-GPU: batch-sharded replicas + ONE all-gather of the finished motions (SURVEY.md section 8e).
 * One process (handle) per GPU; NCCL is bound at run time (dlopen libnccl.so.2).  Either build the
 * communicator here - rank 0 calls mldb_comm_unique_id, ships the 128 bytes to the other ranks by any means
 * (torch.distributed object broadcast, MPI, a file), every rank calls mldb_comm_init - or attach an existing
 * ncclComm_t with mldb_comm_attach.  The communicator is destroyed with the handle when it was built here. */
int mldb_comm_unique_id(void* out128 /* HOST, 128 bytes */);
int mldb_comm_init(mldb_handle* h, const void* unique_id128, int32_t nranks, int32_t rank);
int mldb_comm_attach(mldb_handle* h, void* nccl_comm, int32_t nranks, int32_t rank);
int mldb_comm_info(const mldb_handle* h, int32_t* nranks, int32_t* rank);
/* ncclAllGather of `count` floats per rank on `stream` (in place when local == global + rank * count). */
int mldb_allgather(mldb_handle* h, const float* local, float* global, int64_t count, void* stream);
/* mldb_sample on this rank's shard, the joints of all ranks gathered into joints_global
 * [nranks * B, T, njoints, 3]: this rank's joints are written straight into its slot and the in-place
 * all-gather runs on a side stream, overlapping whatever is enqueued next on `stream`.  Alternate two
 * joints_global buffers between consecutive calls; mldb_gather_wait makes `stream` wait for the last gather. */
int mldb_sample_gather(mldb_handle* h, const void* cond, const float* init_noise, const int32_t* lengths,
                       int32_t B, int32_t S_ctx, int32_t T, float* joints_global, void* stream);
int mldb_gather_wait(mldb_handle* h, void* stream);

/* Profiling aid used by bench.py's roofline leg: time one operator of denoiser layer 0 in
 * isolation on the (B, S_ctx) workspace (`iters` back-to-back launches between CUDA events on an
 * internal stream; synchronous).  op: "qkv" | "attn" | "outproj_ln" | "ffn1" | "ffn2_ln" | "layer".
 * avg_ms_out: HOST float. */
int mldb_profile_op(mldb_handle* h, const char* op, int32_t B, int32_t S_ctx, int32_t iters,
                    float* avg_ms_out);

/* Profiling aid: device time of every scheduler step of the reverse loop (the kernels of the captured graph
 * launched eagerly on an internal stream with a CUDA event between steps).  ms_out: HOST float[n_steps].
 * Synchronous.  bench.py reports the median as the step p50. */
int mldb_profile_steps(mldb_handle* h, const void* cond, const float* init_noise, int32_t B, int32_t S_ctx,
                       float* ms_out);

/* Debug aid: in-kernel timeline of the wgmma kernels (GEMM / FFN / attention).  enable != 0 starts recording:
 * every warp role of CTA 0 appends {tag | warp << 16 | aux << 24, SM clock} at its pipeline events (tags in the
 * kernels' tl_event calls).  enable == 0 copies the events into out (HOST int64[2 * cap]), sets *count and stops.
 * Process-wide; recording costs one atomic per event in CTA 0 only. */
int mldb_debug_timeline(int32_t enable, int64_t* out, int32_t cap, int32_t* count);

/* Debug aid for the kernel unit tests: y = act(A W^T + b), or LayerNorm(A W^T + b + R) when gamma is
 * given, through the engine's GEMM operators (use_tc: 1 = wgmma path, 0 = CUDA-core path).
 * A [M,K], R [M,N], out [M,N]: fp32 DEVICE; W [N,K], bias/gamma/beta [N]: fp32 HOST.  0 < K1 < K feeds
 * A as two concatenated sources (the skip-connection GEMM).  split_out != 0: the plain epilogue writes
 * split16 planes (the production path; N % 8 == 0) which are then widened to fp32.  Synchronous. */
int mldb_debug_gemm(mldb_handle* h, const float* A, const float* W, const float* bias, const float* gamma,
                    const float* beta, const float* R, int32_t M, int32_t N, int32_t K, int32_t K1,
                    int32_t act, int32_t use_tc, int32_t split_out, float* out, void* stream);

/* Debug aid: one post-norm FFN block y = LayerNorm(x + W2 gelu(W1 x + b1) + b2) through the engine's
 * operators (cross_attention.py:266-271).  mode 0 = CUDA-core kernels, 1 = wgmma GEMMs as two
 * launches, 2 = the fused wgmma FFN kernel.  X, out [M,d]: fp32 DEVICE; W1 [ff,d], W2 [d,ff],
 * b1 [ff], b2/gamma/beta [d]: fp32 HOST.  Synchronous. */
int mldb_debug_ffn(mldb_handle* h, const float* X, const float* W1, const float* b1, const float* W2,
                   const float* b2, const float* gamma, const float* beta, int32_t M, int32_t d, int32_t ff,
                   int32_t mode, float* out, void* stream);

/* Debug aid: the multi-head attention core softmax(Q K^T / sqrt(hd)) V per (sequence, head).
 *   KV == NULL: Q is a packed QKV [nseq*Lq, 3*heads*hd] fp32 DEVICE tensor (q | k | v column blocks, torch
 *               in_proj order; self-attention, Lk == Lq) - the layout the denoiser / VAE stacks use;
 *   KV != NULL: Q [nseq*Lq, heads*hd] and KV [nseq*Lk, 2*heads*hd] (k | v) - cross-attention.
 * lengths (device int32 [nseq], nullable): valid keys per sequence = min(Lk, kv_prefix + lengths[s]).
 * mode 0 = CUDA-core kernel, 1 = mma.sync kernel, 2 = wgmma kernel (product path).
 * out [nseq*Lq, heads*hd] fp32 DEVICE.  Synchronous. */
int mldb_debug_attention(mldb_handle* h, const float* Q, const float* KV, const int32_t* lengths, int32_t kv_prefix,
                         int32_t nseq, int32_t Lq, int32_t Lk, int32_t heads, int32_t hd, int32_t mode, float* out,
                         void* stream);

/* Introspection */
const char* mldb_last_error(void);
int mldb_abi_version(void);
/* number of kernel launches the library has issued (graph replays count their nodes) */
int64_t mldb_launch_count(const mldb_handle* h);
/* Which kernel every operator of the path was ENQUEUED on since the last reset (recorded launches: a CUDA
 * graph counts once, at capture).  out: HOST int64[MLDB_KSTAT_COUNT], index = MLDB_KSTAT_*.  Lets a caller
 * (and the tests) assert that nothing fell back from the wgmma kernels to the CUDA-core kernels. */
#define MLDB_KSTAT_GEMM_TC 0      /* k_gemm_tc, plain epilogue */
#define MLDB_KSTAT_GEMM_LN_TC 1   /* k_gemm_tc, fused residual + LayerNorm epilogue */
#define MLDB_KSTAT_FFN_TC 2       /* k_ffn_tc (fused FFN block) */
#define MLDB_KSTAT_ATTN_TC 3      /* k_attn_tc (wgmma attention) */
#define MLDB_KSTAT_ATTN_MMA 4     /* k_attn_mma (mma.sync attention; option attn=mma) */
#define MLDB_KSTAT_ATTN_SIMT 5    /* k_attn_simt (CUDA cores) */
#define MLDB_KSTAT_GEMM_SIMT 6    /* k_gemm_simt (CUDA cores: odd-K embeddings, time MLP, gemm=simt) */
#define MLDB_KSTAT_LN_SIMT 7      /* k_ln stand-alone LayerNorm (stack-final norms, cross-attention collapse) */
#define MLDB_KSTAT_LN_UNFUSED 8   /* k_ln behind a GEMM whose LayerNorm could NOT be fused (a fallback) */
#define MLDB_KSTAT_MISC 9         /* token assembly, scheduler step, feats2joints, ... */
#define MLDB_KSTAT_COUNT 10
int mldb_kernel_stats(const mldb_handle* h, int64_t* out, int32_t n);
int mldb_reset_kernel_stats(mldb_handle* h);

/* Set an engine option by name.  Options only change HOW the same arithmetic is scheduled; results are
 * identical (gemm, attn: to fp32 re-association noise) for every setting (tests/test_gpu_kernels.py).
 *   "gemm"       "tc" | "simt"          wgmma kernels (default) or the CUDA-core reference kernels  MLDB_GEMM
 *   "attn"       "tc" | "mma" | "simt"  attention core: wgmma (default), mma.sync, CUDA cores       MLDB_ATTN
 *   "ffn_fused"  0 | 1                  fused FFN kernel k_ffn_tc (default 1)                         MLDB_FFN_FUSED
 *   "ffn_split"  0 | 1                  fused FFN: cut the tile groups that do not fill a whole round of the
 *                                        persistent grid along the hidden dimension (default 1; env MLDB_FFN_SPLIT).
 *                                        Results stay bit-identical run to run, but the rows of a split tile are
 *                                        summed in a different order, so they depend on the batch size in the last bits
 *   "branches"   1..4                   concurrent sub-batch branches inside a denoiser step (2)      MLDB_BRANCHES
 *   "graph"      0 | 1                  CUDA-graph replay of the step loop (1)                        MLDB_GRAPH
 * Environment only: MLDB_PDL (programmatic dependent launch, 1); MLDB_SNAKE (1: attention and the fused FFN walk
 * the token tiles downwards, the GEMMs upwards, so every kernel starts on the rows its producer wrote last). */
int mldb_set_option(mldb_handle* h, const char* name, const char* value);

#ifdef __cplusplus
}
#endif
#endif /* MLDB_H_ */
