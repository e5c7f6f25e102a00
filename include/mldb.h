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

#define MLDB_ABI_VERSION 4

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
/* beta schedules (diffusers beta_schedule) */
#define MLDB_BETA_SCALED_LINEAR 0       /* linspace(sqrt(beta_start), sqrt(beta_end), T, fp32) ** 2 */
#define MLDB_BETA_LINEAR 1              /* linspace(beta_start, beta_end, T, fp32) */
#define MLDB_BETA_SQUAREDCOS_CAP_V2 2   /* betas_for_alpha_bar: cosine alpha_bar, double math, max_beta 0.999 */
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
  double  beta_end;           /* 0.012 */
  int32_t steps_offset;       /* DDIM: 1 */
  int32_t set_alpha_to_one;   /* DDIM: 0 */
  float   eta;                /* DDIM: 0.0, in [0, 1].  eta > 0 adds std_dev_t * N(0,1) at every step; the
                                 caller passes those draws as step_noise (the library draws no random numbers).
                                 DDPM ignores it (its steps at t > 0 always add noise). */
  int32_t njoints;            /* 22 (HumanML3D) for feats2joints */
  int32_t beta_schedule;      /* MLDB_BETA_*: scaled_linear (0, the shipped config) */
  int32_t clip_sample;        /* 0; != 0 clamps the predicted x0 to [-1, 1] (DDIM and DDPM) */
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

/* Replaces: scheduler.step(model_output, t, sample, eta=cfg.eta).prev_sample (mld.py:345), with the
 * configured beta_schedule and clip_sample.  `noise` is the injected N(0,1) tensor (diffusers' variance_noise,
 * count floats), required when the step adds noise: DDIM with eta > 0, DDPM at t > 0; else it may be NULL
 * and is not read.  count = number of floats in sample. */
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
 *   step_noise  the N(0,1) draws of scheduler.step, [n_steps, B, n_lat, d] (or [n_steps, B, T, nfeats] when
 *               diffusion_only), slice i for step i.  Required when some step adds noise (DDIM with eta > 0,
 *               DDPM); then only the slices of steps that add noise are read (DDPM: not the last, t == 0).
 *               May be NULL, and is ignored, when no step adds noise (DDIM with eta == 0)
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
 * (mld_vae.py:124-178): mu, logvar [n_lat, B, d]; the rsample() at :181-183 stays in torch.
 * ActorVae (actor_vae.py:62-75,120-170): mu, logvar [1, B, d] (n_lat != 1 is MLDB_ERR_UNSUPPORTED); T + 2 may
 * reach the 5000 rows of its sine PE table.  Its "vae.encoder.*" keys are all or none: a decoder-only state dict
 * finalizes and decodes, and this call then returns MLDB_ERR_STATE; a partial set fails mldb_finalize_weights,
 * which names the first missing key.
 * feats [B, T, nfeats] fp32 device; lengths device int32[B], each in [1, T]; frames past a length must be finite. */
int mldb_vae_encode(mldb_handle* h, const float* feats, const int32_t* lengths, int32_t B,
                    int32_t T, float* mu, float* logvar, void* stream);

/* Replaces: datamodule.feats2joints(feats) (mld/data/HumanML3D.py:41-45 ->
 * motion_process.py:415-431, 362-381; quaternion.py:16-20,54-73).
 * feats [B, T, 263] -> joints [B, T, njoints, 3]; uses the mean/std set above. */
int mldb_feats2joints(mldb_handle* h, const float* feats, int32_t B, int32_t T,
                      float* joints_out, void* stream);

/* Replaces: MLD.forward(batch) after the text encoder (mld.py:232-264): reverse diffusion ->
 * vae.decode -> feats2joints, replayed as one CUDA graph.  Buffers as above; feats_out and
 * joints_out may each be NULL when not wanted.  step_noise as for mldb_diffusion_reverse. */
int mldb_sample(mldb_handle* h, const void* cond, const float* init_noise,
                const int32_t* lengths, int32_t B, int32_t S_ctx, int32_t T,
                float* latents_out, float* feats_out, float* joints_out, void* stream,
                const float* step_noise);

/* Same as mldb_sample but through HOST buffers (pinned or pageable): copies cond/noise/
 * lengths (and step_noise_host when given) host->device, runs, copies joints device->host, all on `stream`;
 * returns after enqueue (synchronise the stream before reading joints_host).  This is the call the
 * end-to-end benchmark times.  With a communicator attached joints_host receives the GATHERED motions
 * [nranks * B, T, njoints, 3]. */
int mldb_sample_host(mldb_handle* h, const void* cond_host, const float* init_noise_host,
                     const int32_t* lengths_host, int32_t B, int32_t S_ctx, int32_t T,
                     float* joints_host, void* stream, const float* step_noise_host);

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
 * joints_global buffers between consecutive calls; mldb_gather_wait makes `stream` wait for the last gather.
 * step_noise is this rank's shard [n_steps, B, n_lat, d] of the global per-step draws (or NULL, as for mldb_sample). */
int mldb_sample_gather(mldb_handle* h, const void* cond, const float* init_noise, const int32_t* lengths,
                       int32_t B, int32_t S_ctx, int32_t T, float* joints_global, void* stream,
                       const float* step_noise);
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
 * split16 planes (the production path; N % 8 == 0) which are then widened to fp32.  Synchronous.
 * R given without gamma selects the residual-add epilogue out = A W^T + b + R (fp32 output, act must be 0 on
 * the wgmma path; R == out runs it in place, as the text tower does).  act: 0 none, 1 GELU, 2 ReLU, 3 SiLU,
 * 4 quick-GELU x * sigmoid(1.702 x) (CLIP), 5 LeakyReLU(0.2) (T2M evaluator).  N up to 4096 runs on the wgmma kernel here. */
int mldb_debug_gemm(mldb_handle* h, const float* A, const float* W, const float* bias, const float* gamma,
                    const float* beta, const float* R, int32_t M, int32_t N, int32_t K, int32_t K1,
                    int32_t act, int32_t use_tc, int32_t split_out, float* out, void* stream);

/* Debug aid: mldb_debug_gemm with the GEMM's whole output placement (mldb_debug_gemm is this with the identity map
 * and a dense [M, N] output).  Row r of the product goes to output row
 *   (r / in_group) * out_group + out_off + r % in_group
 * (in_group = 1 << 30, out_group = out_off = 0: the identity), and columns [out_col0, out_col0 + N) of it:
 *   y[r] = act(A[r] W^T + b + addtab[out_off + r % in_group]);  y[r] = 0 when r % in_group >= zero_lengths[r / in_group]
 * out is a caller-filled fp32 DEVICE [out_rows, out_cols] buffer.  split_out != 0: its cells go into split16 planes
 * before the op, the op writes the planes, and the planes are widened back into out after it, so the cells the op
 * does not address come back as they were whenever they survive the split16 round trip (11 significant bits).
 * split_out == 0: the op writes fp32 at out + out_col0 with leading dimension out_cols.  R (DEVICE, nullable) without
 * gamma: the residual-add epilogue, R laid out like the fp32 output; with gamma: LayerNorm(A W^T + b + R), identity map
 * and out [M, N] only.  a_kind: 0 split16 A, 1 fp32 A, 2 fp32 A through ReLU (1 and 2 run on the CUDA cores only:
 * use_tc must be 0).  vec_f32: the fp32 output may take the wgmma kernel's vectorised epilogue (identity map).
 * Every row and column the map addresses is checked against the buffers.  Synchronous on `stream`. */
typedef struct mldb_gemm_rows_args {
  const float* A;                  /* [M, K] fp32 DEVICE */
  const float* W;                  /* [N, K] fp32 HOST */
  const float* bias;               /* [N] HOST, nullable */
  const float* gamma;              /* [N] HOST, nullable: LayerNorm epilogue */
  const float* beta;               /* [N] HOST */
  const float* R;                  /* DEVICE, nullable */
  int32_t M, N, K, K1;             /* 0 < K1 < K: A as two concatenated sources */
  int32_t act, use_tc, a_kind;
  int32_t in_group, out_group, out_off;
  const float* addtab;             /* [tab_rows, N] HOST, nullable */
  int32_t tab_rows;
  const int32_t* zero_lengths;     /* [ceil(M / in_group)] HOST, nullable */
  int32_t vec_f32, split_out;
  float* out;                      /* [out_rows, out_cols] fp32 DEVICE */
  int32_t out_rows, out_cols, out_col0;
} mldb_gemm_rows_args;
int mldb_debug_gemm_rows(mldb_handle* h, const mldb_gemm_rows_args* a, void* stream);

/* Debug aid: the CUDA-core LayerNorm of every unfused norm,
 *   out[r] = act(LayerNorm(c[i] + res[i] + rowvec[i / rv_group]) * gamma + beta),  i = input row of r:
 *   i = r (in_group == 0) or (r / sel_group) * in_group + r % sel_group (the kept tokens of each sequence).
 * c: fp32 DEVICE [M_in, ldc] (nullable); res: fp32 DEVICE [M_in, d], fed as split16 (nullable); rowvec: fp32 HOST
 * [ceil(M_in / rv_group), d] (nullable); gamma, beta: fp32 HOST [d].  out: caller-filled fp32 DEVICE [M, ld_out];
 * split_out != 0: through split16 planes [M, ld_out] filled from out and widened back, as in mldb_debug_gemm_rows.
 * act: 0 none or 5 LeakyReLU(0.2).  d > 1024 is refused (MLDB_ERR_UNSUPPORTED).  Synchronous on `stream`. */
typedef struct mldb_ln_args {
  const float* c;
  int32_t ldc;
  const float* res;
  const float* rowvec;
  int32_t rv_group;
  const float* gamma;
  const float* beta;
  int32_t M_in, M, d;
  int32_t sel_group, in_group;
  int32_t act, split_out;
  float* out;
  int32_t ld_out;
} mldb_ln_args;
int mldb_debug_ln(mldb_handle* h, const mldb_ln_args* a, void* stream);

/* Debug aid: fp32 rows into a split16 buffer with the GEMM's row map (the condition tokens and the VAE decoder's
 * queries):  X[(r / in_group) * out_group + out_off + r % in_group, n] =
 *   relu?(src[src_bcast ? r % in_group : r, n]) + tab[out_off + r % in_group, n]        for n < d
 * src: fp32 DEVICE [*, ld_src] (nullable: zeros); tab: fp32 HOST [tab_rows, d] (nullable).  out: caller-filled fp32
 * DEVICE [out_rows, out_cols] (d <= out_cols) that goes into the split16 X before the op and is widened back after it.
 * scalar != 0: the one-column-per-thread kernel even where the 128-bit one applies.  Synchronous on `stream`. */
int mldb_debug_rows_to_split(mldb_handle* h, const float* src, int32_t ld_src, int32_t M, int32_t d, int32_t in_group,
                             int32_t out_group, int32_t out_off, int32_t src_bcast, const float* tab, int32_t tab_rows,
                             int32_t relu, int32_t scalar, float* out, int32_t out_rows, int32_t out_cols,
                             void* stream);

/* Debug aid: one post-norm FFN block y = LayerNorm(x + W2 gelu(W1 x + b1) + b2) through the engine's
 * operators (cross_attention.py:266-271).  mode 0 = CUDA-core kernels, 1 = wgmma GEMMs as two
 * launches, 2 = the fused wgmma FFN kernel.  X, out [M,d]: fp32 DEVICE; W1 [ff,d], W2 [d,ff],
 * b1 [ff], b2/gamma/beta [d]: fp32 HOST.  Synchronous. */
int mldb_debug_ffn(mldb_handle* h, const float* X, const float* W1, const float* b1, const float* W2,
                   const float* b2, const float* gamma, const float* beta, int32_t M, int32_t d, int32_t ff,
                   int32_t mode, float* out, void* stream);

/* Debug aid: an encoder layer after its attention, as the stacks run it:
 *   x1 = LayerNorm1(att Wo^T + bo + X),  out = LayerNorm2(x1 + W2 gelu(W1 x1 + b1) + b2)
 * att, X: [M, d] fp32 DEVICE; the weights HOST ([d,d], [ff,d], [d,ff]; biases nullable).  out: [out_rows, d] fp32
 * DEVICE, out_rows >= M: rows >= M go into the output buffer's rows past M before the op and are read back after it
 * (an op must leave them as they were).  mode 0 = CUDA cores, 1 = the two wgmma kernels (out-projection + LN GEMM,
 * then the fused FFN), 2 = one fused launch (the fused FFN with its out-projection prefix; d = 256).  Synchronous
 * on `stream`. */
int mldb_debug_tail(mldb_handle* h, const float* att, const float* X, const float* Wo, const float* bo,
                    const float* gamma1, const float* beta1, const float* W1, const float* b1, const float* W2,
                    const float* b2, const float* gamma2, const float* beta2, int32_t M, int32_t d, int32_t ff,
                    int32_t mode, int32_t out_rows, float* out, void* stream);

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

/* Debug aid: mldb_debug_attention with a causal mask (query i attends to keys j <= i; self-attention only:
 * KV must be NULL, Lq == Lk).  mode 1 (mma.sync) has no causal mask and returns MLDB_ERR_UNSUPPORTED. */
int mldb_debug_attention_causal(mldb_handle* h, const float* Q, const float* KV, const int32_t* lengths,
                                int32_t kv_prefix, int32_t nseq, int32_t Lq, int32_t Lk, int32_t heads, int32_t hd,
                                int32_t mode, float* out, void* stream);

/* ---- CLIP text encoder (MldTextEncoder, mld/models/architectures/mld_clip.py): token ids -> the denoiser's context.
 * The CLIP ViT-L/14 text tower: token + position embedding, `layers` pre-norm blocks (LN1 -> causal self-attention
 * -> + residual, LN2 -> fc1 -> quick-GELU -> fc2 -> + residual), final LayerNorm; pooled mode adds the eos-row
 * gather and text_projection.  The tokenizer stays on the host (Hugging Face's); this path starts at int64 ids. */
#define MLDB_TEXT_ABI_VERSION 1
#define MLDB_TEXT_HIDDEN 0   /* "clip_hidden": text_model(ids).last_hidden_state            [n, L, hidden] */
#define MLDB_TEXT_POOLED 1   /* "clip": get_text_features(ids) (the shipped config)            [n, projection_dim] */
typedef struct mldb_text_config {
  int32_t abi_version;       /* must be MLDB_TEXT_ABI_VERSION */
  int32_t vocab_size;        /* 49408 */
  int32_t max_positions;     /* 77 */
  int32_t hidden;            /* 768 (a multiple of 128, <= 1024) */
  int32_t heads;             /* 12 (head_dim hidden / heads must be 64 or 128 for the wgmma attention) */
  int32_t layers;            /* 12 */
  int32_t ff;                /* 3072 */
  int32_t projection_dim;    /* 768 */
  int32_t eos_token_id;      /* 49407; 2 selects the legacy argmax(ids) pooling rule */
  float   ln_eps;            /* 1e-5 */
} mldb_text_config;
void mldb_default_text_config(mldb_text_config* cfg);
/* Add the text tower's keys to the strict key spec; call after mldb_create, before mldb_finalize_weights.  Keys are
 * "text_encoder." + MldTextEncoder.state_dict() keys of the text tower ("text_encoder.text_model.text_model.encoder.
 * layers.0.self_attn.q_proj.weight", "text_encoder.text_model.text_projection.weight", ...); the position_ids buffer
 * of older checkpoints is not one of them.  q/k/v_proj are packed into one [3 * hidden, hidden] operand at finalize. */
int mldb_text_configure(mldb_handle* h, const mldb_text_config* cfg);
/* Replaces: MldTextEncoder.forward after the tokenizer (mld_clip.py:53-97).
 *   ids  device int64 [n, L], 1 <= L <= max_positions; an id outside [0, vocab_size) yields a NaN row
 *   out  MLDB_TEXT_HIDDEN: [n, L, hidden]; MLDB_TEXT_POOLED: [n, projection_dim]
 * Enqueued eagerly on `stream` (no graph); the workspace grows on demand (outside any capture: synchronises the
 * device when it does).  The GEMMs and the attention count under MLDB_KSTAT_GEMM_TC / ATTN_TC (or the *_SIMT
 * indices with gemm=simt / attn=simt), the row LayerNorms under MLDB_KSTAT_TEXT_LN. */
int mldb_text_encode(mldb_handle* h, const int64_t* ids, int32_t n, int32_t L, int32_t mode, float* out, void* stream);

/* ---- BERT text encoder (MldTextEncoder with a "bert" model path, mld_clip.py:44-46,65-68,83-86): token ids and the
 * attention mask -> last_hidden_state, the denoiser's context.  DistilBERT (the shipped distilbert-base-uncased) or
 * BERT: word + position (+ token-type row 0) embedding and LayerNorm, then `layers` post-norm blocks (non-causal
 * self-attention over the row's real tokens -> + residual -> LayerNorm, lin1 -> exact GELU -> lin2 -> + residual ->
 * LayerNorm).  A handle holds one text tower: this and mldb_text_configure exclude each other (MLDB_ERR_STATE). */
#define MLDB_BERT_ABI_VERSION 1
#define MLDB_BERT_DISTILBERT 0  /* DistilBertModel: keys embeddings.word_embeddings / position_embeddings / LayerNorm,
                                   transformer.layer.{i}.attention.{q,k,v,out}_lin, sa_layer_norm, ffn.lin1 / lin2,
                                   output_layer_norm */
#define MLDB_BERT_BERT 1        /* BertModel: embeddings.{word,position,token_type}_embeddings / LayerNorm,
                                   encoder.layer.{i}.attention.self.{query,key,value}, attention.output.dense /
                                   LayerNorm, intermediate.dense, output.dense / LayerNorm; pooler.dense.* accepted and
                                   not uploaded (it does not reach last_hidden_state) */
typedef struct mldb_bert_config {
  int32_t abi_version;       /* must be MLDB_BERT_ABI_VERSION */
  int32_t family;            /* MLDB_BERT_DISTILBERT | MLDB_BERT_BERT */
  int32_t vocab_size;        /* 30522 */
  int32_t max_positions;     /* 512; 1 .. 512 */
  int32_t type_vocab;        /* BERT: token_type_embeddings rows (2); ignored for DistilBERT */
  int32_t hidden;            /* 768 (a multiple of 128, <= 1024) */
  int32_t heads;             /* 12 (head_dim 64 or 128 runs the wgmma attention) */
  int32_t layers;            /* 6 */
  int32_t ff;                /* 3072 */
  float   ln_eps;            /* 1e-12 */
} mldb_bert_config;
void mldb_default_bert_config(mldb_bert_config* cfg);   /* distilbert-base-uncased */
/* Add the tower's keys to the strict key spec; after mldb_create, before mldb_finalize_weights.  Keys are
 * "text_encoder.text_model." + the Hugging Face model's state_dict() keys ("text_encoder.text_model.transformer.layer.0.
 * attention.q_lin.weight", ...); an embeddings.position_ids buffer is not one of them.  q/k/v are packed into one
 * [3 * hidden, hidden] operand at finalize. */
int mldb_bert_configure(mldb_handle* h, const mldb_bert_config* cfg);
/* Replaces: MldTextEncoder.forward after the tokenizer for "bert" (text_model(**text_inputs).last_hidden_state).
 *   ids      device int64 [n, L], 1 <= L <= max_positions; an id outside [0, vocab_size) yields a NaN row
 *   lengths  device int32 [n], each in [1, L]: row s's attention mask is lengths[s] ones then zeros (right padding);
 *            token types are all zero.  Copied to the host and checked before anything is launched (the call
 *            synchronises `stream`)
 *   out      [n, L, hidden]: every position, padding positions included (a padding query attends to the real keys)
 * Enqueued eagerly on `stream`; the workspace grows on demand (outside any capture: synchronises the device when it
 * does).  Per call: 1 + 2 * layers MLDB_KSTAT_TEXT_LN, 4 * layers GEMMs and `layers` attentions.  The attention is
 * k_attn_tc (ATTN_TC) for L <= 256 and the CUDA-core kernel (ATTN_SIMT) for longer rows. */
int mldb_bert_encode(mldb_handle* h, const int64_t* ids, const int32_t* lengths, int32_t n, int32_t L, float* out,
                     void* stream);

/* ---- T2M evaluator (MLD.t2m_eval, mld/models/modeltype/mld.py:618-708): the movement, motion and text encoders of
 * Guo et al.'s text-motion matching model (mld/models/architectures/t2m_motionenc.py, t2m_textenc.py) whose embeddings
 * feed R-precision, matching score, FID, diversity and MultiModality.  Weights come from finest.tar (keys text_encoder,
 * movement_encoder, motion_encoder), in eval mode (dropout is the identity). */
#define MLDB_T2M_ABI_VERSION 1
#define MLDB_T2M_TEXT 1       /* parts: TextEncoderBiGRUCo      keys "t2m_textencoder."   + its state_dict keys */
#define MLDB_T2M_MOVEMENT 2   /* parts: MovementConvEncoder     keys "t2m_moveencoder."   */
#define MLDB_T2M_MOTION 4     /* parts: MotionEncoderBiGRUCo    keys "t2m_motionencoder." */
typedef struct mldb_t2m_config {
  int32_t abi_version;        /* must be MLDB_T2M_ABI_VERSION */
  int32_t parts;              /* MLDB_T2M_* mask: only these modules' keys are expected (strict) */
  int32_t dim_word;           /* model.t2m_textencoder.dim_word 300 */
  int32_t dim_pos_ohot;       /* dim_pos_ohot 15 */
  int32_t dim_text_hidden;    /* dim_text_hidden 512 (GRU hidden: a multiple of 64, <= 1024) */
  int32_t dim_coemb_hidden;   /* dim_coemb_hidden 512 (text embedding) */
  int32_t dim_pose;           /* movement input_size = DATASET.NFEATS - 4 = 259 */
  int32_t dim_move_hidden;    /* model.t2m_motionencoder.dim_move_hidden 512 (a multiple of 64) */
  int32_t dim_move_latent;    /* dim_move_latent 512 (a multiple of 64) */
  int32_t dim_motion_hidden;  /* dim_motion_hidden 1024 (GRU hidden: a multiple of 64, <= 1024) */
  int32_t dim_motion_latent;  /* dim_motion_latent 512 (motion embedding) */
} mldb_t2m_config;
void mldb_default_t2m_config(mldb_t2m_config* cfg);
/* Add the configured parts' keys to the strict key spec; after mldb_create, before mldb_finalize_weights. */
int mldb_t2m_configure(mldb_handle* h, const mldb_t2m_config* cfg);
/* Replaces: MovementConvEncoder.forward(x) (t2m_motionenc.py:21-25), no length mask (as the reference: every one of
 * the T frames is read, padding frames included).
 *   x    [B, T, dim_pose] with a row stride of ld >= dim_pose floats (ld = 263 passes feats[..., :-4] uncopied), T >= 4
 *   out  [B, (T / 2) / 2, dim_move_latent] */
int mldb_t2m_movement(mldb_handle* h, const float* x, int32_t ld, int32_t B, int32_t T, float* out, void* stream);
/* Replaces: MotionEncoderBiGRUCo.forward(x, m_lens) (t2m_motionenc.py:51-64).
 *   x        [B, L, dim_move_latent];  lengths  device int32 [B], any order, each in [1, L] (values outside are
 *            clamped; the torch module rejects them, as pack_padded_sequence does)
 *   out      [B, dim_motion_latent] */
int mldb_t2m_motion(mldb_handle* h, const float* x, const int32_t* lengths, int32_t B, int32_t L, float* out,
                    void* stream);
/* Replaces: TextEncoderBiGRUCo.forward(word_embs, pos_ohot, cap_lens) (t2m_textenc.py:33-48).
 *   word_embs [B, L, dim_word]; pos_ohot [B, L, dim_pos_ohot]; lengths as above; out [B, dim_coemb_hidden] */
int mldb_t2m_text(mldb_handle* h, const float* word_embs, const float* pos_ohot, const int32_t* lengths, int32_t B,
                  int32_t L, float* out, void* stream);
/* All three run eagerly on `stream` in batch chunks that bound the workspace (which grows on demand, outside any
 * capture, and synchronises the device when it does).  Every sequence is computed independently of the others and
 * of the chunking.  The GEMMs count under MLDB_KSTAT_GEMM_TC (GEMM_SIMT with gemm=simt), the recurrent steps under
 * MLDB_KSTAT_GRU_TC (with gemm=simt: two GEMM_SIMT and one MISC gate kernel per step). */

/* ---- HumanAct12 action classifier (HUMANACTMetrics, mld/models/metrics/gru.py): MotionDiscriminator and
 * MotionDiscriminatorForFID (mld/models/architectures/humanact12_gru.py), whose logits feed the action model's accuracy
 * and whose tanh(linear1) features feed its FID, diversity and multimodality.  nn.GRU(input_size, hidden_size,
 * hidden_layer) -> the output at lengths - 1 -> Linear(hidden_size, 30) -> tanh -> Linear(30, output_size).
 * Keys (strict) under "gru_classifier.": recurrent.{weight_ih,weight_hh,bias_ih,bias_hh}_l{k}, linear1.weight /
 * .bias [30, hidden_size] / [30], linear2.weight / .bias [output_size, 30] / [output_size]. */
#define MLDB_A2M_ABI_VERSION 1
typedef struct mldb_a2m_config {
  int32_t abi_version;        /* must be MLDB_A2M_ABI_VERSION */
  int32_t input_size;         /* 72 (24 joints x 3) */
  int32_t hidden_size;        /* 128; 64 or 128: the layer's split16 W_hh must fit in shared memory */
  int32_t hidden_layer;       /* 2; 1 .. 8 */
  int32_t output_size;        /* 12 action classes */
} mldb_a2m_config;
void mldb_default_a2m_config(mldb_a2m_config* cfg);
/* Add the classifier's keys to the strict key spec; after mldb_create, before mldb_finalize_weights. */
int mldb_a2m_configure(mldb_handle* h, const mldb_a2m_config* cfg);
/* Replaces: MotionDiscriminator.forward / MotionDiscriminatorForFID.forward with an explicit hidden_unit.
 *   x        [B, input_size, T] fp32 (the reference's motion_sequence.reshape(bs, njoints * nfeats, T))
 *   lengths  device int32 [B], each in [1, T]; frames t >= lengths[b] are never read
 *   h0       [hidden_layer, B, hidden_size] fp32, each sequence's own initial state
 *   logits   [B, output_size] (may be NULL);  features  [B, 30] tanh(linear1) (may be NULL)
 * The lengths are copied to the host and checked before anything is launched (the call synchronises `stream`).
 * Runs eagerly on `stream` in batch chunks that bound the workspace (which grows on demand, outside any capture, and
 * synchronises the device when it does); every sequence is computed independently of the others and of the chunking.
 * Each layer is one k_gru_seq_tc launch per chunk (MLDB_KSTAT_GRU_TC) behind its input GEMM (MLDB_KSTAT_GEMM_TC); with
 * gemm=simt, every step is one GEMM_SIMT and one MISC gate kernel. */
int mldb_a2m_classify(mldb_handle* h, const float* x, const int32_t* lengths, const float* h0, int32_t B, int32_t T,
                      float* logits, float* features, void* stream);

/* ---- UESTC action classifier (UESTCMetrics, mld/models/metrics/stgcn.py): STGCN (mld/models/architectures/
 * uestc_stgcn.py) with layout "smpl", strategy "spatial" and edge importance weighting, whose yhat feeds the action
 * model's accuracy and whose pooled features feed its FID, diversity and multimodality.  data_bn -> ten st_gcn blocks
 * (64, 64, 64, 64, 128/s2, 128, 128, 256/s2, 256, 256 channels) -> the mean over (T_out, 24) -> fcn (1 x 1 conv).
 * Keys (strict, 172 with the defaults) under "stgcn_classifier.": A [3, 24, 24]; edge_importance.{0..9} [3, 24, 24];
 * data_bn.{weight,bias,running_mean,running_var} [24 in_channels] and data_bn.num_batches_tracked (0-d, value
 * ignored); for each block i, st_gcn_networks.{i}.gcn.conv.weight [3 C_out, C_in, 1, 1] / .bias [3 C_out],
 * .tcn.0.* and .tcn.3.* (BatchNorm2d(C_out), the same five keys), .tcn.2.weight [C_out, C_out, 9, 1] / .bias [C_out],
 * and for i = 4, 7 .residual.0.weight [C_out, C_in, 1, 1] / .bias [C_out] and .residual.1.* (BatchNorm2d(C_out));
 * fcn.weight [num_class, 256, 1, 1], fcn.bias [num_class].  Every BatchNorm is applied in eval mode (eps 1e-5). */
#define MLDB_STGCN_ABI_VERSION 1
typedef struct mldb_stgcn_config {
  int32_t abi_version;        /* must be MLDB_STGCN_ABI_VERSION */
  int32_t in_channels;        /* 6 (rot6d); 1 .. 64 */
  int32_t num_class;          /* 40 UESTC actions; 1 .. 4096 */
} mldb_stgcn_config;
void mldb_default_stgcn_config(mldb_stgcn_config* cfg);
/* Add the classifier's keys to the strict key spec; after mldb_create, before mldb_finalize_weights. */
int mldb_stgcn_configure(mldb_handle* h, const mldb_stgcn_config* cfg);
/* Replaces: STGCN.forward.
 *   x         [B, 24, in_channels, T] fp32, contiguous (the reference's `motion`)
 *   yhat      [B, num_class] (may be NULL);  features  [B, 256], the pooled features (may be NULL)
 * Padding frames are computed like any other frame (there is no mask, as in the reference).  Runs eagerly on
 * `stream` in batch chunks that bound the workspace (which grows on demand, outside any capture, and synchronises
 * the device when it does); every sequence is computed independently of the others and of the chunking.
 * Kernels per chunk: for each of the ten blocks one graph mix (MLDB_KSTAT_MISC), one gcn GEMM and one k_tconv_tc
 * temporal convolution (both MLDB_KSTAT_GEMM_TC), then one head (MISC): 20 GEMM_TC + 11 MISC.  With gemm=simt, each
 * block runs the mix, the gcn GEMM, an im2col, the temporal-convolution GEMM and a residual + ReLU kernel: 20
 * GEMM_SIMT + 31 MISC per chunk. */
int mldb_stgcn_classify(mldb_handle* h, const float* x, int32_t B, int32_t T, float* yhat, float* features,
                        void* stream);

/* ---- SMPL layer (Rotation2xyz, mld/transforms/rotation2xyz.py, as MLD.a2m_eval calls it: pose_rep "rot6d",
 * glob, translation, zero betas): smplx 0.1.28's SMPLLayer -> lbs(..., pose2rot=False) with the 24 joints of
 * `parents`.  Keys (strict) under "smpl.": v_template [V, 3], posedirs [207, 3 V] (smplx's layout: row 9 (j - 1) + 3 r
 * + c of (R_j - I), column 3 v + c), J_regressor [24, V], lbs_weights [V, 24], parents [24] (parents[0] = -1 and
 * 0 <= parents[j] < j; checked at mldb_finalize_weights).  The rest joints J_regressor v_template are computed once
 * there, in double.  There is no CUDA-core twin of this path: option gemm=simt does not apply to it (the float64
 * oracle is its yardstick). */
#define MLDB_SMPL_ABI_VERSION 1
#define MLDB_SMPL_JOINTS 0      /* jointstype "smpl": the 24 posed joints, joint 0 subtracted per frame */
#define MLDB_SMPL_VERTICES 1    /* jointstype "vertices": the V skinned vertices */
typedef struct mldb_smpl_config {
  int32_t abi_version;        /* must be MLDB_SMPL_ABI_VERSION */
  int32_t num_vertices;       /* V: 6890 (SMPL); 1 .. 2^20 */
} mldb_smpl_config;
void mldb_default_smpl_config(mldb_smpl_config* cfg);
/* Add the model's keys to the strict key spec; after mldb_create, before mldb_finalize_weights. */
int mldb_smpl_configure(mldb_handle* h, const mldb_smpl_config* cfg);
/* Replaces: Rotation2xyz.__call__(x, mask, pose_rep="rot6d", translation=True, glob=True, jointstype, vertstrans).
 *   feats       [B, T, 150] fp32: frame t's joint j rotation at feats[b, t, c * 25 + j] (c < 6, j < 24), its translation
 *               at feats[b, t, c * 25 + 24] (c < 3) - MLD's sample.view(B, T, 6, 25) before the permute
 *   mask        device uint8 [B, T] (any pattern; 0: the frame's features are never read and its output is zero before
 *               the translation), or NULL for every frame
 *   jointstype  MLDB_SMPL_JOINTS -> out [B, 24, 3, T];  MLDB_SMPL_VERTICES -> out [B, V, 3, T]
 *   vertstrans  1: every frame, masked or not, gets trans[t] - trans[0] of its sequence added (as the reference)
 * The arguments are checked on the host before anything is launched.  Runs eagerly on `stream`; the vertex path's
 * workspace grows on demand (outside any capture, synchronising the device when it does) and long batches run in
 * chunks of whole sequences (option smpl_chunk); every sequence is computed independently of the others and of the
 * chunking.  Kernels: one k_smpl_fk (MLDB_KSTAT_MISC) per chunk, and for the vertices one
 * k_smpl_lbs (MLDB_KSTAT_GEMM_TC: the split16 pose-blend GEMM with skinning in its epilogue). */
int mldb_smpl_forward(mldb_handle* h, const float* feats, const uint8_t* mask, int32_t B, int32_t T,
                      int32_t jointstype, int32_t vertstrans, float* out, void* stream);

/* ---- APE / AVE of the text-to-motion test (TemosMetric: ComputeMetrics.update, mld/models/metrics/compute.py, with
 * the Rifke round trip of transforms/joints2jfeats/rifke.py).  Needs no weights and no finalize: any handle runs it.
 * The joint tables (mld/utils/joints.py) and the meter factors live in the library. */
#define MLDB_APE_AVE_ABI_VERSION 1
#define MLDB_JOINTS_HUMANML3D 0   /* J = 22, force_in_meter factor 1000 * 0.75 / 480 */
#define MLDB_JOINTS_MMM 1         /* KIT: J = 21, factor 1000 */
/* Replaces: the per-batch increments of ComputeMetrics.update(jts_text, jts_ref, lengths).
 *   jts_text, jts_ref  [B, T, J, 3] fp32, padded to T; every frame, padding included, enters the floor (softmin of
 *                      the lowest foot height), as in the reference
 *   lengths            device int32 [B], each in [2, T] (the caller checks them: a sequence whose length is not
 *                      gives NaN in every output)
 *   force_in_meter     1: positions divided by the jointstype's factor; 0: by 1
 *   out                fp32 [4 J + 2], in ComputeMetrics.metrics order: APE_root [1], APE_traj [1], APE_pose [J - 1],
 *                      APE_joints [J], AVE_root [1], AVE_traj [1], AVE_pose [J - 1], AVE_joints [J]: the sums over
 *                      the batch that update adds to the metric's states
 * The arguments are checked on the host before anything is launched.  Enqueued on `stream` with no host
 * synchronisation; the handle's partial-row workspace is allocated once, at the first call.  Two kernels
 * (MLDB_KSTAT_MISC): k_ape_ave, one CTA per sequence in double, and k_ape_ave_reduce, the fixed-order sum over the
 * batch, so a call gives the same bits every time. */
int mldb_ape_ave(mldb_handle* h, const float* jts_text, const float* jts_ref, const int32_t* lengths, int32_t B,
                 int32_t T, int32_t J, int32_t jointstype, int32_t force_in_meter, float* out, void* stream);

/* Introspection */
const char* mldb_last_error(void);
int mldb_abi_version(void);
/* number of kernel launches the library has issued (graph replays count their nodes) */
int64_t mldb_launch_count(const mldb_handle* h);
/* Which kernel every operator of the path was ENQUEUED on since the last reset (recorded launches: a CUDA
 * graph counts once, at capture).  out: HOST int64[MLDB_KSTAT_COUNT], index = MLDB_KSTAT_*.  Lets a caller
 * (and the tests) assert that nothing fell back from the wgmma kernels to the CUDA-core kernels. */
#define MLDB_KSTAT_GEMM_TC 0      /* k_gemm_tc, plain epilogue; k_proj_tc (its K = 256 split16 projections);
                                     k_tconv_tc (the UESTC classifier's temporal convolutions); k_smpl_lbs (the SMPL
                                     layer's pose-blend GEMM + skinning) */
#define MLDB_KSTAT_GEMM_LN_TC 1   /* k_gemm_tc, fused residual + LayerNorm epilogue */
#define MLDB_KSTAT_FFN_TC 2       /* k_ffn_tc (fused FFN block; in the encoder layers it also runs the folded
                                     out-projection + residual + LayerNorm in front of the FFN) */
#define MLDB_KSTAT_ATTN_TC 3      /* k_attn_tc (wgmma attention) */
#define MLDB_KSTAT_ATTN_MMA 4     /* k_attn_mma (mma.sync attention; option attn=mma) */
#define MLDB_KSTAT_ATTN_SIMT 5    /* k_attn_simt (CUDA cores) */
#define MLDB_KSTAT_GEMM_SIMT 6    /* k_gemm_simt (CUDA cores: odd-K embeddings, time MLP, gemm=simt) */
#define MLDB_KSTAT_LN_SIMT 7      /* k_ln stand-alone LayerNorm (stack-final norms, cross-attention collapse) */
#define MLDB_KSTAT_LN_UNFUSED 8   /* k_ln behind a GEMM whose LayerNorm could NOT be fused (a fallback) */
#define MLDB_KSTAT_MISC 9         /* token assembly, scheduler step, feats2joints, k_smpl_fk, ... */
#define MLDB_KSTAT_TEXT_LN 10     /* k_text_ln: the text tower's row LayerNorm (+ embedding / eos gather) */
#define MLDB_KSTAT_GRU_TC 11      /* k_gru_step_tc: one recurrent step of the T2M evaluator's bidirectional GRU;
                                     k_gru_seq_tc: one whole layer of the action classifier's GRU */
#define MLDB_KSTAT_COUNT 12
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
 *   "t2m_chunk"  0 | n                  T2M evaluator: sequences per batch chunk (0: sized from the workspace budget)
 *   "a2m_chunk"  0 | n                  action classifier: sequences per batch chunk (0: from the workspace budget)
 *   "stgcn_chunk" 0 | n                 UESTC classifier: sequences per batch chunk (0: from the workspace budget)
 *   "smpl_chunk" 0 | n                  SMPL layer: sequences per batch chunk (0: from the vertex path's workspace budget;
 *                                        the joint path needs no workspace and then runs unchunked)
 * Environment only: MLDB_PDL (programmatic dependent launch, 1); MLDB_SNAKE (1: attention and the fused FFN walk
 * the token tiles downwards, the GEMMs upwards, so every kernel starts on the rows its producer wrote last). */
int mldb_set_option(mldb_handle* h, const char* name, const char* value);

#ifdef __cplusplus
}
#endif
#endif /* MLDB_H_ */
