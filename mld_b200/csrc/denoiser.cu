// The denoisers (trans_enc on the VAE latents, trans_dec on the motion itself), the reverse-diffusion loop and the
// sampling entry points.
#include "engine.h"

#include <algorithm>

#include "misc_kernels.cuh"

// ----------------------------------------------------------------------------- denoiser (trans_enc)
// Gather + place the action tokens (EmbedAction.forward, mld_denoiser.py:250-262): rows of the
// first (uncond) half are zero when guidance is on.
__global__ void k_action_tokens(ActBuf X, int Ntok, int Bx, int pos, int d, const int64_t* __restrict__ ids,
                                const float* __restrict__ table, int nclasses, int cfg_on,
                                const float* __restrict__ pe_row) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)Bx * d) return;
  const int n = (int)(idx % d), s = (int)(idx / d);
  float v = 0.0f;
  if (!(cfg_on && s < Bx / 2)) {
    int64_t id = ids[s];
    id = id < 0 ? 0 : (id >= nclasses ? nclasses - 1 : id);
    v = table[id * d + n];
  }
  v += pe_row[n];
  __half hh, ll;
  split_f32(v, hh, ll);
  const int64_t o = ((int64_t)s * Ntok + pos) * X.cols + n;
  X.hi[o] = hh;
  X.lo()[o] = ll;
}

int enc_plan(mldb_handle* h, PlanKind kind, int B, int Bx, int S, Plan** out) {
  Plan* p = find_plan(h, kind, B, S, 0);
  if (!p) {
    const mldb_config& c = h->cfg;
    p = add_plan(h, kind, B, S, 0);
    p->Bx = Bx;
    const int Sc = c.cond_kind == MLDB_COND_TEXT ? S : 1;
    p->Ntok = c.n_lat + 1 + Sc;
    if (p->Ntok > 500) FAIL(MLDB_ERR_INVALID, "sequence of %d tokens exceeds the learned PE table (500)", p->Ntok);
    TRY(alloc_stack_ws(h, h->den, Bx, p->Ntok, 0, &p->ws, h->den.layers >= 3 ? c.n_lat : 0));
    const size_t per = (size_t)c.n_lat * c.latent_dim;
    TRY(dev_alloc(h, (void**)&p->latents, (size_t)B * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->eps, (size_t)Bx * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->tt_single, (size_t)3 * std::max(c.text_dim, c.latent_dim) * sizeof(float) + 64));
    if (c.cond_kind == MLDB_COND_TEXT && c.text_dim != c.latent_dim)
      TRY(alloc_act(h, Bx * S, c.text_dim, &p->ctx_split));
  }
  *out = p;
  return MLDB_OK;
}

// condition tokens -> X0 (once per batch; step invariant, hoisted out of the loop although the
// reference recomputes emb_proj every step, mld_denoiser.py:165)
int place_condition(mldb_handle* h, Plan* p, const void* cond, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim, Bx = p->Bx;
  if (c.cond_kind == MLDB_COND_TEXT) {
    const int S = p->S;
    if (c.text_dim != d) {
      // emb_proj = ReLU -> Linear (mld_denoiser.py:67-68): ReLU + hi/lo split in one pass over the
      // CLIP context, then the tensor-core GEMM writes the tokens (+ PE) straight into X0
      GemmArgs g; g.M = Bx * S; g.w = h->emb_proj; g.out = p->ws.x0;
      g.in_group = S; g.out_group = p->Ntok; g.out_off = c.n_lat + 1; g.addtab = h->query_pe;
      if (h->use_tc && p->ctx_split.hi && c.text_dim % 64 == 0) {
        rows_to_split(h, p->ctx_split, (const float*)cond, c.text_dim, Bx * S, c.text_dim, 1 << 30, 0, 0, 0, nullptr, 1, st);
        g.a1 = p->ctx_split; g.K1 = c.text_dim;
      } else {
        g.a_kind = A_F32_RELU; g.a_f32 = (const float*)cond; g.lda = c.text_dim;
      }
      op_gemm(h, g, st);
    } else {
      rows_to_split(h, p->ws.x0, (const float*)cond, d, Bx * S, d, S, p->Ntok, c.n_lat + 1, 0, h->query_pe, 0, st);
    }
  } else {
    const int cfg_on = c.guidance_scale > 1.0f;
    k_action_tokens<<<nblk((int64_t)Bx * d), 256, 0, st>>>(p->ws.x0, p->Ntok, Bx, c.n_lat + 1, d, (const int64_t*)cond,
                                                          h->action_emb, c.nclasses, cfg_on,
                                                          h->query_pe + (size_t)(c.n_lat + 1) * d);
    kcount(h, MLDB_KSTAT_MISC);
  }
  CK(cudaGetLastError());
  return MLDB_OK;
}

// the stack + final norm over the n sequences of workspace (slice) wsv: eps[n, n_lat*d]
static void denoiser_range(mldb_handle* h, Plan* p, const StackWs& wsv, int n, float* eps, cudaStream_t s) {
  const mldb_config& c = h->cfg;
  SeqInfo si;
  StackWs w = wsv;
  ActBuf x = run_stack(h, h->den, w.x0, ActBuf{}, w, si, s);
  // encoder.norm on the latent tokens only (cross_attention.py:62-63, mld_denoiser.py:206)
  LnArgs l; l.res = x; l.gamma = h->den.norm.g; l.beta = h->den.norm.b; l.M = n * c.n_lat; l.d = c.latent_dim;
  if (w.n_sel == 0) { l.sel_group = c.n_lat; l.in_group = p->Ntok; }   // else x is already compact
  l.out_f32 = eps; l.ld_out = c.latent_dim;
  op_ln(h, l, s);
}

// one denoiser pass over the assembled tokens: eps[Bx, n_lat*d] = norm(stack(X0))[:n_lat]
void denoiser_pass(mldb_handle* h, Plan* p, const float* latents, int lat_mod, const float* tt, float* eps_out,
                   cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim;
  launch_pdl(k_assemble_tokens, dim3(nblk((int64_t)p->Bx * (c.n_lat + 1) * d)), dim3(256), 0, st,
             p->ws.x0, p->Ntok, p->Bx, lat_mod, c.n_lat, d, latents, (const float*)h->query_pe, tt);
  kcount(h, MLDB_KSTAT_MISC);
  // Sequences are independent: the stack runs as `branches` contiguous sequence ranges with their own
  // workspace rows on parallel streams (parallel chains inside the captured graph).
  const int nbr = (h->branches > 1 && p->Bx * p->Ntok >= 2 * 128 * h->branches) ? h->branches : 1;
  if (nbr == 1) {
    denoiser_range(h, p, p->ws, p->Bx, eps_out, st);
    return;
  }
  // fork: every range waits for the token assembly; join: the caller's stream waits for every range
  cudaEventRecord(h->ev_fork, st);
  for (int k = 0; k < nbr; ++k) {
    cudaStream_t s = k == 0 ? st : h->br_stream[k - 1];
    if (k) cudaStreamWaitEvent(s, h->ev_fork, 0);
    const int s0 = (int)((int64_t)p->Bx * k / nbr), s1 = (int)((int64_t)p->Bx * (k + 1) / nbr);
    denoiser_range(h, p, ws_slice(p->ws, s0, s1 - s0), s1 - s0, eps_out + (size_t)s0 * c.n_lat * d, s);
    if (k) cudaEventRecord(h->ev_join[k - 1], s);
  }
  for (int k = 1; k < nbr; ++k) cudaStreamWaitEvent(st, h->ev_join[k - 1], 0);
}

// ----------------------------------------------------------------------------- denoiser (trans_dec)
// The no-VAE model (configs/modules_novae/denoiser.yaml): frames are the decoder targets, the
// memory is [time, text...] (mld_denoiser.py:208-221).  No key-padding mask is passed on either
// attention (padded frames attend and are attended, like the reference); padded output frames are
// zeroed after pose_proj (:219-221).
static int decden_plan(mldb_handle* h, PlanKind kind, int B, int Bx, int S, int T, Plan** out) {
  Plan* p = find_plan(h, kind, B, S, T);
  if (!p) {
    const mldb_config& c = h->cfg;
    if (T > 500 || 1 + S > 500) FAIL(MLDB_ERR_INVALID, "sequence exceeds the learned PE table (500)");
    p = add_plan(h, kind, B, S, T);
    p->Bx = Bx;
    p->Ntok = T;
    const int Lmem = 1 + (c.cond_kind == MLDB_COND_TEXT ? S : 1);
    TRY(alloc_stack_ws(h, h->den, Bx, T, Lmem, &p->ws));
    TRY(alloc_act(h, Bx * Lmem, c.latent_dim, &p->mem));
    const size_t per = (size_t)T * c.nfeats;
    TRY(dev_alloc(h, (void**)&p->latents, (size_t)B * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->eps, (size_t)Bx * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->stage_f32, (size_t)Bx * per * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->lengths, (size_t)Bx * sizeof(int32_t)));
    TRY(dev_alloc(h, (void**)&p->tt_single, (size_t)3 * std::max(c.text_dim, c.latent_dim) * sizeof(float) + 64));
    TRY(dev_alloc(h, (void**)&p->d_step, sizeof(int)));
    if (h->pose_embd.K % 64 == 0 && h->pose_embd.K >= c.nfeats) TRY(alloc_act(h, Bx * T, h->pose_embd.K, &p->in_split));
  }
  *out = p;
  return MLDB_OK;
}

static int place_condition_dec(mldb_handle* h, Plan* p, const void* cond, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim, Bx = p->Bx, Lmem = p->ws.Lmem;
  if (c.cond_kind == MLDB_COND_TEXT) {
    const int S = p->S;
    if (c.text_dim != d) {
      GemmArgs g; g.a_kind = A_F32_RELU; g.a_f32 = (const float*)cond; g.lda = c.text_dim;
      g.M = Bx * S; g.w = h->emb_proj; g.out = p->mem;
      g.in_group = S; g.out_group = Lmem; g.out_off = 1; g.addtab = h->mem_pe;
      op_gemm(h, g, st);
    } else {
      rows_to_split(h, p->mem, (const float*)cond, d, Bx * S, d, S, Lmem, 1, 0, h->mem_pe, 0, st);
    }
  } else {
    const int cfg_on = c.guidance_scale > 1.0f;
    k_action_tokens<<<nblk((int64_t)Bx * d), 256, 0, st>>>(p->mem, Lmem, Bx, 1, d, (const int64_t*)cond, h->action_emb,
                                                          c.nclasses, cfg_on, h->mem_pe + (size_t)d);
    kcount(h, MLDB_KSTAT_MISC);
  }
  CK(cudaGetLastError());
  return MLDB_OK;
}

// model_in: [rows_in, T, F] fp32 (device) fed `rep` times (rep * rows_in == Bx: torch.cat([latents] * 2),
// mld.py:325); lengths: device int32[Bx]; eps_out [Bx, T, F].  tt: time token(s); step_ptr != null selects
// row *step_ptr of tt (replayed step graph).
static void denoiser_pass_dec(mldb_handle* h, Plan* p, const float* model_in, int rep, const float* tt,
                              const int* step_ptr, float* eps_out, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int d = c.latent_dim, Bx = p->Bx, T = p->T, F = c.nfeats, Lmem = p->ws.Lmem;
  // memory row 0 = time token (mem_pos.pe[0] already added)
  k_rows_to_split<<<nblk((int64_t)Bx * d), 256, 0, st>>>(p->mem, tt, d, Bx, d, 1, Lmem, 0, 1, nullptr, 0, step_ptr, (int64_t)d);
  kcount(h, MLDB_KSTAT_MISC);
  // pose_embd + query_pos (mld_denoiser.py:210,214): the 263 features zero-padded to the packed K (320)
  // so that the embedding runs on the tensor cores
  GemmArgs g; g.M = Bx * T; g.w = h->pose_embd;
  g.out = p->ws.x0; g.in_group = T; g.out_group = T; g.out_off = 0; g.addtab = h->query_pe;
  if (h->use_tc && p->in_split.hi) {
    k_f32_to_split_pad<<<nblk((int64_t)(Bx / rep) * T * p->in_split.cols), 256, 0, st>>>(p->in_split, model_in, F, (Bx / rep) * T, F, rep);
    kcount(h, MLDB_KSTAT_MISC);
    g.a1 = p->in_split; g.K1 = p->in_split.cols;
  } else {
    if (rep > 1) {   // CUDA-core reference path: materialise the duplicated input
      for (int k = 0; k < rep; ++k)
        cudaMemcpyAsync(p->stage_f32 + (size_t)k * (Bx / rep) * T * F, model_in, (size_t)(Bx / rep) * T * F * sizeof(float),
                        cudaMemcpyDeviceToDevice, st);
      model_in = p->stage_f32;
    }
    g.a_kind = A_F32; g.a_f32 = model_in; g.lda = F;
  }
  op_gemm(h, g, st);
  SeqInfo si;
  ActBuf x = run_stack(h, h->den, p->ws.x0, p->mem, p->ws, si, st);
  LnArgs l; l.res = x; l.gamma = h->den.norm.g; l.beta = h->den.norm.b; l.M = Bx * T; l.d = d; l.out = p->ws.x1;
  op_ln(h, l, st);
  GemmArgs go; go.a1 = p->ws.x1; go.K1 = d; go.M = Bx * T; go.w = h->pose_proj; go.out_f32 = eps_out; go.ldc = F;
  go.in_group = T; go.out_group = T; go.out_off = 0; go.zero_lengths = p->lengths;
  op_gemm(h, go, st);
}

__global__ void k_dup_lengths(const int32_t* __restrict__ src, int32_t* __restrict__ dst, int B, int Bx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Bx) dst[i] = src[i % B];
}

extern "C" int mldb_denoise(mldb_handle* h, const float* sample, int64_t timestep, const void* cond,
                            const int32_t* lengths, int32_t Bx, int32_t S_ctx, int32_t T, float* out,
                            void* stream) {
  (void)lengths; (void)T;
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!sample || !cond || !out || Bx <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  const mldb_config& c = h->cfg;
  if (c.num_layers == 0) FAIL(MLDB_ERR_STATE, "this handle has no denoiser");
  if (c.cond_kind == MLDB_COND_TEXT && S_ctx <= 0) FAIL(MLDB_ERR_INVALID, "S_ctx must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  Plan* p = nullptr;
  if (c.arch == MLDB_ARCH_TRANS_DEC) {
    if (!c.diffusion_only) FAIL(MLDB_ERR_UNSUPPORTED, "arch trans_dec is built for the no-VAE model (diffusion_only)");
    if (!lengths || T <= 0) FAIL(MLDB_ERR_INVALID, "the no-VAE denoiser needs lengths and T");
    TRY(decden_plan(h, PLAN_DENOISE_DEC, Bx, Bx, S_ctx, T, &p));
    TRY(place_condition_dec(h, p, cond, st));
    CK(cudaMemcpyAsync(p->lengths, lengths, (size_t)Bx * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    const int d = c.latent_dim;
    const int tdim = c.cond_kind == MLDB_COND_TEXT ? c.text_dim : d;
    float* feats = p->tt_single + 16;
    float* hid = feats + tdim;
    float* tt = hid + std::max(tdim, d);
    TRY(time_tokens(h, nullptr, timestep, 1, h->mem_pe, tt, feats, hid, st));
    denoiser_pass_dec(h, p, sample, 1, tt, nullptr, out, st);
    return ops_done(h);
  }
  TRY(enc_plan(h, PLAN_DENOISE, Bx, Bx, S_ctx, &p));
  TRY(place_condition(h, p, cond, st));
  // time token for this timestep
  const int d = c.latent_dim;
  const int tdim = c.cond_kind == MLDB_COND_TEXT ? c.text_dim : d;
  float* feats = p->tt_single + 16;
  float* hid = feats + tdim;
  float* tt = hid + std::max(tdim, d);
  TRY(time_tokens(h, nullptr, timestep, 1, h->query_pe + (size_t)c.n_lat * d, tt, feats, hid, st));
  denoiser_pass(h, p, sample, Bx, tt, out, st);
  return ops_done(h);
}

// Does some step of the current timestep schedule add noise (non-zero std / sigma)?
static bool steps_add_noise(const mldb_handle* h) {
  for (const StepCoef& k : h->coefs_host)
    if (k.sigma != 0.0f) return true;
  return false;
}

static int run_reverse(mldb_handle* h, const void* cond, const float* init_noise, const float* step_noise,
                       const int32_t* lengths, int B, int S, int T, float* latents_out, cudaStream_t st,
                       Plan** plan_out) {
  const mldb_config& c = h->cfg;
  if (c.num_layers == 0) FAIL(MLDB_ERR_STATE, "this handle has no denoiser");
  const bool cfg_on = c.guidance_scale > 1.0f;
  const int Bx = cfg_on ? 2 * B : B;
  if (c.arch == MLDB_ARCH_TRANS_DEC) {
    // no-VAE model: latents are the motion itself, [B, T, F]; DDPM (and DDIM with eta > 0) adds noise at
    // its steps, which the caller injects (step_noise [n_steps, B, T, F]).  One captured step, replayed.
    if (!c.diffusion_only) FAIL(MLDB_ERR_UNSUPPORTED, "arch trans_dec is built for the no-VAE model (diffusion_only)");
    if (!lengths || T <= 0) FAIL(MLDB_ERR_INVALID, "the no-VAE model needs lengths and T");
    const int nsteps = (int)h->timesteps.size();
    const bool needs_noise = steps_add_noise(h);
    if (needs_noise && !step_noise)
      FAIL(MLDB_ERR_INVALID, "this scheduler adds noise at its steps (%s): pass step_noise [%d, %d, %d, %d] (N(0,1) per step)",
           c.sched_kind == MLDB_SCHED_DDIM ? "DDIM eta > 0" : "DDPM", nsteps, B, T, c.nfeats);
    Plan* p = nullptr;
    TRY(decden_plan(h, PLAN_REVERSE_DEC, B, Bx, S, T, &p));
    const int64_t per = (int64_t)T * c.nfeats;
    TRY(place_condition_dec(h, p, cond, st));
    k_dup_lengths<<<nblk(Bx), 256, 0, st>>>(lengths, p->lengths, B, Bx);
    kcount(h, MLDB_KSTAT_MISC);
    CK(cudaMemcpyAsync(p->latents, init_noise, (size_t)B * per * sizeof(float), cudaMemcpyDeviceToDevice, st));
    // ONE captured step, replayed n_steps times: the step index lives on the device (k_step_inc), the
    // kernels that depend on it (time token, scheduler coefficients, noise slice) read it through p->d_step.
    // The graph holds the caller's noise pointer: a different buffer re-captures.
    if (p->noise_ptr != step_noise && p->exec) { cudaGraphExecDestroy(p->exec); p->exec = nullptr; }
    p->noise_ptr = step_noise;
    k_step_set<<<1, 1, 0, st>>>(p->d_step, 0);
    kcount(h, MLDB_KSTAT_MISC);
    for (int i = 0; i < nsteps; ++i) {
      TRY(run_graphed(h, p, st, [&](cudaStream_t s) {
        denoiser_pass_dec(h, p, p->latents, cfg_on ? 2 : 1, h->d_tt, p->d_step, p->eps, s);
        k_cfg_sched<<<nblk(B * per), 256, 0, s>>>(p->eps, p->latents, needs_noise ? step_noise : nullptr, B * per,
                                                cfg_on ? 1 : 0, c.guidance_scale, h->d_coefs, 0, p->d_step);
        kcount(h, MLDB_KSTAT_MISC);
        k_step_inc<<<1, 1, 0, s>>>(p->d_step);
        kcount(h, MLDB_KSTAT_MISC);
      }));
    }
    if (latents_out) {                                        // [T, B, F] (mld.py:359)
      k_permute_01<<<nblk(B * per), 256, 0, st>>>(p->latents, latents_out, B, T, c.nfeats);
      kcount(h, MLDB_KSTAT_MISC);
    }
    CK(cudaGetLastError());
    if (plan_out) *plan_out = p;
    return MLDB_OK;
  }
  Plan* p = nullptr;
  TRY(enc_plan(h, PLAN_REVERSE, B, Bx, S, &p));
  const int d = c.latent_dim;
  const int64_t per = (int64_t)c.n_lat * d;
  TRY(place_condition(h, p, cond, st));
  // latents = init_noise * init_noise_sigma (== 1 for DDIM/DDPM), mld.py:310
  CK(cudaMemcpyAsync(p->latents, init_noise, (size_t)B * per * sizeof(float), cudaMemcpyDeviceToDevice, st));
  const int nsteps = (int)h->timesteps.size();
  // DDPM (every step with t > 0) and DDIM with eta > 0 (every step) add std * N(0,1) (diffusers
  // scheduler.step draws it): the caller injects the draws
  const float* nz_all = nullptr;
  if (steps_add_noise(h)) {
    if (!step_noise)
      FAIL(MLDB_ERR_INVALID, "this scheduler adds noise at its steps (%s): pass step_noise [%d, %d, %d, %d] (N(0,1) per step)",
           c.sched_kind == MLDB_SCHED_DDIM ? "DDIM eta > 0" : "DDPM", nsteps, B, c.n_lat, d);
    if (p->noise_cap < (size_t)nsteps * B * per) {
      TRY(dev_alloc(h, (void**)&p->step_noise, (size_t)nsteps * B * per * sizeof(float)));
      p->noise_cap = (size_t)nsteps * B * per;
      if (p->exec) { cudaGraphExecDestroy(p->exec); p->exec = nullptr; }   // the graph holds the old pointer
    }
    CK(cudaMemcpyAsync(p->step_noise, step_noise, (size_t)nsteps * B * per * sizeof(float), cudaMemcpyDeviceToDevice, st));
    nz_all = p->step_noise;
  }
  TRY(run_graphed(h, p, st, [&](cudaStream_t s) {
    for (int i = 0; i < nsteps; ++i) {                                           // mld.py:323
      denoiser_pass(h, p, p->latents, B, h->d_tt + (size_t)i * d, p->eps, s);
      launch_pdl(k_cfg_sched, dim3(nblk(B * per)), dim3(256), 0, s, (const float*)p->eps, p->latents,
                 nz_all, (int64_t)(B * per), cfg_on ? 1 : 0, c.guidance_scale, (const StepCoef*)h->d_coefs, i,
                 (const int*)nullptr);
      kcount(h, MLDB_KSTAT_MISC);
    }
  }));
  if (latents_out) {                                                             // mld.py:359
    k_permute_01<<<nblk(B * per), 256, 0, st>>>(p->latents, latents_out, B, c.n_lat, d);
    kcount(h, MLDB_KSTAT_MISC);
  }
  CK(cudaGetLastError());
  if (plan_out) *plan_out = p;
  return MLDB_OK;
}

extern "C" int mldb_diffusion_reverse(mldb_handle* h, const void* cond, const float* init_noise,
                                      const float* step_noise, const int32_t* lengths, int32_t B,
                                      int32_t S_ctx, int32_t T, float* latents_out, void* stream) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!cond || !init_noise || !latents_out || B <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  return run_reverse(h, cond, init_noise, step_noise, lengths, B, S_ctx, T, latents_out, (cudaStream_t)stream, nullptr);
}

// ----------------------------------------------------------------------------- full sample
extern "C" int mldb_sample(mldb_handle* h, const void* cond, const float* init_noise,
                           const int32_t* lengths, int32_t B, int32_t S_ctx, int32_t T,
                           float* latents_out, float* feats_out, float* joints_out, void* stream,
                           const float* step_noise) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!cond || !init_noise || !lengths || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  Plan *rp = nullptr, *dp = nullptr;
  TRY(dec_plan(h, B, T, &dp));
  const mldb_config& c = h->cfg;
  // reverse diffusion writes [n_lat, B, d] into the decode plan's staging buffer
  float* z = latents_out;
  if (!z) {
    if (!dp->stage_f32) TRY(dev_alloc(h, (void**)&dp->stage_f32, (size_t)B * c.n_lat * c.latent_dim * sizeof(float)));
    z = dp->stage_f32;
  }
  if (c.arch != MLDB_ARCH_TRANS_ENC) FAIL(MLDB_ERR_UNSUPPORTED, "mldb_sample is built for the latent (VAE) models");
  TRY(run_reverse(h, cond, init_noise, step_noise, lengths, B, S_ctx, T, z, st, &rp));
  TRY(run_decode(h, z, lengths, B, T, feats_out, st, &dp));
  if (joints_out) TRY(run_f2j(h, feats_out ? feats_out : dp->feats, B, T, joints_out, st));
  return MLDB_OK;
}

// Multi-GPU: this rank samples its shard and the finished joints of every rank are gathered into
// joints_global [nranks * B, T, njoints, 3] (k_feats2joints writes straight into this rank's slot, ONE in-place
// ncclAllGather on the handle's side stream).  The call returns after enqueue; the gather of this batch
// overlaps whatever the caller enqueues next on `stream` - call mldb_gather_wait(h, stream) before reading
// joints_global on `stream`, and alternate (at least) two joints_global buffers between consecutive calls.
extern "C" int mldb_sample_gather(mldb_handle* h, const void* cond, const float* init_noise,
                                  const int32_t* lengths, int32_t B, int32_t S_ctx, int32_t T,
                                  float* joints_global, void* stream, const float* step_noise) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!joints_global) FAIL(MLDB_ERR_INVALID, "bad argument");
  const int64_t count = (int64_t)B * T * h->cfg.njoints * 3;
  cudaStream_t st = (cudaStream_t)stream;
  if (!h->nccl_comm) {      // single rank: the gather is the identity
    return mldb_sample(h, cond, init_noise, lengths, B, S_ctx, T, nullptr, nullptr, joints_global, stream, step_noise);
  }
  TRY(mldb_gather_begin(h, st));
  TRY(mldb_sample(h, cond, init_noise, lengths, B, S_ctx, T, nullptr, nullptr, joints_global + h->comm_rank * count, stream,
                  step_noise));
  return mldb_gather_async(h, joints_global, count, st);
}

// Host-buffer entry point.  With a communicator attached joints_host receives the GATHERED motions
// [nranks * B, T, njoints, 3] (every rank holds all of them after the all-gather), else [B, T, njoints, 3].
extern "C" int mldb_sample_host(mldb_handle* h, const void* cond_host, const float* init_noise_host,
                                const int32_t* lengths_host, int32_t B, int32_t S_ctx, int32_t T,
                                float* joints_host, void* stream, const float* step_noise_host) {
  TRY(check_ready(h, true));
  DeviceGuard guard(h->device);
  if (!cond_host || !init_noise_host || !lengths_host || !joints_host || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  const mldb_config& c = h->cfg;
  Plan* dp = nullptr;
  TRY(dec_plan(h, B, T, &dp));
  const bool cfg_on = c.guidance_scale > 1.0f;
  const int Bx = cfg_on ? 2 * B : B;
  const size_t cond_bytes = c.cond_kind == MLDB_COND_TEXT ? (size_t)Bx * S_ctx * c.text_dim * sizeof(float)
                                                         : (size_t)Bx * sizeof(int64_t);
  const size_t noise_bytes = (size_t)B * c.n_lat * c.latent_dim * sizeof(float);
  if (dp->cond_cap < cond_bytes) {
    TRY(dev_alloc(h, (void**)&dp->cond_f, cond_bytes));
    dp->cond_cap = cond_bytes;
  }
  if (!dp->noise_in) {
    TRY(dev_alloc(h, (void**)&dp->noise_in, noise_bytes));
    TRY(dev_alloc(h, (void**)&dp->cond_i, (size_t)B * sizeof(int32_t)));
  }
  const int world = h->nccl_comm ? h->comm_world : 1;
  const size_t joints_elems = (size_t)B * T * c.njoints * 3;
  if (world > 1 && !dp->joints_all) TRY(dev_alloc(h, (void**)&dp->joints_all, world * joints_elems * sizeof(float)));
  CK(cudaMemcpyAsync(dp->cond_f, cond_host, cond_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(dp->noise_in, init_noise_host, noise_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(dp->cond_i, lengths_host, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  // per-step noise [n_steps, B, n_lat, d]: staged in the decode plan's step_noise buffer (unused by decoding)
  const float* step_noise = nullptr;
  if (step_noise_host) {
    const size_t n = h->timesteps.size() * (size_t)B * c.n_lat * c.latent_dim;
    if (dp->noise_cap < n) {
      TRY(dev_alloc(h, (void**)&dp->step_noise, n * sizeof(float)));
      dp->noise_cap = n;
    }
    CK(cudaMemcpyAsync(dp->step_noise, step_noise_host, n * sizeof(float), cudaMemcpyHostToDevice, st));
    step_noise = dp->step_noise;
  }
  if (world > 1) {
    TRY(mldb_sample_gather(h, dp->cond_f, dp->noise_in, (const int32_t*)dp->cond_i, B, S_ctx, T, dp->joints_all, stream,
                           step_noise));
    TRY(mldb_gather_wait(h, stream));
    CK(cudaMemcpyAsync(joints_host, dp->joints_all, world * joints_elems * sizeof(float), cudaMemcpyDeviceToHost, st));
    return MLDB_OK;
  }
  TRY(mldb_sample(h, dp->cond_f, dp->noise_in, (const int32_t*)dp->cond_i, B, S_ctx, T, nullptr, nullptr, dp->joints, stream,
                  step_noise));
  CK(cudaMemcpyAsync(joints_host, dp->joints, joints_elems * sizeof(float), cudaMemcpyDeviceToHost, st));
  return MLDB_OK;
}
