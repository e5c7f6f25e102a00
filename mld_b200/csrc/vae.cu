// The VAE (MldVae and ActorVae): latents to motion features, motion features to the latent distribution, and
// feats2joints.
#include "engine.h"
#include "misc_kernels.cuh"

// ----------------------------------------------------------------------------- VAE decode
// z rows: [n_lat, B, d] fp32 -> memory tokens split [B * n_lat, d] (row = b * n_lat + j)
__global__ void k_mem_tokens(ActBuf mem, const float* __restrict__ z, int n_lat, int B, int d) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_lat * B * d) return;
  const int n = (int)(idx % d);
  const int b = (int)((idx / d) % B);
  const int j = (int)(idx / ((int64_t)d * B));
  __half hh, ll;
  split_f32(z[idx], hh, ll);
  const int64_t o = ((int64_t)b * n_lat + j) * mem.cols + n;
  mem.hi[o] = hh;
  mem.lo()[o] = ll;
}

int dec_plan(mldb_handle* h, int B, int T, Plan** out) {
  Plan* p = find_plan(h, PLAN_VAE_DECODE, B, 0, T);
  if (!p) {
    const mldb_config& c = h->cfg;
    if (T > h->vae_dec_pe_rows) FAIL(MLDB_ERR_INVALID, "T=%d exceeds the positional table (%d rows)", T, h->vae_dec_pe_rows);
    p = add_plan(h, PLAN_VAE_DECODE, B, 0, T);
    TRY(alloc_stack_ws(h, h->vdec, B, T, c.n_lat, &p->ws));
    TRY(alloc_act(h, B * c.n_lat, c.latent_dim, &p->mem));
    TRY(dev_alloc(h, (void**)&p->lengths, (size_t)B * sizeof(int32_t)));
    TRY(dev_alloc(h, (void**)&p->feats, (size_t)B * T * c.vae_nfeats * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->joints, (size_t)B * T * c.njoints * 3 * sizeof(float)));
    TRY(dev_alloc(h, (void**)&p->latents, (size_t)B * c.n_lat * c.latent_dim * sizeof(float)));
  }
  *out = p;
  return MLDB_OK;
}

// z_is_plan_latents: z already sits in [n_lat,B,d] order in a device buffer
int run_decode(mldb_handle* h, const float* z, const int32_t* lengths, int B, int T, float* feats_out, cudaStream_t st,
               Plan** plan_out) {
  const mldb_config& c = h->cfg;
  if (c.vae_kind == MLDB_VAE_NONE) FAIL(MLDB_ERR_STATE, "no VAE configured");
  Plan* p = nullptr;
  TRY(dec_plan(h, B, T, &p));
  const int d = c.latent_dim, F = c.vae_nfeats;
  CK(cudaMemcpyAsync(p->lengths, lengths, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(p->latents, z, (size_t)B * c.n_lat * d * sizeof(float), cudaMemcpyDeviceToDevice, st));
  float* fout = feats_out ? feats_out : p->feats;
  TRY(run_graphed(h, p, st, [&](cudaStream_t s) {
    k_mem_tokens<<<nblk((int64_t)c.n_lat * B * d), 256, 0, s>>>(p->mem, p->latents, c.n_lat, B, d);
    kcount(h, MLDB_KSTAT_MISC);
    // queries = zeros + PE rows (mld_vae.py:190,224; actor_vae.py:219-225)
    rows_to_split(h, p->ws.x0, nullptr, 0, B * T, d, T, T, 0, 0, h->vae_dec_pe, 0, s);
    SeqInfo si; si.lengths = p->lengths; si.kv_prefix = 0;
    ActBuf x = run_stack(h, h->vdec, p->ws.x0, p->mem, p->ws, si, s);
    if (h->vdec.norm.g) {
      LnArgs l; l.res = x; l.gamma = h->vdec.norm.g; l.beta = h->vdec.norm.b; l.M = B * T; l.d = d; l.out = p->ws.x1;
      op_ln(h, l, s);
      x = p->ws.x1;
    }
    // final_layer + output[~mask.T] = 0 (mld_vae.py:243-245); rows are already [B, T]
    GemmArgs g; g.a1 = x; g.K1 = d; g.M = B * T; g.w = h->final_layer; g.out_f32 = p->feats; g.ldc = F;
    g.in_group = T; g.out_group = T; g.out_off = 0; g.zero_lengths = p->lengths;
    op_gemm(h, g, s);
  }));
  if (fout != p->feats)
    CK(cudaMemcpyAsync(fout, p->feats, (size_t)B * T * F * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (plan_out) *plan_out = p;
  return MLDB_OK;
}

extern "C" int mldb_vae_decode(mldb_handle* h, const float* z, const int32_t* lengths, int32_t B,
                               int32_t T, float* feats_out, void* stream) {
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!z || !lengths || !feats_out || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  return run_decode(h, z, lengths, B, T, feats_out, (cudaStream_t)stream, nullptr);
}

// ----------------------------------------------------------------------------- VAE encode
__global__ void k_rows_out_permuted(const float* __restrict__ src, float* __restrict__ mu, float* __restrict__ logvar,
                                    int B, int n_lat, int d) {
  // src rows (b, j) j < 2*n_lat -> mu[j, b, :] (j < n_lat) / logvar[j - n_lat, b, :]
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)B * 2 * n_lat * d) return;
  const int n = (int)(idx % d);
  const int j = (int)((idx / d) % (2 * n_lat));
  const int b = (int)(idx / ((int64_t)d * 2 * n_lat));
  if (j < n_lat) mu[((int64_t)j * B + b) * d + n] = src[idx];
  else logvar[((int64_t)(j - n_lat) * B + b) * d + n] = src[idx];
}

extern "C" int mldb_vae_encode(mldb_handle* h, const float* feats, const int32_t* lengths, int32_t B,
                               int32_t T, float* mu, float* logvar, void* stream) {
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!feats || !lengths || !mu || !logvar || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  const mldb_config& c = h->cfg;
  const bool actor = c.vae_kind == MLDB_VAE_ACTOR;
  if (c.vae_kind != MLDB_VAE_MLD && !actor) FAIL(MLDB_ERR_UNSUPPORTED, "encode needs a VAE (MldVae or ActorVae)");
  if (actor && h->venc.enc.empty())
    FAIL(MLDB_ERR_STATE, "the ActorVae encoder was not loaded: the state dict held no 'vae.encoder.*' keys");
  if (actor && c.n_lat != 1) FAIL(MLDB_ERR_UNSUPPORTED, "the ActorVae encoder yields one latent token, not n_lat = %d", c.n_lat);
  cudaStream_t st = (cudaStream_t)stream;
  const int d = c.latent_dim, G = 2 * c.n_lat, L = G + T;
  if (L > h->vae_enc_pe_rows)
    FAIL(MLDB_ERR_INVALID, "T + %d = %d tokens exceed the encoder's positional table (%d rows)", G, L, h->vae_enc_pe_rows);
  Plan* p = find_plan(h, PLAN_VAE_ENCODE, B, 0, T);
  if (!p) {
    p = add_plan(h, PLAN_VAE_ENCODE, B, 0, T);
    // the last layer runs trimmed to the G distribution rows (ActorVae: always; MldVae: when it has skip blocks)
    TRY(alloc_stack_ws(h, h->venc, B, L, 0, &p->ws, actor || h->venc.layers >= 3 ? G : 0));
    TRY(dev_alloc(h, (void**)&p->lengths, (size_t)B * sizeof(int32_t)));
    TRY(dev_alloc(h, (void**)&p->stage_f32, (size_t)B * G * d * sizeof(float)));
    if (h->skel_emb.K % 64 == 0) TRY(alloc_act(h, B * T, h->skel_emb.K, &p->in_split));
  }
  CK(cudaMemcpyAsync(p->lengths, lengths, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  // skel_embedding rows -> token rows (b, G + t) + PE (mld_vae.py:139-161); the 263 features are
  // zero-padded to the packed K so that the embedding runs on the tensor cores
  GemmArgs g; g.M = B * T; g.w = h->skel_emb;
  g.out = p->ws.x0; g.in_group = T; g.out_group = L; g.out_off = G; g.addtab = h->vae_enc_pe;
  if (h->use_tc && p->in_split.hi) {
    k_f32_to_split_pad<<<nblk((int64_t)B * T * p->in_split.cols), 256, 0, st>>>(p->in_split, feats, c.vae_nfeats, B * T, c.vae_nfeats, 1);
    kcount(h, MLDB_KSTAT_MISC);
    g.a1 = p->in_split; g.K1 = p->in_split.cols;
  } else {
    g.a_kind = A_F32; g.a_f32 = feats; g.lda = c.vae_nfeats;
  }
  op_gemm(h, g, st);
  // global motion tokens (b, 0..G-1) = token + PE (mld_vae.py:146,157; actor_vae.py:144-165)
  k_rows_to_split<<<nblk((int64_t)B * G * d), 256, 0, st>>>(p->ws.x0, h->global_token, d, B * G, d, G, L, 0, 1, h->vae_enc_pe);
  kcount(h, MLDB_KSTAT_MISC);
  SeqInfo si; si.lengths = p->lengths; si.kv_prefix = G;
  ActBuf x = run_stack(h, h->venc, p->ws.x0, ActBuf{}, p->ws, si, st);
  if (actor) {   // no final norm: the trimmed layer's (b, mu | logvar) rows are the distribution (actor_vae.py:169)
    k_split_to_f32<<<nblk((int64_t)B * G * d), 256, 0, st>>>(x, p->stage_f32, (int64_t)B * G * d);
    kcount(h, MLDB_KSTAT_MISC);
    k_rows_out_permuted<<<nblk((int64_t)B * G * d), 256, 0, st>>>(p->stage_f32, mu, logvar, B, 1, d);
    kcount(h, MLDB_KSTAT_MISC);
    return ops_done(h);
  }
  LnArgs l; l.res = x; l.gamma = h->venc.norm.g; l.beta = h->venc.norm.b; l.M = B * G; l.d = d;
  if (p->ws.n_sel == 0) { l.sel_group = G; l.in_group = L; }
  l.out_f32 = p->stage_f32; l.ld_out = d;
  op_ln(h, l, st);
  k_rows_out_permuted<<<nblk((int64_t)B * G * d), 256, 0, st>>>(p->stage_f32, mu, logvar, B, c.n_lat, d);
  kcount(h, MLDB_KSTAT_MISC);
  return ops_done(h);
}

// ----------------------------------------------------------------------------- feats2joints
int run_f2j(mldb_handle* h, const float* feats, int B, int T, float* joints, cudaStream_t st) {
  const mldb_config& c = h->cfg;
  const int F = c.vae_kind != MLDB_VAE_NONE ? c.vae_nfeats : c.nfeats;
  if (!h->mean || h->nstat != F) FAIL(MLDB_ERR_STATE, "call mldb_set_mean_std with %d features first", F);
  if (F < 4 + (c.njoints - 1) * 3) FAIL(MLDB_ERR_UNSUPPORTED, "feats2joints needs the HumanML3D/KIT layout");
  k_feats2joints<<<B, 256, 0, st>>>(feats, h->mean, h->stdv, T, F, c.njoints, joints);
  kcount(h, MLDB_KSTAT_MISC);
  CK(cudaGetLastError());
  return MLDB_OK;
}
extern "C" int mldb_feats2joints(mldb_handle* h, const float* feats, int32_t B, int32_t T,
                                 float* joints_out, void* stream) {
  TRY(check_ready(h, false));
  DeviceGuard guard(h->device);
  if (!feats || !joints_out || B <= 0 || T <= 0) FAIL(MLDB_ERR_INVALID, "bad argument");
  return run_f2j(h, feats, B, T, joints_out, (cudaStream_t)stream);
}
