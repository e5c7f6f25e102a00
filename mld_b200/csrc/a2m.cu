// The HumanAct12 action classifier (MotionDiscriminator / MotionDiscriminatorForFID, humanact12_gru.py) behind the
// action model's accuracy and FID: a unidirectional multi-layer GRU, the output at lengths - 1, and a small head.
#include "engine.h"

#include <string.h>

#include <algorithm>

static const char* const kA2m = "gru_classifier.";   // HUMANACTMetrics.gru_classifier (metrics/gru.py:32)
static constexpr int kA2mFeat = 30;                  // linear1's width (humanact12_gru.py:23)

extern "C" void mldb_default_a2m_config(mldb_a2m_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = MLDB_A2M_ABI_VERSION;
  c->input_size = 72; c->hidden_size = 128; c->hidden_layer = 2; c->output_size = 12;
}

extern "C" int mldb_a2m_configure(mldb_handle* h, const mldb_a2m_config* cfg) {
  if (!h || !cfg) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(may_configure(h, cfg->abi_version, MLDB_A2M_ABI_VERSION, h->a2m.on, "a2m", "the action classifier"));
  const mldb_a2m_config& c = *cfg;
  if (c.input_size < 1 || c.input_size > 4096) FAIL(MLDB_ERR_INVALID, "input_size must be in [1, 4096], got %d", c.input_size);
  if (c.output_size < 1 || c.output_size > 4096) FAIL(MLDB_ERR_INVALID, "output_size must be in [1, 4096], got %d", c.output_size);
  if (c.hidden_layer < 1 || c.hidden_layer > 8) FAIL(MLDB_ERR_UNSUPPORTED, "hidden_layer must be in [1, 8], got %d", c.hidden_layer);
  if (!gru_seq_supported(c.hidden_size))
    FAIL(MLDB_ERR_UNSUPPORTED, "hidden_size must be 64 or 128 (a layer's split16 W_hh must fit in shared memory), got %d",
         c.hidden_size);
  const std::string p = std::string(kA2m) + "recurrent.";
  const int H = c.hidden_size;
  for (int k = 0; k < c.hidden_layer; ++k) {
    const std::string l = "_l" + std::to_string(k);
    spec_add(h, p + "weight_ih" + l, {3 * H, k ? H : c.input_size});
    spec_add(h, p + "weight_hh" + l, {3 * H, H});
    spec_add(h, p + "bias_ih" + l, {3 * H});
    spec_add(h, p + "bias_hh" + l, {3 * H});
  }
  spec_add(h, std::string(kA2m) + "linear1.weight", {kA2mFeat, H});
  spec_add(h, std::string(kA2m) + "linear1.bias", {kA2mFeat});
  spec_add(h, std::string(kA2m) + "linear2.weight", {c.output_size, kA2mFeat});
  spec_add(h, std::string(kA2m) + "linear2.bias", {c.output_size});
  h->a2m.cfg = c;
  h->a2m.on = true;
  return MLDB_OK;
}

int pack_a2m(mldb_handle* h) {
  A2mW& a = h->a2m;
  const mldb_a2m_config& c = a.cfg;
  const int H = c.hidden_size;
  const std::string p = std::string(kA2m) + "recurrent.";
  a.layers.resize(c.hidden_layer);
  for (int k = 0; k < c.hidden_layer; ++k) {
    const std::string l = "_l" + std::to_string(k);
    A2mLayerW& w = a.layers[k];
    TRY(pack_named(h, p + "weight_ih" + l, p + "bias_ih" + l, &w.w_ih, 0, -1, true));
    const std::vector<float>& whh = rt(h, p + "weight_hh" + l).host;
    std::vector<float> W((size_t)3 * H * H);
    for (int gate = 0; gate < 3; ++gate)
      for (int u = 0; u < H; ++u)
        std::copy_n(whh.begin() + (size_t)(gate * H + u) * H, H, W.begin() + (size_t)gru_packed_col(gate, u) * H);
    TRY(pack_linear(h, W.data(), 3 * H, H, nullptr, &w.w_hh));
    TRY(upload_f32(h, rt(h, p + "bias_hh" + l).host.data(), (size_t)3 * H, &w.b_hh));
  }
  const std::string q = kA2m;
  TRY(upload_f32(h, rt(h, q + "linear1.weight").host.data(), (size_t)kA2mFeat * H, &a.l1w));
  TRY(upload_f32(h, rt(h, q + "linear1.bias").host.data(), kA2mFeat, &a.l1b));
  TRY(upload_f32(h, rt(h, q + "linear2.weight").host.data(), (size_t)c.output_size * kA2mFeat, &a.l2w));
  TRY(upload_f32(h, rt(h, q + "linear2.bias").host.data(), c.output_size, &a.l2b));
  return MLDB_OK;
}

// X[b * T + t, c] = x[b, c, t] for c < In and t < len[b], else 0 (split16; X.cols = In padded to 64).  A 32-frame x
// 64-channel tile goes through shared memory so that both the reads (along t) and the writes (along c) are coalesced.
// Frames at t >= len are not read.
__global__ void __launch_bounds__(256) k_a2m_frames(ActBuf X, const float* __restrict__ x, const int32_t* __restrict__ lengths,
                                                    int In, int T) {
  __shared__ float tile[64][33];
  const int b = blockIdx.y, t0 = blockIdx.x * 32;
  int len = lengths[b];
  len = len < 0 ? 0 : (len > T ? T : len);
  for (int c0 = 0; c0 < X.cols; c0 += 64) {
    for (int i = threadIdx.x; i < 64 * 32; i += blockDim.x) {
      const int cc = i >> 5, t = t0 + (i & 31), c = c0 + cc;
      tile[cc][i & 31] = (c < In && t < len) ? x[((int64_t)b * In + c) * T + t] : 0.0f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * 64; i += blockDim.x) {
      const int tt = i >> 6, cc = i & 63, t = t0 + tt;
      if (t < T) {
        const int64_t o = ((int64_t)b * T + t) * X.cols + c0 + cc;
        __half hi, lo;
        split_f32(tile[cc][tt], hi, lo);
        X.hi[o] = hi;
        X.lo()[o] = lo;
      }
    }
    __syncthreads();
  }
}

// The head in fp32 on CUDA cores, one block per sequence: f = tanh(W1 h + b1) [30], logits = W2 f + b2.
__global__ void __launch_bounds__(128) k_a2m_head(const float* __restrict__ hl, int64_t ld, int H, const float* __restrict__ w1,
                                                  const float* __restrict__ b1, const float* __restrict__ w2,
                                                  const float* __restrict__ b2, int out_dim, float* features, float* logits) {
  __shared__ float sh[128];
  __shared__ float sf[kA2mFeat];
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < H; i += blockDim.x) sh[i] = hl[(int64_t)b * ld + i];
  __syncthreads();
  if (threadIdx.x < kA2mFeat) {
    const int j = threadIdx.x;
    float acc = 0.0f;
    for (int k = 0; k < H; ++k) acc = fmaf(w1[j * H + k], sh[k], acc);
    const float f = tanhf(acc + b1[j]);
    sf[j] = f;
    if (features) features[(int64_t)b * kA2mFeat + j] = f;
  }
  __syncthreads();
  if (!logits) return;
  for (int j = threadIdx.x; j < out_dim; j += blockDim.x) {
    float acc = 0.0f;
    for (int k = 0; k < kA2mFeat; ++k) acc = fmaf(w2[j * kA2mFeat + k], sf[k], acc);
    logits[(int64_t)b * out_dim + j] = acc + b2[j];
  }
}

extern "C" int mldb_a2m_classify(mldb_handle* h, const float* x, const int32_t* lengths, const float* h0, int32_t B,
                                 int32_t T, float* logits, float* features, void* stream) {
  if (!h || !x || !lengths || !h0) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(check_configured(h, h->a2m.on, "a2m", "the action classifier"));
  const mldb_a2m_config& c = h->a2m.cfg;
  if (B < 1 || T < 1 || (int64_t)B * T > (1 << 26))
    FAIL(MLDB_ERR_INVALID, "classifier input must be [B >= 1, %d, T >= 1] with B * T <= 2^26, got B=%d T=%d", c.input_size, B, T);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  {
    std::vector<int32_t> ln((size_t)B);
    CK(cudaMemcpyAsync(ln.data(), lengths, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b)
      if (ln[b] < 1 || ln[b] > T) FAIL(MLDB_ERR_INVALID, "lengths[%d] = %d is outside [1, T = %d]", b, ln[b], T);
  }
  A2mW& a = h->a2m;
  const int In = c.input_size, Kp = (In + 63) / 64 * 64, H = c.hidden_size, NL = c.hidden_layer;
  const size_t per_seq = (size_t)T * (4 * Kp + 12 * H + (NL > 1 ? 4 * H : 0)) + (size_t)(h->use_tc ? 4 : 40) * H;
  const int Bc = eval_chunk(a.chunk, B, per_seq, 64);
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0), M = n * T;
    ActBuf xs, seq;
    TRY(grow_act(a.x, M, Kp, &xs));
    if (NL > 1) TRY(grow_act(a.seq, M, H, &seq));
    k_a2m_frames<<<dim3((unsigned)((T + 31) / 32), (unsigned)n), 256, 0, st>>>(xs, x + (int64_t)b0 * In * T, lengths + b0, In, T);
    kcount(h, MLDB_KSTAT_MISC);
    const float* hl = nullptr;                       // the last layer's h at t = len - 1, rows H floats apart
    for (int l = 0; l < NL; ++l) {                   // each layer but the last writes its h_t into seq
      const A2mLayerW& w = a.layers[l];
      const bool last = l == NL - 1;
      TRY(op_gru(h, l ? seq : xs, &w.w_ih, w.w_hh, w.b_hh, h0 + ((int64_t)l * B + b0) * H, H, lengths + b0, n, T, H, 1,
                 a.gi, a.gru, last ? ActBuf{} : seq, nullptr, last ? &hl : nullptr, st));
    }
    k_a2m_head<<<(unsigned)n, 128, 0, st>>>(hl, H, H, a.l1w, a.l1b, a.l2w, a.l2b, c.output_size,
                                            features ? features + (int64_t)b0 * kA2mFeat : nullptr,
                                            logits ? logits + (int64_t)b0 * c.output_size : nullptr);
    kcount(h, MLDB_KSTAT_MISC);
  }
  return ops_done(h);
}
