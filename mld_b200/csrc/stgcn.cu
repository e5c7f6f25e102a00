// The UESTC action classifier (STGCN, uestc_stgcn.py) behind UESTCMetrics: data_bn, ten st_gcn blocks over the SMPL
// graph (spatial partition, K = 3), a global average pool and a 1 x 1 convolution head.  Per block:
//   graph mix   Z[(n,t,w), k Cin + ci] = sum_v A'_k[v, w] X[(n,t,v), ci]         (k_stgcn_mix, CUDA cores)
//   gcn GEMM    Y = relu(Z Wg^T + bias[w])  (the 1 x 1 conv and BN1 folded, bias per joint)   (op_gemm)
//   tcn         X' = relu(conv9_s(Y) (+ conv1_s(X)) + b (+ X))  (BN2 / the residual BN folded)  (tconv_tc)
// Mixing before the 1 x 1 convolution is exact by linearity, and moves 3 Cin columns instead of 3 Cout.
#include "engine.h"

#include <math.h>
#include <string.h>

#include <algorithm>

static const char* const kStgcn = "stgcn_classifier.";   // UESTCMetrics.stgcn_classifier (metrics/stgcn.py:32)
static constexpr int kJ = 24, kK = 3, kTaps = 9, kFeat = 256;
static constexpr int kCout[kStgcnBlocks] = {64, 64, 64, 64, 128, 128, 128, 256, 256, 256};
static constexpr int kStride[kStgcnBlocks] = {1, 1, 1, 1, 2, 1, 1, 2, 1, 1};

static int cin_of(const mldb_stgcn_config& c, int i) { return i ? kCout[i - 1] : c.in_channels; }
static int kg_of(const mldb_stgcn_config& c, int i) { return (kK * cin_of(c, i) + 63) / 64 * 64; }
// residual: 0 none (block 0), 1 identity, 2 a 1 x 1 stride-s convolution + BN
static int res_kind(const mldb_stgcn_config& c, int i) {
  if (i == 0) return 0;
  return (cin_of(c, i) == kCout[i] && kStride[i] == 1) ? 1 : 2;
}

extern "C" void mldb_default_stgcn_config(mldb_stgcn_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = MLDB_STGCN_ABI_VERSION;
  c->in_channels = 6; c->num_class = 40;
}

static void spec_bn(mldb_handle* h, const std::string& p, int n) {
  for (const char* s : {"weight", "bias", "running_mean", "running_var"}) spec_add(h, p + s, {n});
  spec_add(h, p + "num_batches_tracked", {});
}

extern "C" int mldb_stgcn_configure(mldb_handle* h, const mldb_stgcn_config* cfg) {
  if (!h || !cfg) FAIL(MLDB_ERR_INVALID, "null argument");
  if (cfg->abi_version != MLDB_STGCN_ABI_VERSION) FAIL(MLDB_ERR_INVALID, "mldb_stgcn_config abi_version mismatch");
  if (h->finalized) FAIL(MLDB_ERR_STATE, "mldb_stgcn_configure must precede mldb_finalize_weights");
  if (h->stgcn.on) FAIL(MLDB_ERR_STATE, "the UESTC classifier is already configured");
  const mldb_stgcn_config& c = *cfg;
  if (c.in_channels < 1 || c.in_channels > 64) FAIL(MLDB_ERR_INVALID, "in_channels must be in [1, 64], got %d", c.in_channels);
  if (c.num_class < 1 || c.num_class > 4096) FAIL(MLDB_ERR_INVALID, "num_class must be in [1, 4096], got %d", c.num_class);
  const std::string p = kStgcn;
  spec_add(h, p + "A", {kK, kJ, kJ});
  spec_bn(h, p + "data_bn.", c.in_channels * kJ);
  for (int i = 0; i < kStgcnBlocks; ++i) {
    const std::string b = p + "st_gcn_networks." + std::to_string(i) + ".";
    const int ci = cin_of(c, i), co = kCout[i];
    spec_add(h, b + "gcn.conv.weight", {kK * co, ci, 1, 1});
    spec_add(h, b + "gcn.conv.bias", {kK * co});
    spec_bn(h, b + "tcn.0.", co);
    spec_add(h, b + "tcn.2.weight", {co, co, kTaps, 1});
    spec_add(h, b + "tcn.2.bias", {co});
    spec_bn(h, b + "tcn.3.", co);
    if (res_kind(c, i) == 2) {
      spec_add(h, b + "residual.0.weight", {co, ci, 1, 1});
      spec_add(h, b + "residual.0.bias", {co});
      spec_bn(h, b + "residual.1.", co);
    }
    spec_add(h, p + "edge_importance." + std::to_string(i), {kK, kJ, kJ});
  }
  spec_add(h, p + "fcn.weight", {c.num_class, kFeat, 1, 1});
  spec_add(h, p + "fcn.bias", {c.num_class});
  h->stgcn.cfg = c;
  h->stgcn.on = true;
  return MLDB_OK;
}

// eval-mode BatchNorm as y = x * scale + shift, in double (eps 1e-5, torch's default)
static void bn_fold(mldb_handle* h, const std::string& p, int n, std::vector<double>* scale, std::vector<double>* shift) {
  const float *w = rt(h, p + "weight").host.data(), *b = rt(h, p + "bias").host.data();
  const float *m = rt(h, p + "running_mean").host.data(), *v = rt(h, p + "running_var").host.data();
  scale->resize(n); shift->resize(n);
  for (int i = 0; i < n; ++i) {
    (*scale)[i] = (double)w[i] / sqrt((double)v[i] + 1e-5);
    (*shift)[i] = (double)b[i] - (double)m[i] * (*scale)[i];
  }
}

int pack_stgcn(mldb_handle* h) {
  StgcnW& s = h->stgcn;
  const mldb_stgcn_config& c = s.cfg;
  const std::string p = kStgcn;
  std::vector<double> sc, sh;
  bn_fold(h, p + "data_bn.", c.in_channels * kJ, &sc, &sh);
  std::vector<float> f(sc.begin(), sc.end()), g(sh.begin(), sh.end());
  TRY(upload_f32(h, f.data(), f.size(), &s.bn_scale));
  TRY(upload_f32(h, g.data(), g.size(), &s.bn_shift));
  const float* A = rt(h, p + "A").host.data();
  std::vector<float> adj((size_t)kStgcnBlocks * kK * kJ * kJ);
  for (int i = 0; i < kStgcnBlocks; ++i) {
    const std::string b = p + "st_gcn_networks." + std::to_string(i) + ".";
    const int ci = cin_of(c, i), co = kCout[i], kg = kg_of(c, i), rk = res_kind(c, i);
    StgcnBlockW& w = s.blocks[i];
    // A'_i = A * edge_importance[i], in fp32 as the reference computes it every forward
    const float* ei = rt(h, p + "edge_importance." + std::to_string(i)).host.data();
    float* Ai = adj.data() + (size_t)i * kK * kJ * kJ;
    for (int e = 0; e < kK * kJ * kJ; ++e) Ai[e] = A[e] * ei[e];
    // gcn: Wg[c, k ci + j] = s1[c] W[k co + c, j]; bias[w, c] = s1[c] sum_k b[k co + c] sum_v A'_k[v, w] + t1[c]
    std::vector<double> s1, t1;
    bn_fold(h, b + "tcn.0.", co, &s1, &t1);
    const float *gw = rt(h, b + "gcn.conv.weight").host.data(), *gb = rt(h, b + "gcn.conv.bias").host.data();
    std::vector<float> Wg((size_t)co * kK * ci), tab((size_t)kJ * co);
    for (int oc = 0; oc < co; ++oc)
      for (int k = 0; k < kK; ++k)
        for (int j = 0; j < ci; ++j)
          Wg[(size_t)oc * kK * ci + k * ci + j] = (float)(s1[oc] * gw[(size_t)(k * co + oc) * ci + j]);
    for (int v2 = 0; v2 < kJ; ++v2)
      for (int oc = 0; oc < co; ++oc) {
        double acc = 0.0;
        for (int k = 0; k < kK; ++k) {
          double colsum = 0.0;
          for (int v = 0; v < kJ; ++v) colsum += Ai[(k * kJ + v) * kJ + v2];
          acc += (double)gb[k * co + oc] * colsum;
        }
        tab[(size_t)v2 * co + oc] = (float)(s1[oc] * acc + t1[oc]);
      }
    TRY(pack_linear(h, Wg.data(), co, kK * ci, nullptr, &w.gcn, kg));
    TRY(upload_f32(h, tab.data(), tab.size(), &w.gcn_tab));
    // tcn: Wt[c, tap co + j] = s2[c] W2[c, j, tap] (+ the residual conv s3[c] Wr[c, j] as a tenth K segment)
    std::vector<double> s2, t2, s3, t3;
    bn_fold(h, b + "tcn.3.", co, &s2, &t2);
    const float *tw = rt(h, b + "tcn.2.weight").host.data(), *tb = rt(h, b + "tcn.2.bias").host.data();
    const int K = kTaps * co + (rk == 2 ? ci : 0);
    std::vector<float> Wt((size_t)co * K), bias(co);
    for (int oc = 0; oc < co; ++oc) {
      for (int tap = 0; tap < kTaps; ++tap)
        for (int j = 0; j < co; ++j)
          Wt[(size_t)oc * K + tap * co + j] = (float)(s2[oc] * tw[((size_t)oc * co + j) * kTaps + tap]);
      bias[oc] = (float)(s2[oc] * tb[oc] + t2[oc]);
    }
    if (rk == 2) {
      bn_fold(h, b + "residual.1.", co, &s3, &t3);
      const float *rw = rt(h, b + "residual.0.weight").host.data(), *rb = rt(h, b + "residual.0.bias").host.data();
      for (int oc = 0; oc < co; ++oc) {
        for (int j = 0; j < ci; ++j) Wt[(size_t)oc * K + kTaps * co + j] = (float)(s3[oc] * rw[(size_t)oc * ci + j]);
        bias[oc] = (float)(s2[oc] * tb[oc] + t2[oc] + s3[oc] * rb[oc] + t3[oc]);
      }
    }
    TRY(pack_linear(h, Wt.data(), co, K, bias.data(), &w.tcn));
  }
  TRY(upload_f32(h, adj.data(), adj.size(), &s.adj));
  TRY(upload_f32(h, rt(h, p + "fcn.weight").host.data(), (size_t)c.num_class * kFeat, &s.fcn_w));
  TRY(upload_f32(h, rt(h, p + "fcn.bias").host.data(), c.num_class, &s.fcn_b));
  return MLDB_OK;
}

// The graph mix of one block, grid-stride over frames: Z[(f, w), k Cin + ci] = sum_v A'_k[v, w] X[(f, v), ci] for
// k Cin + ci < 3 Cin, zero up to Kg.  X is split16 [frames * 24, Cin], or (block 0, x_raw set) the raw input
// [nseq, 24, Cin, T] through data_bn: X[(n, t, v), ci] = x[n, v, ci, t] * bn_scale[v Cin + ci] + bn_shift[..].
__global__ void __launch_bounds__(256) k_stgcn_mix(ActBuf Z, ActBuf X, const float* __restrict__ x_raw,
                                                   const float* __restrict__ bn_scale, const float* __restrict__ bn_shift,
                                                   const float* __restrict__ adj, int frames, int T, int Cin) {
  extern __shared__ float sm[];
  float* sA = sm;                      // [3][24][24]
  float* sX = sm + kK * kJ * kJ;       // [24][Cin]
  for (int i = threadIdx.x; i < kK * kJ * kJ; i += blockDim.x) sA[i] = adj[i];
  const int kc = kK * Cin, Kg = Z.cols;
  for (int f = blockIdx.x; f < frames; f += gridDim.x) {
    __syncthreads();                   // sA is ready / the previous frame's sX is consumed
    for (int i = threadIdx.x; i < kJ * Cin; i += blockDim.x) {
      const int v = i / Cin, ci = i - v * Cin;
      float val;
      if (x_raw) {
        const int n = f / T, t = f - n * T;
        val = fmaf(x_raw[(((int64_t)n * kJ + v) * Cin + ci) * T + t], bn_scale[i], bn_shift[i]);
      } else {
        const int64_t o = ((int64_t)f * kJ + v) * X.cols + ci;
        val = join_f32(X.hi[o], X.lo()[o]);
      }
      sX[i] = val;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kJ * Kg; i += blockDim.x) {
      const int w = i / Kg, col = i - w * Kg;
      float acc = 0.0f;
      if (col < kc) {
        const int k = col / Cin, ci = col - k * Cin;
        const float* a = sA + k * kJ * kJ + w;
#pragma unroll 8
        for (int v = 0; v < kJ; ++v) acc = fmaf(a[v * kJ], sX[v * Cin + ci], acc);
      }
      __half hi, lo;
      split_f32(acc, hi, lo);
      const int64_t o = ((int64_t)f * kJ + w) * Kg + col;
      Z.hi[o] = hi;
      Z.lo()[o] = lo;
    }
  }
}

// gemm=simt: the temporal convolution's im2col, X[(n, t, v), tap C + ci] = Y[(n, s t + tap - 4, v), ci] (zero outside
// [0, T_in)), then the residual convolution's segment X[(n, t, v), 9 C + cr] = R[(n, s t, v), cr] when R is set.
__global__ void k_stgcn_im2col(ActBuf X, ActBuf Y, ActBuf R, int T_in, int T_out, int stride, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int K = X.cols, C = Y.cols;
  const int64_t row = i / K;
  const int col = (int)(i - row * K);
  const int v = (int)(row % kJ);
  const int64_t ft = row / kJ;
  const int t = (int)(ft % T_out);
  const int64_t n = ft / T_out;
  float val = 0.0f;
  if (col < kTaps * C) {
    const int tap = col / C, ci = col - tap * C, s = stride * t + tap - 4;
    if (s >= 0 && s < T_in) {
      const int64_t o = ((n * T_in + s) * kJ + v) * C + ci;
      val = join_f32(Y.hi[o], Y.lo()[o]);
    }
  } else {
    const int64_t o = ((n * T_in + (int64_t)stride * t) * kJ + v) * R.cols + (col - kTaps * C);
    val = join_f32(R.hi[o], R.lo()[o]);
  }
  __half hi, lo;
  split_f32(val, hi, lo);
  X.hi[i] = hi;
  X.lo()[i] = lo;
}

// gemm=simt: the block's end after the temporal-convolution GEMM, out = relu(acc (+ res)) as split16 or fp32
__global__ void k_stgcn_res_relu(const float* __restrict__ acc, ActBuf res, ActBuf out, float* out_f32, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float v = acc[i];
  if (res.hi) v = (v + __half2float(res.hi[i])) + __half2float(res.lo()[i]);
  v = v < 0.0f ? 0.0f : v;                                       // torch.relu: a NaN stays NaN
  if (out.hi) {
    __half hi, lo;
    split_f32(v, hi, lo);
    out.hi[i] = hi;
    out.lo()[i] = lo;
  } else {
    out_f32[i] = v;
  }
}

// The head, one block per sequence (256 threads, one per feature): features = the mean of the sequence's rows in row
// order (avg_pool2d over (T_out, 24)), yhat = fcn(features).  No atomics: every sequence's result is the same
// whichever batch or chunk it is computed in.
__global__ void __launch_bounds__(kFeat) k_stgcn_head(const float* __restrict__ y, int rows, const float* __restrict__ fw,
                                                     const float* __restrict__ fb, int ncls, float* features, float* yhat) {
  __shared__ float sf[kFeat];
  const int b = blockIdx.x, c = threadIdx.x;
  const float* p = y + (int64_t)b * rows * kFeat + c;
  float s = 0.0f;
  for (int r = 0; r < rows; ++r) s += p[(int64_t)r * kFeat];
  const float m = s / (float)rows;
  sf[c] = m;
  if (features) features[(int64_t)b * kFeat + c] = m;
  __syncthreads();
  if (!yhat) return;
  for (int j = c; j < ncls; j += blockDim.x) {
    float acc = 0.0f;
    for (int k = 0; k < kFeat; ++k) acc = fmaf(fw[(int64_t)j * kFeat + k], sf[k], acc);
    yhat[(int64_t)b * ncls + j] = acc + fb[j];
  }
}

// The workspace of n sequences of T frames (bytes per buffer: the largest any block needs).
struct StgcnSizes {
  size_t z = 0, y = 0, x = 0, col = 0, acc = 0, last = 0;
  size_t sum() const { return z + y + 2 * x + col + acc + last; }
};
static StgcnSizes stgcn_sizes(const mldb_stgcn_config& c, int n, int T, bool tc) {
  StgcnSizes s;
  int Ti = T;
  for (int i = 0; i < kStgcnBlocks; ++i) {
    const int To = (Ti - 1) / kStride[i] + 1, co = kCout[i], ci = cin_of(c, i);
    const int rin = n * Ti * kJ, rout = n * To * kJ;
    s.z = std::max(s.z, split16_bytes(rin, kg_of(c, i)));
    s.y = std::max(s.y, split16_bytes(rin, co));
    if (i < kStgcnBlocks - 1) s.x = std::max(s.x, split16_bytes(rout, co));
    else s.last = (size_t)rout * co * sizeof(float);
    if (!tc) {
      s.col = std::max(s.col, split16_bytes(rout, kTaps * co + (res_kind(c, i) == 2 ? ci : 0)));
      s.acc = std::max(s.acc, (size_t)rout * co * sizeof(float));
    }
    Ti = To;
  }
  return s;
}

// sequences per chunk: the option, else what keeps the chunk's workspace near 1 GiB
static int stgcn_chunk(const mldb_handle* h, int B, size_t per_seq) {
  if (h->stgcn.chunk > 0) return std::min(B, h->stgcn.chunk);
  return std::min(B, (int)std::max<size_t>(1, ((size_t)1 << 30) / per_seq));
}

extern "C" int mldb_stgcn_classify(mldb_handle* h, const float* x, int32_t B, int32_t T, float* yhat, float* features,
                                   void* stream) {
  if (!h || !x) FAIL(MLDB_ERR_INVALID, "null argument");
  if (!h->stgcn.on) FAIL(MLDB_ERR_STATE, "the UESTC classifier is not configured (mldb_stgcn_configure)");
  if (!h->finalized) FAIL(MLDB_ERR_STATE, "finalize weights first");
  StgcnW& s = h->stgcn;
  const mldb_stgcn_config& c = s.cfg;
  if (B < 1 || T < 1 || (int64_t)B * T > (1 << 22))
    FAIL(MLDB_ERR_INVALID, "classifier input must be [B >= 1, 24, %d, T >= 1] with B * T <= 2^22, got B=%d T=%d",
         c.in_channels, B, T);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const bool tc = h->use_tc;
  const int Bc = stgcn_chunk(h, B, stgcn_sizes(c, 1, T, tc).sum());
  const int mix_smem = (kK * kJ * kJ + kJ * std::max(c.in_channels, kFeat)) * (int)sizeof(float);
  for (int b0 = 0; b0 < B; b0 += Bc) {
    const int n = std::min(Bc, B - b0);
    const StgcnSizes sz = stgcn_sizes(c, n, T, tc);
    TRY(grow(s.z, sz.z));
    TRY(grow(s.y, sz.y));
    TRY(grow(s.x[0], sz.x));
    TRY(grow(s.x[1], sz.x));
    TRY(grow(s.last, sz.last));
    if (!tc) {
      TRY(grow(s.col, sz.col));
      TRY(grow(s.acc, sz.acc));
    }
    ActBuf xin{};                                    // the block input (split16), none for block 0
    int Ti = T;
    for (int i = 0; i < kStgcnBlocks; ++i) {
      const StgcnBlockW& w = s.blocks[i];
      const int ci = cin_of(c, i), co = kCout[i], kg = kg_of(c, i), To = (Ti - 1) / kStride[i] + 1, rk = res_kind(c, i);
      const bool last = i == kStgcnBlocks - 1;
      const int rows_in = n * Ti * kJ, rows_out = n * To * kJ;
      const ActBuf Z = split16_at(s.z.p, rows_in, kg), Y = split16_at(s.y.p, rows_in, co);
      const ActBuf X = last ? ActBuf{} : split16_at(s.x[i & 1].p, rows_out, co);
      const int frames = n * Ti;
      k_stgcn_mix<<<(unsigned)std::min(frames, 8 * h->sm_count), 256, mix_smem, st>>>(
          Z, xin, i ? nullptr : x + (int64_t)b0 * kJ * ci * T, s.bn_scale, s.bn_shift, s.adj + (size_t)i * kK * kJ * kJ,
          frames, Ti, ci);
      kcount(h, MLDB_KSTAT_MISC);
      GemmArgs g; g.a1 = Z; g.K1 = kg; g.M = rows_in; g.w = w.gcn; g.act = ACT_RELU; g.out = Y;
      g.addtab = w.gcn_tab; g.in_group = kJ; g.out_group = kJ;
      op_gemm(h, g, st);                             // the gcn's 1 x 1 conv, BN1 and ReLU
      float* yout = last ? (float*)s.last.p : nullptr;
      if (tc) {
        TconvArgs a;
        a.x = Y; a.w = w.tcn; a.nseq = n; a.T_in = Ti; a.T_out = To; a.C = co; a.stride = kStride[i];
        if (rk) { a.res = xin; a.C_res = ci; a.res_conv = rk == 2; }
        a.out = X; a.out_f32 = yout;
        if (!tconv_tc_supported(a)) {
          mldb_set_err("st_gcn block " + std::to_string(i) + ": no temporal-convolution kernel for this shape");
          h->op_failed = true;
        } else if (!tconv_tc(a, h->sm_count, st)) {
          h->op_failed = true;
        }
        kcount(h, MLDB_KSTAT_GEMM_TC);
      } else {
        const int K = w.tcn.K;
        const ActBuf col = split16_at(s.col.p, rows_out, K);
        const int64_t total = (int64_t)rows_out * K;
        k_stgcn_im2col<<<nblk(total), 256, 0, st>>>(col, Y, rk == 2 ? xin : ActBuf{}, Ti, To, kStride[i], total);
        kcount(h, MLDB_KSTAT_MISC);
        GemmArgs gt; gt.a1 = col; gt.K1 = K; gt.M = rows_out; gt.w = w.tcn; gt.out_f32 = (float*)s.acc.p; gt.ldc = co;
        op_gemm(h, gt, st);
        const int64_t n_out = (int64_t)rows_out * co;
        k_stgcn_res_relu<<<nblk(n_out), 256, 0, st>>>((float*)s.acc.p, rk == 1 ? xin : ActBuf{}, X, yout, n_out);
        kcount(h, MLDB_KSTAT_MISC);
      }
      xin = X;
      Ti = To;
    }
    k_stgcn_head<<<(unsigned)n, kFeat, 0, st>>>((float*)s.last.p, Ti * kJ, s.fcn_w, s.fcn_b, c.num_class,
                                               features ? features + (int64_t)b0 * kFeat : nullptr,
                                               yhat ? yhat + (int64_t)b0 * c.num_class : nullptr);
    kcount(h, MLDB_KSTAT_MISC);
  }
  return ops_done(h);
}
