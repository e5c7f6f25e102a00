// The CLIP text tower (MldTextEncoder): token ids to the denoiser's text context, or to the pooled projection.
#include "engine.h"

#include <string.h>

#include <algorithm>

// ----------------------------------------------------------------------------- CLIP text tower: spec / pack
static const std::string kTextPrefix = "text_encoder.text_model.";   // MldTextEncoder.text_model (a CLIPModel)

extern "C" void mldb_default_text_config(mldb_text_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = MLDB_TEXT_ABI_VERSION;
  c->vocab_size = 49408; c->max_positions = 77; c->hidden = 768; c->heads = 12; c->layers = 12; c->ff = 3072;
  c->projection_dim = 768; c->eos_token_id = 49407; c->ln_eps = 1e-5f;
}

extern "C" int mldb_text_configure(mldb_handle* h, const mldb_text_config* cfg) {
  if (!h || !cfg) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(may_configure(h, cfg->abi_version, MLDB_TEXT_ABI_VERSION, h->text.on || h->bert.on, "text", "the text tower"));
  const mldb_text_config& c = *cfg;
  if (c.vocab_size < 1 || c.layers < 1 || c.heads < 1 || c.ff < 1 || c.projection_dim < 1 || !(c.ln_eps > 0.0f))
    FAIL(MLDB_ERR_INVALID, "bad text config");
  if (!text_ln_supported(c.hidden) || c.hidden % c.heads)
    FAIL(MLDB_ERR_UNSUPPORTED, "text hidden size %d: must be a multiple of 128 (<= 1024) and of heads", c.hidden);
  if (!simt_attention_supported(c.hidden / c.heads))
    FAIL(MLDB_ERR_UNSUPPORTED, "text head_dim %d is too wide for the attention kernels", c.hidden / c.heads);
  if (c.max_positions < 1 || c.max_positions > 256) FAIL(MLDB_ERR_UNSUPPORTED, "max_positions must lie in [1, 256]");
  const std::string T = kTextPrefix, M = T + "text_model.";
  const int d = c.hidden;
  spec_add(h, M + "embeddings.token_embedding.weight", {c.vocab_size, d});
  spec_add(h, M + "embeddings.position_embedding.weight", {c.max_positions, d});
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = M + "encoder.layers." + std::to_string(i) + ".";
    for (const char* pr : {"q_proj.", "k_proj.", "v_proj.", "out_proj."}) {
      spec_add(h, p + "self_attn." + pr + "weight", {d, d});
      spec_add(h, p + "self_attn." + pr + "bias", {d});
    }
    spec_ln(h, p + "layer_norm1.", d);
    spec_add(h, p + "mlp.fc1.weight", {c.ff, d});
    spec_add(h, p + "mlp.fc1.bias", {c.ff});
    spec_add(h, p + "mlp.fc2.weight", {d, c.ff});
    spec_add(h, p + "mlp.fc2.bias", {d});
    spec_ln(h, p + "layer_norm2.", d);
  }
  spec_ln(h, M + "final_layer_norm.", d);
  spec_add(h, T + "text_projection.weight", {c.projection_dim, d});
  h->text.cfg = c;
  h->text.on = true;
  return MLDB_OK;
}

int pack_text(mldb_handle* h) {
  TextW& tw = h->text;
  const mldb_text_config& c = tw.cfg;
  const std::string T = kTextPrefix, M = T + "text_model.";
  const int d = c.hidden;
  TRY(upload_pe(h, M + "embeddings.token_embedding.weight", &tw.tok));
  TRY(upload_pe(h, M + "embeddings.position_embedding.weight", &tw.pos));
  tw.layers.resize(c.layers);
  for (int i = 0; i < c.layers; ++i) {
    const std::string p = M + "encoder.layers." + std::to_string(i) + ".";
    TextLayerW& w = tw.layers[i];
    // one [3d, d] operand: rows q | k | v (the attention kernels' packed-QKV layout)
    std::vector<float> W((size_t)3 * d * d), b((size_t)3 * d);
    const char* names[3] = {"q_proj.", "k_proj.", "v_proj."};
    for (int j = 0; j < 3; ++j) {
      const RawTensor& wt = rt(h, p + "self_attn." + names[j] + "weight");
      const RawTensor& bt = rt(h, p + "self_attn." + names[j] + "bias");
      std::copy(wt.host.begin(), wt.host.end(), W.begin() + (size_t)j * d * d);
      std::copy(bt.host.begin(), bt.host.end(), b.begin() + (size_t)j * d);
    }
    TRY(pack_linear(h, W.data(), 3 * d, d, b.data(), &w.qkv));
    TRY(pack_named(h, p + "self_attn.out_proj.weight", p + "self_attn.out_proj.bias", &w.out));
    TRY(pack_named(h, p + "mlp.fc1.weight", p + "mlp.fc1.bias", &w.fc1));
    TRY(pack_named(h, p + "mlp.fc2.weight", p + "mlp.fc2.bias", &w.fc2));
    TRY(pack_ln(h, p + "layer_norm1.", d, &w.ln1));
    TRY(pack_ln(h, p + "layer_norm2.", d, &w.ln2));
  }
  TRY(pack_ln(h, M + "final_layer_norm.", d, &tw.final_ln));
  TRY(pack_named(h, T + "text_projection.weight", "", &tw.proj));
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- CLIP text tower: forward
void op_text_ln(mldb_handle* h, const TextLnArgs& a, cudaStream_t st) { text_ln(a, st); kcount(h, MLDB_KSTAT_TEXT_LN); }

extern "C" int mldb_text_encode(mldb_handle* h, const int64_t* ids, int32_t n, int32_t L, int32_t mode, float* out,
                                void* stream) {
  if (!h || !ids || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  TextW& tw = h->text;
  TRY(check_configured(h, tw.on, "text", "the text tower"));
  const mldb_text_config& c = tw.cfg;
  if (n < 1 || L < 1 || L > c.max_positions) FAIL(MLDB_ERR_INVALID, "ids must be [n >= 1, 1 <= L <= %d]", c.max_positions);
  if ((int64_t)n * L > (1 << 30)) FAIL(MLDB_ERR_INVALID, "too many tokens");
  if (mode != MLDB_TEXT_HIDDEN && mode != MLDB_TEXT_POOLED) FAIL(MLDB_ERR_INVALID, "mode must be MLDB_TEXT_HIDDEN or MLDB_TEXT_POOLED");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const int M = n * L, d = c.hidden;
  ActBuf a, qkv, att, hid, pooled;
  TRY(grow(tw.x, (size_t)M * d * sizeof(float)));
  TRY(grow_act(tw.a, M, d, &a));
  TRY(grow_act(tw.qkv, M, 3 * d, &qkv));
  TRY(grow_act(tw.att, M, d, &att));
  TRY(grow_act(tw.h, M, c.ff, &hid));
  TRY(grow_act(tw.pooled, n, d, &pooled));
  float* x = (float*)tw.x.p;
  auto ln = [&](int m, const LnW& w) {
    TextLnArgs l; l.mode = m; l.x = x; l.ids = ids; l.L = L; l.tok = tw.tok; l.pos = tw.pos; l.vocab = c.vocab_size;
    l.eos_id = c.eos_token_id; l.gamma = w.g; l.beta = w.b; l.eps = c.ln_eps; l.M = M; l.d = d; l.out = a;
    return l;
  };
  op_text_ln(h, ln(TEXT_LN_EMBED, tw.layers[0].ln1), st);          // x = tok[id] + pos[t]; a = LN1_0(x)
  for (int i = 0; i < c.layers; ++i) {
    const TextLayerW& w = tw.layers[i];
    GemmArgs g; g.a1 = a; g.K1 = d; g.M = M; g.w = w.qkv; g.out = qkv; g.wide_n = 1;
    op_gemm(h, g, st);
    AttnArgs at; at.q = qkv; at.q_col0 = 0; at.Lq = L; at.kv = qkv; at.k_col0 = d; at.v_col0 = 2 * d; at.Lk = L;
    at.nseq = n; at.heads = c.heads; at.hd = d / c.heads; at.causal = 1; at.out = att;
    op_attn(h, at, st);
    GemmArgs go; go.a1 = att; go.K1 = d; go.M = M; go.w = w.out; go.out_f32 = x; go.ldc = d; go.res_f32 = x;
    op_gemm(h, go, st);                                              // x += out_proj(att), in place
    op_text_ln(h, ln(TEXT_LN_ROWS, w.ln2), st);
    GemmArgs g1; g1.a1 = a; g1.K1 = d; g1.M = M; g1.w = w.fc1; g1.act = ACT_QUICKGELU; g1.out = hid; g1.wide_n = 1;
    op_gemm(h, g1, st);
    GemmArgs g2; g2.a1 = hid; g2.K1 = c.ff; g2.M = M; g2.w = w.fc2; g2.out_f32 = x; g2.ldc = d; g2.res_f32 = x;
    op_gemm(h, g2, st);                                              // x += fc2(quick_gelu(fc1(LN2(x))))
    if (i + 1 < c.layers) op_text_ln(h, ln(TEXT_LN_ROWS, tw.layers[i + 1].ln1), st);
  }
  if (mode == MLDB_TEXT_HIDDEN) {
    TextLnArgs l = ln(TEXT_LN_ROWS, tw.final_ln);
    l.out = ActBuf{}; l.out_f32 = out;                             // last_hidden_state, every row
    op_text_ln(h, l, st);
  } else {
    TextLnArgs l = ln(TEXT_LN_EOS, tw.final_ln);
    l.M = n; l.out = pooled;                                       // only the n eos rows
    op_text_ln(h, l, st);
    GemmArgs gp; gp.a1 = l.out; gp.K1 = d; gp.M = n; gp.w = tw.proj; gp.out_f32 = out; gp.ldc = c.projection_dim;
    gp.wide_n = 1;
    op_gemm(h, gp, st);                                              // text_projection (no bias)
  }
  return ops_done(h);
}
