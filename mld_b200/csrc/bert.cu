// The BERT / DistilBERT text tower (MldTextEncoder with a "bert" model path): token ids and right-padded attention
// masks to last_hidden_state, the denoiser's context.
#include "engine.h"

#include <string.h>

#include <algorithm>

// ----------------------------------------------------------------------------- spec / pack
static const std::string kBertPrefix = "text_encoder.text_model.";   // MldTextEncoder.text_model (AutoModel)

// The state-dict names of one layer's tensors, per family: q, k, v, out-projection, attention LN, lin1, lin2, output LN
struct BertNames { std::string q, k, v, out, ln1, fc1, fc2, ln2; };
static BertNames layer_names(const mldb_bert_config& c, int i) {
  const std::string M = kBertPrefix, n = std::to_string(i);
  if (c.family == MLDB_BERT_DISTILBERT) {
    const std::string p = M + "transformer.layer." + n + ".";
    return {p + "attention.q_lin.", p + "attention.k_lin.", p + "attention.v_lin.", p + "attention.out_lin.",
            p + "sa_layer_norm.", p + "ffn.lin1.", p + "ffn.lin2.", p + "output_layer_norm."};
  }
  const std::string p = M + "encoder.layer." + n + ".";
  return {p + "attention.self.query.", p + "attention.self.key.", p + "attention.self.value.",
          p + "attention.output.dense.", p + "attention.output.LayerNorm.", p + "intermediate.dense.",
          p + "output.dense.", p + "output.LayerNorm."};
}

extern "C" void mldb_default_bert_config(mldb_bert_config* c) {
  memset(c, 0, sizeof *c);
  c->abi_version = MLDB_BERT_ABI_VERSION;
  c->family = MLDB_BERT_DISTILBERT;
  c->vocab_size = 30522; c->max_positions = 512; c->type_vocab = 2; c->hidden = 768; c->heads = 12; c->layers = 6;
  c->ff = 3072; c->ln_eps = 1e-12f;
}

extern "C" int mldb_bert_configure(mldb_handle* h, const mldb_bert_config* cfg) {
  if (!h || !cfg) FAIL(MLDB_ERR_INVALID, "null argument");
  TRY(may_configure(h, cfg->abi_version, MLDB_BERT_ABI_VERSION, h->text.on || h->bert.on, "bert", "the text tower"));
  const mldb_bert_config& c = *cfg;
  if (c.family != MLDB_BERT_DISTILBERT && c.family != MLDB_BERT_BERT) FAIL(MLDB_ERR_INVALID, "bad BERT family %d", c.family);
  if (c.vocab_size < 1 || c.layers < 1 || c.heads < 1 || c.ff < 1 || !(c.ln_eps > 0.0f) ||
      (c.family == MLDB_BERT_BERT && c.type_vocab < 1))
    FAIL(MLDB_ERR_INVALID, "bad BERT config");
  if (!text_ln_supported(c.hidden) || c.hidden % c.heads)
    FAIL(MLDB_ERR_UNSUPPORTED, "BERT hidden size %d: must be a multiple of 128 (<= 1024) and of heads", c.hidden);
  if (!simt_attention_supported(c.hidden / c.heads))
    FAIL(MLDB_ERR_UNSUPPORTED, "BERT head_dim %d is too wide for the attention kernels", c.hidden / c.heads);
  if (c.max_positions < 1 || c.max_positions > 512) FAIL(MLDB_ERR_UNSUPPORTED, "max_positions must lie in [1, 512]");
  const std::string E = kBertPrefix + "embeddings.";
  const int d = c.hidden;
  spec_add(h, E + "word_embeddings.weight", {c.vocab_size, d});
  spec_add(h, E + "position_embeddings.weight", {c.max_positions, d});
  if (c.family == MLDB_BERT_BERT) spec_add(h, E + "token_type_embeddings.weight", {c.type_vocab, d});
  spec_ln(h, E + "LayerNorm.", d);
  for (int i = 0; i < c.layers; ++i) {
    const BertNames n = layer_names(c, i);
    for (const std::string* p : {&n.q, &n.k, &n.v, &n.out}) {
      spec_add(h, *p + "weight", {d, d});
      spec_add(h, *p + "bias", {d});
    }
    spec_ln(h, n.ln1, d);
    spec_add(h, n.fc1 + "weight", {c.ff, d});
    spec_add(h, n.fc1 + "bias", {c.ff});
    spec_add(h, n.fc2 + "weight", {d, c.ff});
    spec_add(h, n.fc2 + "bias", {d});
    spec_ln(h, n.ln2, d);
  }
  if (c.family == MLDB_BERT_BERT) {                 // AutoModel's pooler: loaded (strict), never uploaded
    spec_add(h, kBertPrefix + "pooler.dense.weight", {d, d});
    spec_add(h, kBertPrefix + "pooler.dense.bias", {d});
  }
  h->bert.cfg = c;
  h->bert.on = true;
  return MLDB_OK;
}

int pack_bert(mldb_handle* h) {
  BertW& bw = h->bert;
  const mldb_bert_config& c = bw.cfg;
  const std::string E = kBertPrefix + "embeddings.";
  const int d = c.hidden;
  TRY(upload_pe(h, E + "word_embeddings.weight", &bw.word));
  TRY(upload_pe(h, E + "position_embeddings.weight", &bw.pos));
  if (c.family == MLDB_BERT_BERT)                    // token types are all zero: only row 0 is ever read
    TRY(upload_f32(h, rt(h, E + "token_type_embeddings.weight").host.data(), d, &bw.type0));
  TRY(pack_ln(h, E + "LayerNorm.", d, &bw.emb_ln));
  bw.layers.resize(c.layers);
  for (int i = 0; i < c.layers; ++i) {
    const BertNames n = layer_names(c, i);
    TextLayerW& w = bw.layers[i];
    // one [3d, d] operand: rows q | k | v (the attention kernels' packed-QKV layout)
    std::vector<float> W((size_t)3 * d * d), b((size_t)3 * d);
    const std::string* qkv[3] = {&n.q, &n.k, &n.v};
    for (int j = 0; j < 3; ++j) {
      const RawTensor& wt = rt(h, *qkv[j] + "weight");
      const RawTensor& bt = rt(h, *qkv[j] + "bias");
      std::copy(wt.host.begin(), wt.host.end(), W.begin() + (size_t)j * d * d);
      std::copy(bt.host.begin(), bt.host.end(), b.begin() + (size_t)j * d);
    }
    TRY(pack_linear(h, W.data(), 3 * d, d, b.data(), &w.qkv));
    TRY(pack_named(h, n.out + "weight", n.out + "bias", &w.out));
    TRY(pack_named(h, n.fc1 + "weight", n.fc1 + "bias", &w.fc1));
    TRY(pack_named(h, n.fc2 + "weight", n.fc2 + "bias", &w.fc2));
    TRY(pack_ln(h, n.ln1, d, &w.ln1));
    TRY(pack_ln(h, n.ln2, d, &w.ln2));
  }
  return MLDB_OK;
}

// ----------------------------------------------------------------------------- forward
extern "C" int mldb_bert_encode(mldb_handle* h, const int64_t* ids, const int32_t* lengths, int32_t n, int32_t L,
                                float* out, void* stream) {
  if (!h || !ids || !lengths || !out) FAIL(MLDB_ERR_INVALID, "null argument");
  BertW& bw = h->bert;
  TRY(check_configured(h, bw.on, "bert", "the BERT text tower"));
  const mldb_bert_config& c = bw.cfg;
  if (n < 1 || L < 1 || L > c.max_positions) FAIL(MLDB_ERR_INVALID, "ids must be [n >= 1, 1 <= L <= %d]", c.max_positions);
  if ((int64_t)n * L > (1 << 30)) FAIL(MLDB_ERR_INVALID, "too many tokens");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  {
    std::vector<int32_t> ln((size_t)n);
    CK(cudaMemcpyAsync(ln.data(), lengths, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int s = 0; s < n; ++s)
      if (ln[s] < 1 || ln[s] > L) FAIL(MLDB_ERR_INVALID, "lengths[%d] = %d is outside [1, L = %d]", s, ln[s], L);
  }
  const int M = n * L, d = c.hidden;
  ActBuf a, qkv, att, hid;
  TRY(grow(bw.x, (size_t)M * d * sizeof(float)));
  TRY(grow_act(bw.a, M, d, &a));
  TRY(grow_act(bw.qkv, M, 3 * d, &qkv));
  TRY(grow_act(bw.att, M, d, &att));
  TRY(grow_act(bw.h, M, c.ff, &hid));
  float* x = (float*)bw.x.p;
  // post-norm LayerNorm: x = LN(x) in place and a = split16(x) for the next GEMM; the last one writes `out` only
  auto ln = [&](int mode, const LnW& w, float* dst) {
    TextLnArgs l; l.mode = mode; l.x = x; l.ids = ids; l.L = L; l.tok = bw.word; l.pos = bw.pos; l.type0 = bw.type0;
    l.vocab = c.vocab_size; l.gamma = w.g; l.beta = w.b; l.eps = c.ln_eps; l.M = M; l.d = d;
    l.out = dst == x ? a : ActBuf{}; l.out_f32 = dst;
    op_text_ln(h, l, st);
  };
  ln(TEXT_LN_EMBED_LN, bw.emb_ln, x);                                // x = LN_emb(word[id] + pos[t] (+ type[0]))
  for (int i = 0; i < c.layers; ++i) {
    const TextLayerW& w = bw.layers[i];
    GemmArgs g; g.a1 = a; g.K1 = d; g.M = M; g.w = w.qkv; g.out = qkv; g.wide_n = 1;
    op_gemm(h, g, st);
    AttnArgs at; at.q = qkv; at.q_col0 = 0; at.Lq = L; at.kv = qkv; at.k_col0 = d; at.v_col0 = 2 * d; at.Lk = L;
    at.nseq = n; at.heads = c.heads; at.hd = d / c.heads; at.lengths = lengths; at.out = att;
    op_attn(h, at, st);                                              // keys t >= lengths[s] masked, every query row
    GemmArgs go; go.a1 = att; go.K1 = d; go.M = M; go.w = w.out; go.out_f32 = x; go.ldc = d; go.res_f32 = x;
    op_gemm(h, go, st);                                              // x += out_lin(att), in place
    ln(TEXT_LN_ROWS, w.ln1, x);                                      // x = LN_sa(x)
    GemmArgs g1; g1.a1 = a; g1.K1 = d; g1.M = M; g1.w = w.fc1; g1.act = ACT_GELU; g1.out = hid; g1.wide_n = 1;
    op_gemm(h, g1, st);
    GemmArgs g2; g2.a1 = hid; g2.K1 = c.ff; g2.M = M; g2.w = w.fc2; g2.out_f32 = x; g2.ldc = d; g2.res_f32 = x;
    op_gemm(h, g2, st);                                              // x += lin2(gelu(lin1(x)))
    ln(TEXT_LN_ROWS, w.ln2, i + 1 < c.layers ? x : out);             // x = LN_out(x); the last layer's rows go to out
  }
  return ops_done(h);
}
