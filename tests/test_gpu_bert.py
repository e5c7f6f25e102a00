"""GPU tests of the native BERT text encoder (pytest -m gpu): the full DistilBERT tower against float64 over the
sequence lengths the API accepts, with random right padding, the reference fixture for both layouts, kernel selection,
the CUDA-core twins, row independence and the exact deduplication, packed weights at split16 exponents other than
14, and text -> joints end to end against the oracle chain."""
import os

import pytest
import torch

from conftest import golden
from mld_b200 import synth
from oracle import mld_oracle as O
from oracle.bert_text import BertTextCfg, bert_text_forward
from oracle.make_golden_bert import BERT_SEED, BERT_SHAPE, WEIGHT_SEED, write_vocab

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
TOL = 1e-4              # per sequence, relative to the sequence's largest value (the CLIP tower's gate)
LAYERS = 6


def _rel_rows(a, b):
    """Worst per-sequence relative-to-max error (a, b: [n, ...])."""
    a, b = a.double().flatten(1), b.double().to(a.device).flatten(1)
    return float(((a - b).abs().max(1).values / b.abs().max(1).values).max())


def _engine(sd, cfg, options=()):
    from mld_b200.engine import Engine, make_config
    from mld_b200.text import BertTextConfig
    e = Engine(make_config(num_layers=0, vae="none"), 0)
    for k, v in options:
        e.set_option(k, v)
    e.bert_configure(BertTextConfig(**vars(cfg)).to_c())
    e.load_state_dict(sd, "text_encoder.")
    e.finalize()
    return e


@pytest.fixture(scope="module")
def tower(built_lib):
    """A text-only engine with the full DistilBERT tower (synthetic weights) and the float64 weights on the GPU."""
    sd = synth.bert_text_state_dict(WEIGHT_SEED)
    return _engine(sd, BertTextCfg()), sd, {k: v.double().cuda() for k, v in sd.items()}


def _oracle(sd64, ids, lengths, cfg=None, chunk=32):
    out = [bert_text_forward(sd64, ids[c:c + chunk].cuda(), lengths[c:c + chunk].cuda(), cfg or BertTextCfg())
           for c in range(0, ids.shape[0], chunk)]
    return torch.cat(out)


@pytest.mark.parametrize("n,L", [(512, 1), (512, 2), (256, 7), (128, 31), (96, 77), (64, 128), (48, 256), (24, 257),
                                 (512, 512)])
def test_tower_vs_float64(tower, n, L):
    """Every row of every sequence, padding rows included; wgmma attention up to 256 keys, the documented CUDA-core
    attention past that."""
    e, _, sd64 = tower
    ids, lengths = synth.bert_text_ids(n, L, seed=n + L, len_lo=1, len_hi=L)
    e.kernel_stats(reset=True)
    out = e.bert_encode(ids, lengths)
    torch.cuda.synchronize()
    st = e.kernel_stats()
    attn = "attn_tc" if L <= 256 else "attn_simt"
    expect = {"gemm_tc": 4 * LAYERS, attn: LAYERS, "text_ln": 1 + 2 * LAYERS}
    assert {k: v for k, v in st.items() if v} == expect, st
    assert torch.isfinite(out).all()
    err = _rel_rows(out, _oracle(sd64, ids, lengths))
    print(f"\n[bert] n={n} L={L}: {err:.2e} vs float64")
    assert err < TOL


@pytest.mark.parametrize("tag", ["distil", "bert"])
def test_tower_vs_reference_golden(built_lib, tower, tag):
    g = golden("bert_text.npz")
    if tag == "distil":
        e = tower[0]
    else:
        e = _engine(synth.bert_text_state_dict(BERT_SEED, **BERT_SHAPE), BertTextCfg(**BERT_SHAPE))
    ids, mask = torch.from_numpy(g[f"{tag}_ids"]), torch.from_numpy(g[f"{tag}_mask"])
    out = e.bert_encode(ids, mask.sum(1))[:, torch.from_numpy(g[f"{tag}_pos"]).cuda()]
    err = _rel_rows(out, torch.from_numpy(g[f"{tag}_hidden"]))
    print(f"\n[bert] {tag} fixture: {err:.2e}")
    assert err < TOL


@pytest.mark.parametrize("option", ["gemm", "attn"])
def test_cuda_core_twins(tower, option):
    _, sd, sd64 = tower
    e = _engine(sd, BertTextCfg(), [(option, "simt")])
    for n, L in ((40, 77), (6, 300)):
        ids, lengths = synth.bert_text_ids(n, L, seed=L, len_lo=1, len_hi=L)
        e.kernel_stats(reset=True)
        out = e.bert_encode(ids, lengths)
        torch.cuda.synchronize()
        st = e.kernel_stats()
        assert st["attn_simt"] == LAYERS and st["attn_tc"] == 0, st
        assert st["gemm_simt" if option == "gemm" else "gemm_tc"] == 4 * LAYERS, st
        err = _rel_rows(out, _oracle(sd64, ids, lengths))
        print(f"\n[bert] {option}=simt n={n} L={L}: {err:.2e} vs float64")
        assert err < TOL


def test_rows_are_independent_and_dedupe_exact(tower):
    from mld_b200.text import B200TextEncoder, BertTextConfig
    e, sd, _ = tower
    ids, lengths = synth.bert_text_ids(40, 50, seed=3, len_lo=2, len_hi=50)
    base = e.bert_encode(ids, lengths).clone()
    ids2, len2 = ids.clone(), lengths.clone()
    ids2[7, 1] = (ids2[7, 1] + 1) % 30522                        # one row's ids
    len2[12] = max(1, int(len2[12]) - 1)                         # another row's length
    out = e.bert_encode(ids2, len2)
    keep = torch.ones(40, dtype=torch.bool)
    keep[[7, 12]] = False
    assert torch.equal(out[keep.cuda()], base[keep.cuda()])
    assert not torch.equal(out[7], base[7]) and not torch.equal(out[12], base[12])
    enc = B200TextEncoder.from_state_dict(sd, config=BertTextConfig()).cuda()
    enc._engine, enc._engine_epoch = e, enc._weights_epoch      # reuse the module-scoped engine
    empty = torch.zeros(8, 50, dtype=torch.long)
    empty[:, 0], empty[:, 1] = 101, 102
    cfg_ids, cfg_len = torch.cat([empty, ids]), torch.cat([torch.full((8,), 2), lengths])
    mask = (torch.arange(50)[None] < cfg_len[:, None]).long()
    assert torch.equal(enc.encode_ids(cfg_ids, mask), e.bert_encode(cfg_ids, cfg_len))


def test_weights_off_exponent_14(built_lib):
    """Outliers put the packed q|k|v, out_lin, lin1 and lin2 operands at split16 exponents 12, 13, 11 and 12."""
    from weight_scales import engine_exponent
    cfg = BertTextCfg(layers=2)
    sd = synth.bert_text_state_dict(9, layers=2)
    for i in range(2):
        p = f"text_model.transformer.layer.{i}."
        for key, mag in (("attention.k_lin", 3.0), ("attention.out_lin", 1.5), ("ffn.lin1", 6.0), ("ffn.lin2", -3.0)):
            sd[p + key + ".weight"][i, 5] = mag
        qkv = torch.cat([sd[p + f"attention.{x}_lin.weight"] for x in "qkv"])
        assert [engine_exponent(w) for w in (qkv, sd[p + "attention.out_lin.weight"], sd[p + "ffn.lin1.weight"],
                                            sd[p + "ffn.lin2.weight"])] == [12, 13, 11, 12]
    e = _engine(sd, cfg)
    ids, lengths = synth.bert_text_ids(64, 77, seed=5, len_lo=1, len_hi=77)
    err = _rel_rows(e.bert_encode(ids, lengths), _oracle({k: v.double().cuda() for k, v in sd.items()}, ids, lengths,
                                                         cfg))
    print(f"\n[bert] weights at exponents 11-13: {err:.2e} vs float64")
    assert err < TOL


def test_text_to_joints_end_to_end(built_lib, tmp_path):
    """B200MLD(text_encoder=B200TextEncoder(saved DistilBERT)) against the oracle chain (float64 BERT ->
    oracle.mld_forward), under classifier-free guidance; two batches with different padded lengths in one session."""
    import transformers as T
    from mld_b200.pipeline import B200MLD
    from mld_b200.text import B200TextEncoder
    path = str(tmp_path / "distilbert-2layer")
    os.makedirs(path)
    write_vocab(os.path.join(path, "vocab.txt"))
    T.DistilBertTokenizer(os.path.join(path, "vocab.txt")).save_pretrained(path)
    sd = synth.bert_text_state_dict(WEIGHT_SEED, layers=2)
    m = T.DistilBertModel(T.DistilBertConfig(n_layers=2))
    m.load_state_dict({k[len("text_model."):]: v for k, v in sd.items()}, strict=True)
    m.save_pretrained(path)
    enc = B200TextEncoder(path).cuda()
    assert enc.name == "bert" and enc.text_encoded_dim == 768
    dsd, vsd = synth.denoiser_state_dict(1234), synth.mld_vae_state_dict(4321)
    mean, std = synth.mean_std()
    model = B200MLD(dsd, vsd, mean=mean, std=std, text_encoder=enc)
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    seen_L = set()
    for texts, lengths, seed in ((["a person walks forward and turns left", "jump", "someone waves"], [196, 64, 120], 5),
                                 (["the man slowly circles around the room then sits down on the chair", "run"],
                                  [80, 160], 6)):
        noise = synth.init_noise(len(texts), seed=seed)
        joints = model({"text": texts, "length": lengths, "init_noise": noise})
        tok = enc.tokenizer([""] * len(texts) + texts, return_tensors="pt", padding=True)
        ctx = bert_text_forward(sd64, tok["input_ids"].cuda(), tok["attention_mask"].sum(1).cuda(),
                                BertTextCfg(layers=2)).float().cpu()
        seen_L.add(ctx.shape[1])
        jo, _, _ = O.mld_forward(dsd, O.DenoiserCfg(), vsd, O.VaeCfg(), O.DDIMScheduler(), 50, ctx, noise, lengths,
                                 mean, std)
        err = max(float((a - r).abs().max() / r.abs().max()) for a, r in zip(joints, jo))
        print(f"\n[bert] text -> joints, S_ctx {ctx.shape[1]}: {err:.2e} vs the oracle chain")
        assert err < 1e-3
    assert len(seen_L) == 2
