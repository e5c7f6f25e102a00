"""CPU: the BERT text tower's float64 restatement against the reference's MldTextEncoder and transformers' BertModel
(tests/golden/bert_text.npz), the synthetic state dict's key contract, and B200TextEncoder's host side for "bert"
paths (loading a saved model, refusals, mask handling, the exact row deduplication) - none of which needs a GPU."""
import os

import pytest
import torch

from conftest import golden
from mld_b200 import synth
from mld_b200.text import (B200TextEncoder, BertTextConfig, bert_config_from_hf, mask_lengths, plan_bert_rows)
from oracle.bert_text import BertTextCfg, bert_text_forward
from oracle.make_golden_bert import BERT_SEED, BERT_SHAPE, WEIGHT_SEED, write_vocab

torch.set_grad_enabled(False)
SMALL = dict(vocab_size=400, max_positions=64, type_vocab=2, hidden=128, heads=2, layers=2, ff=256)


def _rel_rows(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return max(float((a[i] - b[i]).abs().max() / b[i].abs().max()) for i in range(a.shape[0]))


@pytest.mark.parametrize("tag", ["distil", "bert"])
def test_oracle_matches_reference_golden(tag):
    g = golden("bert_text.npz")
    if tag == "distil":
        sd, cfg = synth.bert_text_state_dict(WEIGHT_SEED), BertTextCfg()
    else:
        sd, cfg = synth.bert_text_state_dict(BERT_SEED, **BERT_SHAPE), BertTextCfg(**BERT_SHAPE)
    ids, mask = torch.from_numpy(g[f"{tag}_ids"]), torch.from_numpy(g[f"{tag}_mask"])
    pos = torch.from_numpy(g[f"{tag}_pos"])
    ref = bert_text_forward(sd, ids, mask_lengths(mask, *ids.shape), cfg)
    assert _rel_rows(ref[:, pos], g[f"{tag}_hidden"]) < 1e-5
    lengths = mask.sum(1)
    assert bool((pos[None] >= lengths[:, None]).any()), "the fixture keeps padding positions"


@pytest.mark.parametrize("family", ["distilbert", "bert"])
def test_synth_keys_are_the_hf_model(family):
    T = pytest.importorskip("transformers")
    sd = synth.bert_text_state_dict(3, family=family, **SMALL)
    if family == "distilbert":
        m = T.DistilBertModel(T.DistilBertConfig(vocab_size=400, max_position_embeddings=64, dim=128, n_heads=2,
                                                 n_layers=2, hidden_dim=256))
    else:
        m = T.BertModel(T.BertConfig(vocab_size=400, max_position_embeddings=64, hidden_size=128, num_attention_heads=2,
                                     num_hidden_layers=2, intermediate_size=256))
    hf = {"text_model." + k: tuple(v.shape) for k, v in m.state_dict().items() if not k.endswith("position_ids")}
    assert {k: tuple(v.shape) for k, v in sd.items()} == hf
    m.load_state_dict({k[len("text_model."):]: v for k, v in sd.items()}, strict=True)
    enc = B200TextEncoder.from_state_dict(sd, config=BertTextConfig(family=family, **SMALL))
    assert set(enc.state_dict()) == set(sd) and enc.name == "bert" and enc.text_encoded_dim == 128


def _save_tiny(path, family="distilbert"):
    T = pytest.importorskip("transformers")
    os.makedirs(path)
    write_vocab(os.path.join(path, "vocab.txt"), 400)
    T.DistilBertTokenizer(os.path.join(path, "vocab.txt")).save_pretrained(path)
    m = T.DistilBertModel(T.DistilBertConfig(vocab_size=400, max_position_embeddings=64, dim=128, n_heads=2,
                                             n_layers=2, hidden_dim=256))
    m.save_pretrained(path)
    return m


def test_load_saved_model(tmp_path):
    path = str(tmp_path / "tiny-distilbert")
    m = _save_tiny(path)
    enc = B200TextEncoder(path, last_hidden_state=True)          # last_hidden_state is ignored for bert
    assert enc.name == "bert" and enc.text_encoded_dim == 128
    assert enc.text_cfg == BertTextConfig(family="distilbert", **{**SMALL, "type_vocab": 2})
    assert set(enc.state_dict()) == {"text_model." + k for k in m.state_dict()}
    tok = enc.tokenizer(["", "a person walks"], return_tensors="pt", padding=True)
    assert tok["input_ids"][0, :2].tolist() == [101, 102] and tok["attention_mask"][0, 2:].sum() == 0


def test_refusals_before_touching_a_device(tmp_path):
    T = pytest.importorskip("transformers")
    with pytest.raises(NotImplementedError):
        B200TextEncoder("./deps/distilbert-base-uncased", finetune=True)
    with pytest.raises(ValueError):                               # not a saved model directory
        B200TextEncoder(str(tmp_path / "missing-bert"))
    d = tmp_path / "tiny-roberta"                                  # "roberta" contains "bert"
    d.mkdir()
    T.RobertaConfig(vocab_size=50, hidden_size=32, num_hidden_layers=1, num_attention_heads=2,
                    intermediate_size=64).save_pretrained(str(d))
    with pytest.raises(NotImplementedError):
        B200TextEncoder(str(d))
    for bad in (T.DistilBertConfig(sinusoidal_pos_embds=True), T.DistilBertConfig(activation="relu"),
                T.BertConfig(hidden_act="gelu_new"), T.BertConfig(is_decoder=True),
                T.BertConfig(add_cross_attention=True), T.RobertaConfig()):
        with pytest.raises(NotImplementedError):
            bert_config_from_hf(bad)
    rel = T.BertConfig()
    rel.position_embedding_type = "relative_key"
    with pytest.raises(NotImplementedError):
        bert_config_from_hf(rel)
    assert bert_config_from_hf(T.DistilBertConfig()) == BertTextConfig()
    assert bert_config_from_hf(T.BertConfig(layer_norm_eps=1e-6)) == BertTextConfig(
        family="bert", layers=12, ln_eps=1e-6)


def test_mask_and_id_checks():
    sd = synth.bert_text_state_dict(1, **SMALL)
    enc = B200TextEncoder.from_state_dict(sd, config=BertTextConfig(**SMALL))
    ids = torch.ones(2, 5, dtype=torch.long)
    assert mask_lengths(None, 2, 5).tolist() == [5, 5]
    assert mask_lengths(torch.tensor([[1, 1, 0, 0, 0], [1, 1, 1, 1, 1]]), 2, 5).tolist() == [2, 5]
    for bad in (torch.tensor([[1, 0, 1, 0, 0], [1] * 5]),       # not a prefix
                torch.tensor([[0] * 5, [1] * 5]),                # no token
                torch.tensor([[2, 1, 0, 0, 0], [1] * 5]),        # not 0 / 1
                torch.ones(2, 4)):                               # wrong shape
        with pytest.raises(ValueError):
            enc.encode_ids(ids, bad)
    for bad in (torch.tensor([[1, 400]]), torch.tensor([[-1, 3]]), torch.ones(1, 65, dtype=torch.long),
                torch.ones(2, 3)):
        with pytest.raises((ValueError, TypeError)):
            enc.encode_ids(bad)

    def tokenizer(texts, return_tensors, padding):
        assert return_tensors == "pt" and padding is True
        return {"input_ids": torch.ones(len(texts), 3, dtype=torch.long),
                "attention_mask": torch.ones(len(texts), 3, dtype=torch.long),
                "token_type_ids": torch.tensor([[0, 0, 1]] * len(texts))}
    enc.tokenizer = tokenizer
    with pytest.raises(ValueError):                              # a second segment
        enc(["a b"])
    enc.tokenizer = lambda texts, **kw: {"input_ids": torch.ones(1, 65, dtype=torch.long)}
    with pytest.raises(ValueError):                              # longer than max_positions: the reference fails too
        enc(["a"])
    clip = B200TextEncoder.from_state_dict(synth.clip_text_state_dict(1, vocab_size=1000, hidden=128, layers=1, ff=256,
                                                                      projection_dim=64))
    with pytest.raises(ValueError):                              # CLIP takes no mask
        clip.encode_ids(torch.ones(1, 77, dtype=torch.long), torch.ones(1, 77))


def test_position_ids_buffer():
    sd = synth.bert_text_state_dict(1, **SMALL)
    cfg = BertTextConfig(**SMALL)
    enc = B200TextEncoder.from_state_dict({**sd, "text_model.embeddings.position_ids": torch.arange(64)[None]},
                                          config=cfg)
    assert set(enc.state_dict()) == set(sd)
    with pytest.raises(ValueError):
        B200TextEncoder.from_state_dict({**sd, "text_model.embeddings.position_ids": torch.zeros(1, 64)}, config=cfg)


def test_dedupe_is_exact():
    """The CFG batch [""] * B + prompts: every distinct (ids, length) row once, gathered back, gives every row."""
    sd = synth.bert_text_state_dict(2, **SMALL)
    cfg = BertTextCfg(**SMALL)
    ids, lengths = synth.bert_text_ids(6, 20, seed=4, len_lo=3, len_hi=20, vocab_size=400)
    empty = torch.zeros(3, 20, dtype=torch.long)
    empty[:, 0], empty[:, 1] = 101, 102
    ids, lengths = torch.cat([empty, ids]), torch.cat([torch.full((3,), 2), lengths])
    same_ids = ids[3:4].clone()                                   # the same ids under another mask: a distinct row
    ids, lengths = torch.cat([ids, same_ids]), torch.cat([lengths, (lengths[3:4] - 1).clamp(min=1)])
    rows, row_len, inv = plan_bert_rows(ids, lengths)
    assert rows.shape[0] == ids.shape[0] - 2
    assert torch.equal(rows[inv], ids) and torch.equal(row_len[inv], lengths)
    full = bert_text_forward(sd, ids, lengths, cfg)
    assert float((bert_text_forward(sd, rows, row_len, cfg)[inv] - full).abs().max()) == 0.0
