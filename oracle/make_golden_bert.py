"""Generate tests/golden/bert_text.npz with the reference's own MldTextEncoder and transformers' BertModel (TEST
INFRASTRUCTURE).

    python -m oracle.make_golden_bert REFERENCE_ROOT      (or MLD_REFERENCE=REFERENCE_ROOT python -m ...)

DistilBERT: the seeded synthetic weights of ``mld_b200.synth.bert_text_state_dict`` (distilbert-base-uncased's
shape) are loaded into transformers' ``DistilBertModel`` with ``strict=True`` and saved, with a generated 30522-line
WordPiece ``vocab.txt``, into a temporary directory whose name contains ``bert``.  The reference's
``mld/models/architectures/mld_clip.py`` is imported by file path and its ``MldTextEncoder(modelpath=that
directory)`` is run in fp32 on PROMPTS, as ``MLD`` calls it under classifier-free guidance: one right-padded batch
(``""`` first, one prompt past 256 tokens).  BERT: a small seeded ``BertModel`` (``BERT_SHAPE``) runs on seeded id
rows with their attention masks and zero token types.  Only ids, masks and the hidden rows at HIDDEN_POS are stored
(padding positions included); the weights are rebuilt from the seeds by the tests.  Nothing leaves the machine:
transformers runs offline.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import tempfile

os.environ.setdefault("HF_HUB_OFFLINE", "1")
os.environ.setdefault("TRANSFORMERS_OFFLINE", "1")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "bert_text.npz")
WEIGHT_SEED, BERT_SEED, BERT_IDS_SEED = 5151, 5252, 77
# a "" prompt (uncond row), two short prompts, and one that fills more than 256 positions
PROMPTS = ("", "a person walks forward and turns left", "someone jumps twice then waves with both hands",
           " ".join(["the man slowly circles around the room"] * 40))
HIDDEN_POS = 12          # positions kept per row: every row's [SEP], the positions around it and a spread of pads
BERT_SHAPE = dict(family="bert", vocab_size=1000, max_positions=128, type_vocab=2, hidden=256, heads=4, layers=2,
                  ff=1024, ln_eps=1e-12)
BERT_N, BERT_L = 5, 40


def write_vocab(path: str, size: int = 30522):
    """A WordPiece vocabulary laid out like bert-base-uncased's: [PAD] 0, [UNK] 100, [CLS] 101, [SEP] 102,
    [MASK] 103, then single characters, their ## continuations and filler words up to ``size`` lines."""
    special = {0: "[PAD]", 100: "[UNK]", 101: "[CLS]", 102: "[SEP]", 103: "[MASK]"}
    toks = [special.get(i, f"[unused{i}]") for i in range(104)]
    chars = [chr(c) for c in range(ord("a"), ord("z") + 1)] + [str(i) for i in range(10)] + list(".,!?'-")
    toks += chars + ["##" + c for c in chars]
    words = sorted(set(" ".join(PROMPTS[1:]).split()))
    toks += [w for w in words if w not in toks]
    toks += [f"w{i}" for i in range(size - len(toks))]
    with open(path, "w") as f:
        f.write("\n".join(toks) + "\n")


def positions(lengths, L: int):
    """At least HIDDEN_POS positions over a batch of right-padded rows: 0, L - 1, each row's last real position and
    the one after it, then evenly spread others (so every padded row has real and padding positions)."""
    pos = {0, L - 1}
    for n in lengths:
        pos |= {n - 1, min(n, L - 1)}
    for p in np.linspace(0, L - 1, HIDDEN_POS).astype(int).tolist():
        if len(pos) >= HIDDEN_POS:
            break
        pos.add(p)
    return np.array(sorted(pos), dtype=np.int64)


def load_reference_encoder(ref_root: str):
    sys.path.insert(0, ref_root)
    path = os.path.join(ref_root, "mld", "models", "architectures", "mld_clip.py")
    spec = importlib.util.spec_from_file_location("ref_mld_clip", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.MldTextEncoder


def main(ref_root: str = ""):
    ref_root = ref_root or os.environ.get("MLD_REFERENCE", "")
    if not ref_root:
        raise SystemExit("give the reference checkout (ChenFengYe/motion-latent-diffusion) as an argument or MLD_REFERENCE")
    import transformers as T
    from mld_b200 import synth
    torch.set_grad_enabled(False)
    MldTextEncoder = load_reference_encoder(ref_root)
    out = {}
    sd = synth.bert_text_state_dict(WEIGHT_SEED)
    with tempfile.TemporaryDirectory() as tmp:
        d = os.path.join(tmp, "distilbert-base-uncased")
        os.makedirs(d)
        write_vocab(os.path.join(d, "vocab.txt"))
        T.DistilBertTokenizer(os.path.join(d, "vocab.txt")).save_pretrained(d)
        m = T.DistilBertModel(T.DistilBertConfig())
        m.load_state_dict({k[len("text_model."):]: v for k, v in sd.items()}, strict=True)
        m.save_pretrained(d)
        enc = MldTextEncoder(modelpath=d).eval()
        assert enc.name == "bert" and enc.text_encoded_dim == 768
        hidden = enc(list(PROMPTS))
        tok = enc.tokenizer(list(PROMPTS), return_tensors="pt", padding=True)
    ids, mask = tok["input_ids"], tok["attention_mask"]
    lengths = mask.sum(1).tolist()
    assert ids.shape[1] > 256 and max(lengths) == ids.shape[1], ids.shape
    pos = positions(lengths, ids.shape[1])
    out.update(distil_ids=ids.numpy(), distil_mask=mask.numpy(), distil_pos=pos,
               distil_hidden=hidden[:, torch.from_numpy(pos)].numpy())

    bsd = synth.bert_text_state_dict(BERT_SEED, **BERT_SHAPE)
    c = BERT_SHAPE
    bm = T.BertModel(T.BertConfig(vocab_size=c["vocab_size"], hidden_size=c["hidden"], num_hidden_layers=c["layers"],
                                  num_attention_heads=c["heads"], intermediate_size=c["ff"],
                                  max_position_embeddings=c["max_positions"], type_vocab_size=c["type_vocab"],
                                  layer_norm_eps=c["ln_eps"])).eval()
    bm.load_state_dict({k[len("text_model."):]: v for k, v in bsd.items()}, strict=True)
    bids, blen = synth.bert_text_ids(BERT_N, BERT_L, seed=BERT_IDS_SEED, len_lo=1, len_hi=BERT_L,
                                     vocab_size=c["vocab_size"])
    bmask = (torch.arange(BERT_L)[None] < blen[:, None]).long()
    bh = bm(input_ids=bids, attention_mask=bmask, token_type_ids=torch.zeros_like(bids)).last_hidden_state
    bpos = positions(blen.tolist(), BERT_L)
    out.update(bert_ids=bids.numpy(), bert_mask=bmask.numpy(), bert_pos=bpos,
               bert_hidden=bh[:, torch.from_numpy(bpos)].numpy())

    from oracle.bert_text import BertTextCfg, bert_text_forward
    for tag, w, cfg in (("distil", sd, BertTextCfg()), ("bert", bsd, BertTextCfg(**BERT_SHAPE))):
        i, mk, p = (torch.from_numpy(out[f"{tag}_{k}"]) for k in ("ids", "mask", "pos"))
        ref = bert_text_forward(w, i, mk.sum(1), cfg)[:, p]
        err = float((ref - torch.from_numpy(out[f"{tag}_hidden"]).double()).abs().max())
        print(f"{tag}: oracle vs transformers, max abs {err:.3e}")
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main(*sys.argv[1:])
