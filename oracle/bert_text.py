"""Plain-torch restatement of the BERT text tower behind ``MldTextEncoder`` with a ``"bert"`` model path (TEST
INFRASTRUCTURE ONLY).

``mld/models/architectures/mld_clip.py:65-68,83-86`` tokenizes with ``padding=True`` and returns
``text_model(**text_inputs).last_hidden_state`` of transformers' ``DistilBertModel`` (distilbert-base-uncased) or
``BertModel``.  This file restates that without importing transformers: word + position (+ token-type row 0 for BERT,
added before the position) embedding and LayerNorm, then post-norm layers (non-causal multi-head self-attention with
the padding keys masked -> residual -> LayerNorm, lin1 -> exact GELU -> lin2 -> residual -> LayerNorm).  Every
position is returned, padding positions included.  It runs in any dtype: float64 is the GPU tests' yardstick, float32
the eager torch baseline.  Pinned against the reference's own ``MldTextEncoder`` and transformers' ``BertModel``
through ``tests/golden/bert_text.npz`` (``oracle/make_golden_bert.py``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


@dataclass
class BertTextCfg:
    """distilbert-base-uncased's shape; ``family="bert"`` adds the token-type row and BertModel's key names."""
    family: str = "distilbert"
    vocab_size: int = 30522
    max_positions: int = 512
    type_vocab: int = 2
    hidden: int = 768
    heads: int = 12
    layers: int = 6
    ff: int = 3072
    ln_eps: float = 1e-12


def _layer_keys(cfg: BertTextCfg, i: int):
    if cfg.family == "distilbert":
        p = f"text_model.transformer.layer.{i}."
        return (p + "attention.q_lin.", p + "attention.k_lin.", p + "attention.v_lin.", p + "attention.out_lin.",
                p + "sa_layer_norm.", p + "ffn.lin1.", p + "ffn.lin2.", p + "output_layer_norm.")
    p = f"text_model.encoder.layer.{i}."
    return (p + "attention.self.query.", p + "attention.self.key.", p + "attention.self.value.",
            p + "attention.output.dense.", p + "attention.output.LayerNorm.", p + "intermediate.dense.",
            p + "output.dense.", p + "output.LayerNorm.")


def bert_text_forward(sd: Dict[str, Tensor], ids: Tensor, lengths: Tensor, cfg: BertTextCfg = None,
                      dtype: torch.dtype = torch.float64) -> Tensor:
    """``sd``: ``MldTextEncoder`` keys (``text_model.`` + the HF model's); ``ids`` int64 [n, L]; ``lengths`` [n], each
    in [1, L] (the attention mask as a prefix length).  Returns last_hidden_state [n, L, hidden]."""
    cfg = cfg or BertTextCfg()
    W = lambda k: sd[k].to(device=ids.device, dtype=dtype)          # noqa: E731
    n, L = ids.shape
    d, nh = cfg.hidden, cfg.heads
    hd = d // nh
    e = "text_model.embeddings."
    x = W(e + "word_embeddings.weight")[ids]
    if cfg.family == "bert":
        x = x + W(e + "token_type_embeddings.weight")[0]
    x = x + W(e + "position_embeddings.weight")[:L]

    def ln(t, q):
        return F.layer_norm(t, (d,), W(q + "weight"), W(q + "bias"), cfg.ln_eps)

    def lin(t, q):
        return F.linear(t, W(q + "weight"), W(q + "bias"))

    def heads(t):
        return t.view(n, L, nh, hd).transpose(1, 2)

    x = ln(x, e + "LayerNorm.")
    keep = torch.arange(L, device=ids.device)[None] < lengths.to(ids.device)[:, None]          # [n, L] real keys
    bias = torch.zeros(n, 1, 1, L, dtype=dtype, device=ids.device).masked_fill(~keep[:, None, None], float("-inf"))
    for i in range(cfg.layers):
        q, k, v, o, ln1, fc1, fc2, ln2 = _layer_keys(cfg, i)
        P = torch.softmax(heads(lin(x, q)) @ heads(lin(x, k)).transpose(-1, -2) * hd ** -0.5 + bias, dim=-1)
        a = (P @ heads(lin(x, v))).transpose(1, 2).reshape(n, L, d)
        x = ln(x + lin(a, o), ln1)
        x = ln(x + lin(F.gelu(lin(x, fc1)), fc2), ln2)
    return x
