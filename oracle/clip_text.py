"""Plain-torch restatement of the CLIP text tower behind ``MldTextEncoder`` (TEST INFRASTRUCTURE ONLY).

``mld/models/architectures/mld_clip.py:53-97`` calls transformers' CLIP: ``get_text_features(ids)`` (mode
``clip``) or ``text_model(ids).last_hidden_state`` (mode ``clip_hidden``).  This file restates that tower without
importing transformers: token + position embedding, pre-norm layers (LayerNorm -> causal multi-head
self-attention -> residual, LayerNorm -> fc1 -> quick-GELU -> fc2 -> residual), the final LayerNorm, and for
``clip`` the eos-row gather plus ``text_projection``.  It runs in any dtype (float64 for the GPU tests).
Pinned against transformers' ``CLIPTextModelWithProjection`` through ``tests/golden/clip_text.npz``
(``oracle/make_golden_clip.py``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


@dataclass
class ClipTextCfg:
    """CLIP ViT-L/14 text config (transformers ``CLIPTextConfig`` + ``CLIPConfig.projection_dim``)."""
    vocab_size: int = 49408
    max_positions: int = 77
    hidden: int = 768
    heads: int = 12
    layers: int = 12
    ff: int = 3072
    projection_dim: int = 768
    eos_token_id: int = 49407
    ln_eps: float = 1e-5


def eos_positions(ids: Tensor, eos_token_id: int) -> Tensor:
    """Row index of the pooled token (transformers CLIPTextTransformer.forward): the first id equal to
    ``eos_token_id`` (0 when absent); with the legacy ``eos_token_id == 2``, ``argmax(ids)``."""
    ids32 = ids.to(torch.int32)
    if eos_token_id == 2:
        return ids32.argmax(dim=-1)
    return (ids32 == eos_token_id).int().argmax(dim=-1)


def clip_text_forward(sd: Dict[str, Tensor], ids: Tensor, mode: str = "clip", cfg=None,
                      dtype: torch.dtype = torch.float64) -> Tensor:
    """``sd``: ``MldTextEncoder`` text-tower keys (``text_model.text_model.*``, ``text_model.text_projection.weight``);
    ``ids`` int64 [n, L].  Returns [n, L, hidden] (``clip_hidden``) or [n, 1, projection_dim] (``clip``)."""
    cfg = cfg or ClipTextCfg()
    p = "text_model.text_model."
    W = lambda k: sd[k].to(dtype)                                  # noqa: E731
    n, L = ids.shape
    d, nh = cfg.hidden, cfg.heads
    hd = d // nh
    x = W(p + "embeddings.token_embedding.weight")[ids] + W(p + "embeddings.position_embedding.weight")[:L]
    mask = torch.full((L, L), float("-inf"), dtype=dtype, device=x.device).triu(1)   # key j > query i is masked

    def ln(t, q):
        return F.layer_norm(t, (d,), W(q + "weight"), W(q + "bias"), cfg.ln_eps)

    def heads(t):
        return t.view(n, L, nh, hd).transpose(1, 2)

    for i in range(cfg.layers):
        q = f"{p}encoder.layers.{i}."
        h = ln(x, q + "layer_norm1.")
        a = q + "self_attn."
        Q = heads(F.linear(h, W(a + "q_proj.weight"), W(a + "q_proj.bias")))
        K = heads(F.linear(h, W(a + "k_proj.weight"), W(a + "k_proj.bias")))
        V = heads(F.linear(h, W(a + "v_proj.weight"), W(a + "v_proj.bias")))
        P = torch.softmax(Q @ K.transpose(-1, -2) * hd ** -0.5 + mask, dim=-1)
        o = (P @ V).transpose(1, 2).reshape(n, L, d)
        x = x + F.linear(o, W(a + "out_proj.weight"), W(a + "out_proj.bias"))
        h = F.linear(ln(x, q + "layer_norm2."), W(q + "mlp.fc1.weight"), W(q + "mlp.fc1.bias"))
        h = h * torch.sigmoid(1.702 * h)                           # quick_gelu
        x = x + F.linear(h, W(q + "mlp.fc2.weight"), W(q + "mlp.fc2.bias"))
    x = ln(x, p + "final_layer_norm.")
    if mode == "clip_hidden":
        return x
    if mode != "clip":
        raise ValueError(mode)
    pooled = x[torch.arange(n, device=x.device), eos_positions(ids, cfg.eos_token_id).to(x.device)]
    return F.linear(pooled, W("text_model.text_projection.weight")).unsqueeze(1)
