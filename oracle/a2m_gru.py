"""Float64 restatement of the HumanAct12 action classifier (TEST INFRASTRUCTURE).

``MotionDiscriminator`` / ``MotionDiscriminatorForFID`` (action2motion's classifier as MLD's ``HUMANACTMetrics`` uses
it) written from torch's documented ``nn.GRU`` / ``nn.Linear`` semantics: a stack of GRU layers over the frames, the
last layer's output at ``lengths - 1``, ``tanh(linear1)`` and ``linear2``.  Plain tensor arithmetic and an explicit
cell loop, in whatever dtype and on whatever device the inputs are; the initial state is explicit.
"""
from __future__ import annotations

from typing import Dict, Sequence, Tuple

import torch

Tensor = torch.Tensor


def classify(sd: Dict[str, Tensor], x: Tensor, lengths: Sequence[int], h0: Tensor) -> Tuple[Tensor, Tensor]:
    """x [B, C, T] (or [B, njoints, nfeats, T]), lengths in [1, T], h0 [layers, B, H] -> (logits, features [B, 30]).
    A row's state stops changing after its length, so the last layer's final state is its output at lengths - 1."""
    if x.dim() == 4:
        x = x.reshape(x.shape[0], -1, x.shape[-1])
    w = {k: v.to(x) for k, v in sd.items()}
    B, _, T = x.shape
    H = h0.shape[-1]
    lens = torch.as_tensor(list(lengths), device=x.device)
    inp = x.permute(0, 2, 1)                                     # [B, T, C]
    layers = sum(1 for k in w if k.startswith("recurrent.weight_ih_l"))
    h = None
    for k in range(layers):
        W_ih, W_hh = w[f"recurrent.weight_ih_l{k}"], w[f"recurrent.weight_hh_l{k}"]
        b_ih, b_hh = w[f"recurrent.bias_ih_l{k}"], w[f"recurrent.bias_hh_l{k}"]
        h = h0[k].to(x).clone()
        outs = []
        for s in range(T):
            live = (s < lens)[:, None]
            xt = torch.where(live, inp[:, s], torch.zeros_like(inp[:, s]))   # frames past a length are never used
            gi = xt @ W_ih.T + b_ih
            gh = h @ W_hh.T + b_hh
            r = torch.sigmoid(gi[:, :H] + gh[:, :H])
            z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
            n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
            h = torch.where(live, (1 - z) * n + z * h, h)
            outs.append(h)
        inp = torch.stack(outs, 1)
    feats = torch.tanh(h @ w["linear1.weight"].T + w["linear1.bias"])
    return feats @ w["linear2.weight"].T + w["linear2.bias"], feats


class TorchDiscriminator(torch.nn.Module):
    """The classifier as torch modules (nn.GRU, nn.Linear) with the reference's forward semantics: the initial state
    is ``torch.randn(layers, B, H)`` on the CPU default generator when none is given, then moved to the input's
    device.  The yardstick for fp32 torch (cuDNN) timings and errors, and the seeded-RNG comparisons."""

    def __init__(self, sd: Dict[str, Tensor], input_size: int, hidden_size: int, hidden_layer: int, output_size: int):
        super().__init__()
        self.hidden_size, self.hidden_layer = hidden_size, hidden_layer
        self.recurrent = torch.nn.GRU(input_size, hidden_size, hidden_layer)
        self.linear1 = torch.nn.Linear(hidden_size, 30)
        self.linear2 = torch.nn.Linear(30, output_size)
        self.load_state_dict(sd, strict=True)
        self.eval()

    def both(self, x: Tensor, lengths: Tensor, h0: Tensor = None) -> Tuple[Tensor, Tensor]:
        B, T = x.shape[0], x.shape[-1]
        seq = x.reshape(B, -1, T).permute(2, 0, 1).float()
        if h0 is None:
            h0 = torch.randn(self.hidden_layer, B, self.hidden_size).to(x.device)
        out, _ = self.recurrent(seq, h0)
        last = out[torch.as_tensor(lengths, device=x.device) - 1, torch.arange(B, device=x.device)]
        feats = torch.tanh(self.linear1(last))
        return self.linear2(feats), feats
