"""Float64 restatement of the T2M evaluator's three networks (TEST INFRASTRUCTURE).

Written from the published architecture (Guo et al., "Generating Diverse and Natural 3D Human Motions from Text",
CVPR 2022, as used by MLD's ``t2m_eval``) and torch's documented ``nn.GRU`` / ``nn.Conv1d`` semantics: plain tensor
arithmetic and an explicit GRU cell loop, in whatever dtype and on whatever device the inputs are (the tests pass
float64).  State dicts are the finest.tar ones (``mld_b200.synth.t2m_state_dicts``).
"""
from __future__ import annotations

from typing import Dict, Sequence

import torch

Tensor = torch.Tensor


def _leaky(x: Tensor) -> Tensor:
    return torch.where(x > 0, x, 0.2 * x)


def _conv_k4s2p1(x: Tensor, w: Tensor, b: Tensor) -> Tensor:
    """Conv1d(kernel 4, stride 2, padding 1) over the time axis of x [B, T, C]; w [O, C, 4] -> [B, T // 2, O]."""
    B, T, C = x.shape
    xp = torch.cat([x.new_zeros(B, 1, C), x, x.new_zeros(B, 1, C)], 1)     # zero frame on each side
    To = (T + 2 - 4) // 2 + 1
    y = x.new_zeros(B, To, w.shape[0]) + b
    for k in range(4):
        y = y + xp[:, k:k + 2 * To - 1:2] @ w[:, :, k].T                    # frame 2t + k - 1 of the input
    return y


def movement(sd: Dict[str, Tensor], x: Tensor) -> Tensor:
    """MovementConvEncoder: x [B, T, dim_pose] -> [B, T // 2 // 2, dim_move_latent]; every frame is read."""
    w = {k: v.to(x) for k, v in sd.items()}
    h = _leaky(_conv_k4s2p1(x, w["main.0.weight"], w["main.0.bias"]))
    h = _leaky(_conv_k4s2p1(h, w["main.3.weight"], w["main.3.bias"]))
    return h @ w["out_net.weight"].T + w["out_net.bias"]


def _gru_direction(w: Dict[str, Tensor], sfx: str, x: Tensor, lengths: Sequence[int], h0: Tensor) -> Tensor:
    """Final state of one direction of nn.GRU over each sequence's first lengths[b] steps (gate rows r | z | n).
    The forward direction reads step s at step s, the backward one step len - 1 - s; a finished row keeps its state."""
    B, H = x.shape[0], h0.shape[-1]
    W_ih, W_hh = w["gru.weight_ih_l0" + sfx], w["gru.weight_hh_l0" + sfx]
    b_ih, b_hh = w["gru.bias_ih_l0" + sfx], w["gru.bias_hh_l0" + sfx]
    lens = torch.tensor(list(lengths), device=x.device)
    rows = torch.arange(B, device=x.device)
    h = h0.expand(B, H).clone()
    for s in range(int(lens.max())):
        t = torch.full_like(lens, s) if sfx == "" else (lens - 1 - s).clamp(min=0)
        gi = x[rows, t] @ W_ih.T + b_ih
        gh = h @ W_hh.T + b_hh
        r = torch.sigmoid(gi[:, :H] + gh[:, :H])
        z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
        c = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
        h = torch.where((s < lens)[:, None], (1 - z) * c + z * h, h)
    return h


def _bigru_head(w: Dict[str, Tensor], x: Tensor, lengths: Sequence[int]) -> Tensor:
    hf = _gru_direction(w, "", x, lengths, w["hidden"][0, 0])
    hb = _gru_direction(w, "_reverse", x, lengths, w["hidden"][1, 0])
    y = torch.cat([hf, hb], -1) @ w["output_net.0.weight"].T + w["output_net.0.bias"]
    y = torch.nn.functional.layer_norm(y, y.shape[-1:], w["output_net.1.weight"], w["output_net.1.bias"], 1e-5)
    return _leaky(y) @ w["output_net.3.weight"].T + w["output_net.3.bias"]


def motion(sd: Dict[str, Tensor], x: Tensor, lengths: Sequence[int]) -> Tensor:
    """MotionEncoderBiGRUCo: x [B, L, dim_move_latent], lengths (any order) -> [B, dim_motion_latent]."""
    w = {k: v.to(x) for k, v in sd.items()}
    e = x @ w["input_emb.weight"].T + w["input_emb.bias"]
    return _bigru_head(w, e, [int(n) for n in lengths])


def text(sd: Dict[str, Tensor], word_embs: Tensor, pos_ohot: Tensor, lengths: Sequence[int]) -> Tensor:
    """TextEncoderBiGRUCo: word_embs [B, L, dim_word], pos_ohot [B, L, dim_pos_ohot] -> [B, dim_coemb_hidden]."""
    w = {k: v.to(word_embs) for k, v in sd.items()}
    x = word_embs + (pos_ohot.to(word_embs) @ w["pos_emb.weight"].T + w["pos_emb.bias"])
    e = x @ w["input_emb.weight"].T + w["input_emb.bias"]
    return _bigru_head(w, e, [int(n) for n in lengths])


class TorchNets:
    """The same three networks built from torch.nn layers (Conv1d, Linear, GRU through pack_padded_sequence,
    LayerNorm), run eagerly in the dtype / on the device they are moved to: the fp32 yardstick the tests and
    scripts/bench_t2m.py compare the native path with."""

    def __init__(self, sds: Dict[str, Dict[str, Tensor]], device="cpu", dtype=torch.float32):
        nn = torch.nn

        def lin(w, b):
            m = nn.Linear(w.shape[1], w.shape[0])
            m.weight.data.copy_(w); m.bias.data.copy_(b)
            return m

        def conv(w, b):
            m = nn.Conv1d(w.shape[1], w.shape[0], 4, 2, 1)
            m.weight.data.copy_(w); m.bias.data.copy_(b)
            return m

        def bigru(sd):
            H = sd["hidden"].shape[-1]
            g = nn.GRU(sd["gru.weight_ih_l0"].shape[1], H, batch_first=True, bidirectional=True)
            g.load_state_dict({k[4:]: v for k, v in sd.items() if k.startswith("gru.")})
            ln = nn.LayerNorm(H)
            ln.weight.data.copy_(sd["output_net.1.weight"]); ln.bias.data.copy_(sd["output_net.1.bias"])
            head = nn.Sequential(lin(sd["output_net.0.weight"], sd["output_net.0.bias"]), ln, nn.LeakyReLU(0.2),
                                 lin(sd["output_net.3.weight"], sd["output_net.3.bias"]))
            return nn.ModuleDict({"gru": g, "head": head})

        t, v, m = sds["text_encoder"], sds["movement_encoder"], sds["motion_encoder"]
        self.mods = nn.ModuleDict({
            "pos_emb": lin(t["pos_emb.weight"], t["pos_emb.bias"]), "text_in": lin(t["input_emb.weight"], t["input_emb.bias"]),
            "text": bigru(t),
            "move": nn.Sequential(conv(v["main.0.weight"], v["main.0.bias"]), nn.LeakyReLU(0.2),
                                  conv(v["main.3.weight"], v["main.3.bias"]), nn.LeakyReLU(0.2)),
            "move_out": lin(v["out_net.weight"], v["out_net.bias"]),
            "motion_in": lin(m["input_emb.weight"], m["input_emb.bias"]), "motion": bigru(m),
        }).to(device=device, dtype=dtype).eval()
        self.h0 = {"text": t["hidden"].to(device=device, dtype=dtype), "motion": m["hidden"].to(device=device, dtype=dtype)}

    def _bigru(self, name, x, lengths):
        from torch.nn.utils.rnn import pack_padded_sequence
        packed = pack_padded_sequence(x, torch.as_tensor(lengths).cpu(), batch_first=True, enforce_sorted=False)
        _, last = self.mods[name]["gru"](packed, self.h0[name].expand(2, x.shape[0], -1).contiguous())
        return self.mods[name]["head"](torch.cat([last[0], last[1]], -1))

    def movement(self, x):
        return self.mods["move_out"](self.mods["move"](x.permute(0, 2, 1)).permute(0, 2, 1))

    def motion(self, x, lengths):
        return self._bigru("motion", self.mods["motion_in"](x), lengths)

    def text(self, word_embs, pos_ohot, lengths):
        return self._bigru("text", self.mods["text_in"](word_embs + self.mods["pos_emb"](pos_ohot)), lengths)
