"""Float64 restatement of the UESTC action classifier (TEST INFRASTRUCTURE).

``STGCN`` as MLD's ``UESTCMetrics`` uses it (layout "smpl", strategy "spatial", edge importance weighting), written
from the network's definition: data_bn over channel ``v * C + c``; ten st_gcn blocks, each
    gcn:  a 1 x 1 conv to 3 C_out channels, then x[n, c, t, w] = sum_k sum_v y[n, k, c, t, v] A'_k[v, w]
    tcn:  BatchNorm, ReLU, a (9, 1) conv (padding 4, stride s), BatchNorm
    out:  ReLU(tcn + residual), the residual none (block 0), identity, or a 1 x 1 stride-s conv + BatchNorm
with A'_i = A * edge_importance[i] (in fp32, as the reference forms it); then the mean over (T_out, 24) and a 1 x 1
conv head.  Every BatchNorm is applied unfolded, (x - mean) / sqrt(var + 1e-5) * weight + bias, so a comparison
against this checks the engine's folding.  Plain tensor arithmetic in whatever dtype the input has.

``TorchSTGCN`` is the same network built from ``torch.nn`` layers (fp32 eager, cuDNN convolutions on a GPU), with the
reference's key names: the benchmark's yardstick and the fp32 comparison printed beside the native path's errors.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F
from torch import nn

Tensor = torch.Tensor
CHANNELS = (64, 64, 64, 64, 128, 128, 128, 256, 256, 256)
STRIDES = (1, 1, 1, 1, 2, 1, 1, 2, 1, 1)


def _bn(w: Dict[str, Tensor], p: str, x: Tensor) -> Tensor:
    """Eval-mode BatchNorm over dim 1 of x."""
    shape = (1, -1) + (1,) * (x.dim() - 2)
    m, v = w[p + "running_mean"].reshape(shape), w[p + "running_var"].reshape(shape)
    return (x - m) / torch.sqrt(v + 1e-5) * w[p + "weight"].reshape(shape) + w[p + "bias"].reshape(shape)


def classify(sd: Dict[str, Tensor], motion: Tensor) -> Tuple[Tensor, Tensor]:
    """motion [N, 24, C, T] -> (yhat [N, num_class], features [N, 256]) in motion's dtype."""
    dt = motion.dtype
    w = {k: v.to(device=motion.device, dtype=dt) for k, v in sd.items() if v.is_floating_point()}
    N, V, C, T = motion.shape
    x = _bn(w, "data_bn.", motion.reshape(N, V * C, T)).reshape(N, V, C, T).permute(0, 2, 3, 1)   # [N, C, T, V]
    for i, co in enumerate(CHANNELS):
        p, s = f"st_gcn_networks.{i}.", STRIDES[i]
        A = (sd["A"].float() * sd[f"edge_importance.{i}"].float()).to(device=motion.device, dtype=dt)
        if i == 0:
            res = 0.0
        elif x.shape[1] == co and s == 1:
            res = x
        else:
            r = torch.einsum("oc,nctv->notv", w[p + "residual.0.weight"][:, :, 0, 0], x[:, :, ::s])
            res = _bn(w, p + "residual.1.", r + w[p + "residual.0.bias"].reshape(1, -1, 1, 1))
        y = torch.einsum("oc,nctv->notv", w[p + "gcn.conv.weight"][:, :, 0, 0], x) + w[p + "gcn.conv.bias"].reshape(1, -1, 1, 1)
        y = torch.einsum("nkctv,kvw->nctw", y.reshape(N, 3, co, y.shape[2], V), A)
        y = torch.relu(_bn(w, p + "tcn.0.", y))
        y = F.conv2d(y, w[p + "tcn.2.weight"], w[p + "tcn.2.bias"], stride=(s, 1), padding=(4, 0))
        x = torch.relu(_bn(w, p + "tcn.3.", y) + res)
    features = x.mean(dim=(2, 3))
    yhat = features @ w["fcn.weight"][:, :, 0, 0].t() + w["fcn.bias"]
    return yhat, features


class _Block(nn.Module):
    def __init__(self, cin: int, co: int, stride: int, residual: bool):
        super().__init__()
        self.gcn = nn.Module()
        self.gcn.conv = nn.Conv2d(cin, 3 * co, 1)
        self.tcn = nn.Sequential(nn.BatchNorm2d(co), nn.ReLU(), nn.Conv2d(co, co, (9, 1), (stride, 1), (4, 0)),
                                 nn.BatchNorm2d(co), nn.Dropout(0.0))
        self.kind = "none" if not residual else ("identity" if cin == co and stride == 1 else "conv")
        if self.kind == "conv":
            self.residual = nn.Sequential(nn.Conv2d(cin, co, 1, (stride, 1)), nn.BatchNorm2d(co))

    def forward(self, x: Tensor, A: Tensor) -> Tensor:
        res = 0.0 if self.kind == "none" else (x if self.kind == "identity" else self.residual(x))
        y = self.gcn.conv(x)
        n, kc, t, v = y.shape
        y = torch.einsum("nkctv,kvw->nctw", y.view(n, 3, kc // 3, t, v), A)
        return torch.relu(self.tcn(y) + res)


class TorchSTGCN(nn.Module):
    """The classifier from ``torch.nn`` layers, keys as the reference's ``STGCN``; forward(motion [N, 24, C, T]) ->
    (yhat, features)."""

    def __init__(self, in_channels: int = 6, num_class: int = 40):
        super().__init__()
        self.register_buffer("A", torch.zeros(3, 24, 24))
        self.data_bn = nn.BatchNorm1d(in_channels * 24)
        cins = (in_channels,) + CHANNELS[:-1]
        self.st_gcn_networks = nn.ModuleList(_Block(ci, co, s, i > 0)
                                             for i, (ci, co, s) in enumerate(zip(cins, CHANNELS, STRIDES)))
        self.edge_importance = nn.ParameterList(nn.Parameter(torch.ones(3, 24, 24)) for _ in CHANNELS)
        self.fcn = nn.Conv2d(256, num_class, 1)

    def forward(self, motion: Tensor) -> Tuple[Tensor, Tensor]:
        N, V, C, T = motion.shape
        x = self.data_bn(motion.reshape(N, V * C, T)).view(N, V, C, T).permute(0, 2, 3, 1).contiguous()
        for blk, imp in zip(self.st_gcn_networks, self.edge_importance):
            x = blk(x, self.A * imp)
        f = F.avg_pool2d(x, x.shape[2:])
        return self.fcn(f).view(N, -1), f.view(N, -1)
