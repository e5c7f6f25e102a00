"""A torch restatement of the library's split16 number format, for the accuracy tests.

Activations are stored unscaled as two fp16 planes, hi = fp16(x) and lo = fp16(x - hi) (``split_f32``,
mld_b200/csrc/common.cuh).  Weights are packed the same way after a power-of-two scale 2^s, s = floor(log2(2^14 / max|w|))
clamped to [-14, 14], that puts the largest |w| in (2^13, 2^14] where the clamp allows (``pack_linear``,
mld_b200/csrc/engine.cu).  The wgmma GEMM sums the three products
A_hi W_hi + A_lo W_hi + A_hi W_lo; here they are summed in float64, so ``emul_gemm`` carries the error of the
format alone, without the fp32 accumulator's."""
import math

import torch


def split_f32(x: torch.Tensor):
    """fp32 -> (hi, lo) fp16 planes, both rounded to nearest even as __float2half_rn does."""
    x = x.float()
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi, lo


def join(hi: torch.Tensor, lo: torch.Tensor) -> torch.Tensor:
    return hi.double() + lo.double()


def weight_scale_log2(W: torch.Tensor) -> int:
    mx = float(W.abs().max())
    if mx == 0.0:
        return 0
    return max(-14, min(14, math.floor(math.log2(16384.0 / mx))))


def pack_linear(W: torch.Tensor):
    """[N, K] fp32 weights -> (hi, lo, s): the planes of W * 2^s."""
    s = weight_scale_log2(W)
    hi, lo = split_f32(W.float() * 2.0 ** s)
    return hi, lo, s


def emul_gemm(A: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """A W^T through the split16 format, the three products summed in float64."""
    ah, al = split_f32(A)
    wh, wl, s = pack_linear(W)
    d = lambda t: t.double()
    return (d(ah) @ d(wh).T + d(al) @ d(wh).T + d(ah) @ d(wl).T) * 2.0 ** -s


def rel(a: torch.Tensor, ref: torch.Tensor) -> float:
    """Worst absolute error relative to the reference's largest magnitude."""
    a, ref = a.double().cpu(), ref.double().cpu()
    return float((a - ref).abs().max() / ref.abs().max())
