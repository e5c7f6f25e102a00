"""The split16 number format's envelope, on the CPU (tests/split16_ref.py restates it in torch).

hi + lo carries ~22 significant bits only for 2^-3 <= |x| < 65520.  Below 2^-3 the lo plane is an fp16 subnormal,
so the error has an absolute floor of 2^-25 instead of a relative bound; from 65520 up hi is inf.  Activations are
stored without a scale, so a GEMM on small activations loses accuracy by the same floor; weights get a power-of-two
scale and keep the ~22 bits.  These numbers are what the GPU accuracy tests (tests/test_gpu_value_ranges.py) hold
the kernels to outside the envelope."""
import pytest
import torch

from split16_ref import emul_gemm, join, pack_linear, rel, split_f32


def _values(lo_exp, hi_exp, n=200_000, seed=0):
    """Magnitudes log-uniform in [2^lo_exp, 2^hi_exp), both signs."""
    g = torch.Generator().manual_seed(seed)
    e = lo_exp + (hi_exp - lo_exp) * torch.rand(n, generator=g, dtype=torch.float64)
    s = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()
    return (s * torch.exp2(e)).float()


def test_roundtrip_relative_inside_envelope():
    x = torch.cat([_values(-3, 15.999), torch.tensor([0.125, -0.125, 65504.0, 65519.0, -65519.0, 1.0 + 2 ** -23])])
    x = x[x.abs() < 65520]
    err = (join(*split_f32(x)) - x.double()).abs() / x.double().abs()
    assert float(err.max()) <= 2.0 ** -22
    assert float(err.max()) > 2.0 ** -24          # and the bound is tight: not a wider format in disguise


def test_roundtrip_absolute_floor_below_envelope():
    x = torch.cat([_values(-40, -3), torch.tensor([2 ** -14, 2 ** -24, 2 ** -25, 2 ** -26, 3e-8, 0.0])])
    err = (join(*split_f32(x)) - x.double()).abs()
    assert float(err.max()) <= 2.0 ** -25
    small = x.abs() < 2 ** -6
    rel_err = err[small] / x[small].double().abs().clamp_min(1e-300)
    assert float(rel_err.max()) > 2.0 ** -22 * 8   # the relative bound no longer holds there


def test_inf_from_65520():
    x = torch.tensor([65520.0, -65520.0, 65536.0, 1e5, 3e38])
    hi, lo = split_f32(x)
    assert torch.isinf(hi).all() and (hi.float().sign() == x.sign()).all()
    assert torch.isfinite(split_f32(torch.tensor([65519.996, 65504.0]))[0]).all()


def test_weight_scale():
    """pack_linear's 2^s puts max |w| in (2^13, 2^14] unless the clamp to [-14, 14] binds; every packed weight of
    magnitude 2^-3 or more (after the scale) keeps the relative bound."""
    g = torch.Generator().manual_seed(1)
    for scale in (1e-4, 1e-2, 1.0, 30.0, 1e4, 1e7):
        W = torch.randn(64, 256, generator=g) * scale
        hi, lo, s = pack_linear(W)
        assert (s == 14) == (scale < 0.1)          # the shipped 1/sqrt(K)-scale weights sit at the clamp
        if -14 < s < 14:
            assert 2 ** 13 < float(hi.float().abs().max()) <= 2 ** 14
        back = join(hi, lo) * 2.0 ** -s
        ok = W.abs() * 2.0 ** s >= 2 ** -3
        assert float(((back - W.double()).abs()[ok] / W.double().abs()[ok]).max()) <= 2.0 ** -22


# relative-to-max error of the emulated GEMM (M = N = 256, K = 1024, unit-std A times 1/sqrt(K) weights) scaled by 2^e
EMUL_GEMM = {12: 8.5e-8, 8: 8.5e-8, 4: 8.5e-8, 0: 8.6e-8, -3: 1.5e-7, -6: 1.07e-6, -10: 1.70e-5, -12: 7.8e-5,
             -14: 2.83e-4}


def _gemm_data(M=256, K=1024, N=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / K ** 0.5


@pytest.mark.parametrize("e", sorted(EMUL_GEMM))
def test_emulated_gemm_error_against_scale(e):
    """The split format alone, with a float64 accumulator: scale-free down to 2^-3, then growing about 4x per
    two octaves (the 2^-25 floor of each element against a shrinking output)."""
    A0, W = _gemm_data()
    A = A0 * 2.0 ** e
    ref = (A0.double() @ W.double().T) * 2.0 ** e
    err = rel(emul_gemm(A, W), ref)
    assert EMUL_GEMM[e] / 1.1 < err < EMUL_GEMM[e] * 1.1, f"2^{e}: {err:.3e}"
    # fp32 torch on the same data does not depend on the scale, but its value does depend on how the CPU BLAS orders
    # its sums (2.7e-7 to 5.7e-7 across MKL's code paths), so it is not pinned.  Split16 beats it only inside the
    # envelope: 1.5e-7 at 2^-3, 1.07e-6 at 2^-6.
    f32 = rel(A @ W.T, ref)
    assert (err < f32) == (e >= -3), f"2^{e}: split16 {err:.3e}, fp32 {f32:.3e}"
