"""GPU: every kernel that applies a packed weight's scale, at split16 weight exponents other than 14 (pytest -m gpu).

Each weight is packed as the planes of W * 2^s with its own s (``pack_linear``), and each kernel multiplies its
accumulator by that weight's 2^-s.  Weights of the usual 1/sqrt(K) size all sit at the s = 14 clamp, so these
tests build weights at chosen exponents (tests/weight_scales.py) and check, against float64: the wgmma GEMM's
fp32, residual-add, split16 and LayerNorm epilogues, the CUDA-core GEMM, the K = 256 projection kernel, and the
fused FFN and fused layer tail with a different exponent on each of their two or three weights.  Also: an exact
power-of-two equivariance, an all-zero weight, single large outliers, and inf / NaN weight elements, which poison
their own output column and nothing else.

Gate: 5e-6 relative to the max, scaled with K above 1024 (``_tc_tol``), as the other kernel tests."""
import itertools

import pytest
import torch
import torch.nn.functional as F

from weight_scales import engine_exponent, weight_at

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

D = 256
SMS = 132                                           # H100 SXM: a persistent round of the fused kernels
SWEEP = [-2, 0, 5, 9, 12, 13, 14, None]             # None: max|w| = 0.1, clamped to 14
SPLIT_SWEEP = [9, 10, 11, 12, 13, 14]               # split16 outputs: smaller s pushes |y| past 65520
ACTS = {0: lambda x: x, 2: F.relu, 5: lambda x: torch.where(x > 0, x, 0.2 * x)}     # NONE, RELU, LEAKY


@pytest.fixture(scope="module")
def eng(built_lib):
    from mld_b200.engine import Engine, make_config
    return Engine(make_config(num_layers=0, vae="none"), 0)


def _tc_tol(K):
    return 5e-6 * max(1.0, K / 1024)


def _rel(a, ref):
    a, ref = a.double().cpu(), ref.double().cpu()
    return float((a - ref).abs().max() / ref.abs().max())


def _err(group, y, ref):
    """The error against float64, printed per group (pytest -s) for the table in DESIGN.md section 1."""
    e = _rel(y, ref)
    print(f"[weight-scales] {group}: {e:.2e}")
    return e


def _weight(N, K, s, g):
    if s is None:
        W = torch.randn(N, K, generator=g)
        W = W * (0.1 / W.abs().max())
        assert engine_exponent(W) == 14
        return W
    return weight_at(N, K, s, g)


def _out_scale(W):
    """Typical |A W^T| for randn A: biases and residuals are drawn at this size, so they matter at every s."""
    return float(W.double().std()) * W.shape[1] ** 0.5


def _gemm_inputs(M, N, K, s, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    W = _weight(N, K, s, g)
    c = _out_scale(W)
    # R is an activation, stored as split16 without a scale: it has to stay below 65520
    return A.cuda(), W, 0.3 * c * torch.randn(N, generator=g), min(c, 2.0 ** 12) * torch.randn(M, N, generator=g)


def _sid(s):
    return "clamped" if s is None else f"s{s}"


# --------------------------------------------------------------------------------------- GEMM, exponent sweep
GEMM_CASES = [
    # M,   N,   K,    K1,  act, residual
    (200, 256, 256, 0, 0, False),
    (333, 512, 1024, 0, 2, False),
    (129, 256, 512, 256, 5, False),          # two A sources
    (392, 263, 256, 0, 0, False),            # ragged N
    (1100, 263, 512, 256, 2, False),         # ragged N, two sources, several m-tiles
    (515, 256, 512, 0, 0, True),             # residual-add epilogue
    (200, 768, 256, 128, 0, True),
]


@pytest.mark.parametrize("s", SWEEP, ids=_sid)
@pytest.mark.parametrize("M,N,K,K1,act,res", GEMM_CASES)
def test_gemm_f32_exponent_sweep(eng, M, N, K, K1, act, res, s):
    A, W, b, R = _gemm_inputs(M, N, K, s, M + N + K1 + (s or 99))
    ref = F.linear(A.double(), W.double().cuda(), b.double().cuda())
    ref = ref + R.double().cuda() if res else ACTS[act](ref)
    kw = dict(R=R) if res else {}
    for tc in (True, False):
        eng.kernel_stats(reset=True)
        y = eng.debug_gemm(A, W, b, K1=K1, act=0 if res else act, use_tc=tc, **kw)
        assert eng.kernel_stats()["gemm_tc" if tc else "gemm_simt"] == 1
        assert torch.isfinite(y).all(), tc
        e = _err(f"gemm f32 {'wgmma' if tc else 'cuda-core'} s={s}", y, ref)
        assert e < (_tc_tol(K) if tc else 5e-6), ("wgmma" if tc else "cuda-core", e)


@pytest.mark.parametrize("s", SPLIT_SWEEP, ids=_sid)
@pytest.mark.parametrize("M,N,K,K1,act", [(200, 256, 256, 0, 0),          # k_proj_tc (K up to 512: DESIGN.md section 1)
                                          (333, 512, 512, 0, 2),          # k_gemm_tc fast epilogue
                                          (129, 256, 512, 256, 5),
                                          (1000, 768, 256, 128, 0)])
def test_gemm_split16_exponent_sweep(eng, M, N, K, K1, act, s):
    A, W, b, _ = _gemm_inputs(M, N, K, s, 3 * M + N + K1 + s)
    ref = ACTS[act](F.linear(A.double(), W.double().cuda(), b.double().cuda()))
    assert float(ref.abs().max()) < 65000
    y = eng.debug_gemm(A, W, b, K1=K1, act=act, split_out=True)
    assert torch.isfinite(y).all()
    e = _err(f"gemm split16 s={s}", y, ref)
    assert e < _tc_tol(K), e


@pytest.mark.parametrize("s", SWEEP, ids=_sid)
@pytest.mark.parametrize("M,N,K", [(333, 256, 1024), (640, 256, 256), (1300, 256, 512)])
def test_gemm_layernorm_exponent_sweep(eng, M, N, K, s):
    """The LayerNorm epilogue normalises its output, so it takes every exponent."""
    A, W, b, R = _gemm_inputs(M, N, K, s, 5 * M + K + (s or 99))
    g = torch.Generator().manual_seed(M)
    gamma, beta = 1 + 0.1 * torch.randn(N, generator=g), 0.1 * torch.randn(N, generator=g)
    pre = F.linear(A.double(), W.double().cuda(), b.double().cuda()) + R.double().cuda()
    ref = F.layer_norm(pre, (N,), gamma.double().cuda(), beta.double().cuda(), 1e-5)
    for tc in (True, False):
        eng.kernel_stats(reset=True)
        y = eng.debug_gemm(A, W, b, gamma=gamma, beta=beta, R=R, use_tc=tc)
        assert eng.kernel_stats()["gemm_ln_tc" if tc else "gemm_simt"] == 1
        assert torch.isfinite(y).all(), tc
        e = _err(f"gemm LN {'wgmma' if tc else 'cuda-core'} s={s}", y, ref)
        assert e < (_tc_tol(K) if tc else 5e-6), ("wgmma" if tc else "cuda-core", e)


# --------------------------------------------------------------------------------------- exact equivariance
@pytest.mark.parametrize("tc", [True, False], ids=["wgmma", "cuda-core"])
@pytest.mark.parametrize("act,res", [(0, False), (2, False), (5, False), (0, True)])
@pytest.mark.parametrize("M,N,K,K1", [(200, 256, 256, 0), (129, 263, 512, 256)])
def test_power_of_two_equivariance(eng, M, N, K, K1, act, res, tc):
    """Scaling W, b (and R) by 2^j moves the exponent by -j and leaves the packed planes as they were, so the output
    must be exactly 2^j times the original: the scale is applied once, as a power of two, before the bias."""
    A, W, b, R = _gemm_inputs(M, N, K, 12, M + K + act)
    kw = lambda j: dict(R=R * 2.0 ** j) if res else {}
    y0 = eng.debug_gemm(A, W, b, K1=K1, act=act, use_tc=tc, **kw(0)).clone()
    assert torch.isfinite(y0).all() and float(y0.abs().max()) > 0
    for j in (-2, 3, 10):                               # exponents 14, 9, 2: never clamped
        assert engine_exponent(W * 2.0 ** j) == 12 - j
        y = eng.debug_gemm(A, W * 2.0 ** j, b * 2.0 ** j, K1=K1, act=act, use_tc=tc, **kw(j))
        assert torch.equal(y, y0 * 2.0 ** j), j


# --------------------------------------------------------------------------------------- K = 256 projection
@pytest.mark.parametrize("s", [9, 11, 13], ids=_sid)
@pytest.mark.parametrize("N", [256, 768])
def test_proj_exponents(eng, N, s):
    """k_proj_tc (K = 256, one source, N a multiple of 128, split16 out) against float64, and bit for bit against
    the same product on k_gemm_tc from two A sources."""
    A, W, b, _ = _gemm_inputs(40448, N, 256, s, N + s)
    ref = F.linear(A.double(), W.double().cuda(), b.double().cuda())
    for M in (200, 40448):
        y = eng.debug_gemm(A[:M], W, b, split_out=True)
        assert torch.isfinite(y).all()
        e = _err(f"proj s={s}", y, ref[:M])
        assert e < _tc_tol(256), (M, e)
        assert torch.equal(eng.debug_gemm(A[:M], W, b, K1=128, split_out=True), y), M


# --------------------------------------------------------------------------------------- fused FFN and layer tail
def _ffn_params(ff, s1, s2, seed):
    g = torch.Generator().manual_seed(seed)
    W1, W2 = weight_at(ff, D, s1, g), weight_at(D, ff, s2, g)
    b1 = 0.3 * _out_scale(W1) * torch.randn(ff, generator=g)
    b2 = 0.3 * _out_scale(W2) * torch.randn(D, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    return W1, b1, W2, b2, gamma, beta


def _ffn_ref(X, W1, b1, W2, b2, gamma, beta):
    dd = lambda t: t.double().cuda()
    hid = F.gelu(F.linear(dd(X), dd(W1), dd(b1)))
    return F.layer_norm(dd(X) + F.linear(hid, dd(W2), dd(b2)), (D,), dd(gamma), dd(beta), 1e-5)


PERMS = list(itertools.permutations((13, 11, 9)))
SIZES = [77, 128 * 3 + 5, SMS * 128 * 2 + 20 * 128 - 3]      # < 1 tile; ragged; 2 rounds + 20 leftover tiles, split
FFN_EXPONENTS = sorted({p[1:] for p in PERMS}) + [(12, 12)]


@pytest.mark.parametrize("s1,s2", FFN_EXPONENTS)
@pytest.mark.parametrize("M", SIZES)
def test_ffn_exponents(eng, M, s1, s2):
    ff = 1024
    p = _ffn_params(ff, s1, s2, M + 10 * s1 + s2)
    X = torch.randn(M, D, generator=torch.Generator().manual_seed(M)).cuda()
    ref = _ffn_ref(X, *p)
    ys = [eng.debug_ffn(X, *p, mode=m) for m in (0, 1, 2)]
    for name, y in zip(("cuda-core", "tc unfused", "tc fused"), ys):
        assert torch.isfinite(y).all(), name
        e = _err(f"ffn {name}", y, ref)
        assert e < 5e-6, (name, e)
    assert _rel(ys[2], ys[1]) < 4e-6
    eng.set_option("ffn_split", "0")
    try:
        whole = eng.debug_ffn(X, *p, mode=2)
    finally:
        eng.set_option("ffn_split", "1")
    assert _rel(whole, ref) < 5e-6


def _tail_params(ff, s0, s1, s2, seed):
    g = torch.Generator().manual_seed(seed)
    Wo = weight_at(D, D, s0, g)
    bo = 0.3 * _out_scale(Wo) * torch.randn(D, generator=g)
    g1, be1 = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    return (Wo, bo, g1, be1) + _ffn_params(ff, s1, s2, seed + 1)


def _tail_ref(att, X, Wo, bo, g1, be1, *ffn):
    dd = lambda t: t.double().cuda()
    x1 = F.layer_norm(F.linear(dd(att), dd(Wo), dd(bo)) + dd(X), (D,), dd(g1), dd(be1), 1e-5)
    return _ffn_ref(x1, *ffn)


@pytest.mark.parametrize("s0,s1,s2", PERMS)
@pytest.mark.parametrize("M", SIZES)
def test_tail_exponents(eng, M, s0, s1, s2):
    """The fused tail applies three scales in one launch: W_o's to the out-projection prefix, W1's and W2's in the
    FFN.  The fused launch must give the two-kernel path's bits, with and without the hidden-dimension split."""
    ff = 1024
    p = _tail_params(ff, s0, s1, s2, M + 100 * s0 + 10 * s1 + s2)
    g = torch.Generator().manual_seed(M + 1)
    att = torch.randn(M, D, generator=g).cuda()
    X = (_out_scale(p[0]) * torch.randn(M, D, generator=g)).cuda()          # the size of att W_o^T
    ref = _tail_ref(att, X, *p)
    ys = [eng.debug_tail(att, X, *p, mode=m) for m in (0, 1, 2)]
    for name, y in zip(("cuda-core", "two wgmma kernels", "fused"), ys):
        assert torch.isfinite(y).all(), name
        e = _err(f"tail {name}", y, ref)
        assert e < 5e-6, (name, e)
    assert torch.equal(ys[2], ys[1])
    eng.set_option("ffn_split", "0")
    try:
        y1, y2 = eng.debug_tail(att, X, *p, mode=1), eng.debug_tail(att, X, *p, mode=2)
    finally:
        eng.set_option("ffn_split", "1")
    assert torch.equal(y2, y1)
    assert _rel(y2, ref) < 5e-6


# --------------------------------------------------------------------------------------- zero weight
def test_zero_weight(eng):
    """An all-zero W packs at s = 0 (scale 1): the GEMM returns its bias exactly, and an FFN with W2 = 0 is
    LayerNorm(x + b2)."""
    g = torch.Generator().manual_seed(3)
    A, b = torch.randn(300, 512, generator=g).cuda(), torch.randn(263, generator=g)
    for tc in (True, False):
        y = eng.debug_gemm(A, torch.zeros(263, 512), b, use_tc=tc)
        assert torch.equal(y.cpu(), b.expand(300, 263)), tc
    M, ff = 389, 1024
    W1, b1, _, b2, gamma, beta = _ffn_params(ff, 13, 13, 4)
    X = torch.randn(M, D, generator=g).cuda()
    ref = F.layer_norm(X.double() + b2.double().cuda(), (D,), gamma.double().cuda(), beta.double().cuda(), 1e-5)
    for mode in (0, 1, 2):
        y = eng.debug_ffn(X, W1, b1, torch.zeros(D, ff), b2, gamma, beta, mode=mode)
        assert _rel(y, ref) < 5e-6, mode


# --------------------------------------------------------------------------------------- outliers
def _rel_cols(y, ref):
    """Worst error of each output column relative to that column's largest magnitude."""
    y, ref = y.double().cpu(), ref.double().cpu()
    return ((y - ref).abs().max(0).values / ref.abs().max(0).values).max().item()


def _outlier_weight(N, K, ratio, n0, k0, seed):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    W[n0, k0] = ratio * float(W.abs().max())
    return W


@pytest.mark.parametrize("ratio", [2 ** 8, 2 ** 12, 2 ** 16, 2 ** 20])
@pytest.mark.parametrize("M,N,K,K1", [(300, 256, 256, 0), (257, 263, 512, 256)])
def test_outlier_element(eng, M, N, K, K1, ratio):
    """The bulk randn / sqrt(K), one element `ratio` times larger: the scale follows the outlier and the bulk moves
    towards the bottom of fp16's range.  Every column is gated against its own max, so the outlier's column does
    not hide the others.  Elements of at least 2^-3 after the scale keep 22 bits; the gate holds to 2^16, and the
    error at 2^20 is printed (DESIGN.md section 1), not gated.  K stays at 512: at K = 1024 the fp32 accumulator
    alone takes the smallest of 263 columns past 5e-6, whatever the ratio."""
    W = _outlier_weight(N, K, ratio, N // 3, K // 2, ratio + N)
    A = torch.randn(M, K, generator=torch.Generator().manual_seed(M)).cuda()
    b = 0.1 * torch.randn(N, generator=torch.Generator().manual_seed(N))
    ref = F.linear(A.double(), W.double().cuda(), b.double().cuda())
    for tc in (True, False):
        y = eng.debug_gemm(A, W, b, K1=K1, use_tc=tc)
        err = _rel_cols(y, ref)
        print(f"outlier 2^{ratio.bit_length() - 1} {'wgmma' if tc else 'cuda-core'} K={K} s={engine_exponent(W)}: "
              f"{err:.2e} per column")
        assert torch.isfinite(y).all()
        if ratio <= 2 ** 16:
            assert err < (_tc_tol(K) if tc else 5e-6), (tc, err)


# --------------------------------------------------------------------------------------- non-finite elements
@pytest.mark.parametrize("bad", [float("inf"), float("nan")], ids=["inf", "nan"])
@pytest.mark.parametrize("path", ["wgmma", "cuda-core", "proj"])
def test_nonfinite_weight_element(eng, path, bad):
    """An inf or NaN in W[n0, k0] makes column n0 non-finite, as in torch, and leaves every other column at the
    gate: the scale is taken over the finite elements."""
    M, N, K, n0, k0 = 300, 256, 256, 77, 100
    g = torch.Generator().manual_seed(11)
    A = torch.randn(M, K, generator=g).cuda()
    W, b = torch.randn(N, K, generator=g) / K ** 0.5, 0.1 * torch.randn(N, generator=g)
    ref = F.linear(A.double(), W.double().cuda(), b.double().cuda())
    W[n0, k0] = bad
    kw = {"wgmma": dict(K1=128), "cuda-core": dict(use_tc=False), "proj": dict(split_out=True)}[path]
    y = eng.debug_gemm(A, W, b, **kw).cpu()
    assert not torch.isfinite(y[:, n0]).any()
    keep = torch.arange(N) != n0
    assert torch.isfinite(y[:, keep]).all()
    assert _rel(y[:, keep], ref[:, keep]) < 5e-6, _rel(y[:, keep], ref[:, keep])
