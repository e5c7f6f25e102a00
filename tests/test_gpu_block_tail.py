"""GPU: the encoder layer's tail (out-projection + residual + LayerNorm1, then the FFN block + LayerNorm2) as one
fused launch (k_ffn_tc with its out-projection prefix) against float64, against the two-kernel wgmma path and the
CUDA-core path, through mldb_debug_tail; and the denoiser's encoder layers running it."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

D = 256
SMS = 132          # H100 SXM: a persistent round of the fused kernel


@pytest.fixture(scope="module")
def eng(built_lib):
    from mld_b200.engine import Engine, make_config
    return Engine(make_config(num_layers=0, vae="none"), 0)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _params(seed, ff=1024):
    g = torch.Generator().manual_seed(seed)
    Wo, bo = torch.randn(D, D, generator=g) / D ** 0.5, 0.1 * torch.randn(D, generator=g)
    g1, be1 = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    W1, b1 = torch.randn(ff, D, generator=g) / D ** 0.5, 0.1 * torch.randn(ff, generator=g)
    W2, b2 = torch.randn(D, ff, generator=g) / ff ** 0.5, 0.1 * torch.randn(D, generator=g)
    g2, be2 = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    return Wo, bo, g1, be1, W1, b1, W2, b2, g2, be2


def _inputs(M, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(M, D, generator=g).cuda(), torch.randn(M, D, generator=g).cuda()


def _ref(att, X, Wo, bo, g1, be1, W1, b1, W2, b2, g2, be2):
    dd = lambda t: t.double().cpu()
    x1 = F.layer_norm(F.linear(dd(att), dd(Wo), dd(bo)) + dd(X), (D,), dd(g1), dd(be1), 1e-5)
    hid = F.gelu(F.linear(x1, dd(W1), dd(b1)))
    return F.layer_norm(x1 + F.linear(hid, dd(W2), dd(b2)), (D,), dd(g2), dd(be2), 1e-5)


# M < 128; a ragged M; several rounds of the persistent grid plus a leftover round cut along the hidden dimension
# (2 x 132 whole tiles + 20 tiles in 6 pieces); a leftover round of 26 tiles in 5 pieces (the headline's shape)
SIZES = [(77, 1024), (128 * 3 + 5, 1024), (SMS * 128 * 2 + 20 * 128 - 3, 1024), (26 * 128 - 50, 1024), (1000, 512)]


@pytest.mark.parametrize("M,ff", SIZES)
def test_tail_modes_against_float64(eng, M, ff):
    p = _params(M + ff, ff)
    att, X = _inputs(M, M)
    ref = _ref(att, X, *p)
    ys = [eng.debug_tail(att, X, *p, mode=m).cpu() for m in (0, 1, 2)]
    for name, y in zip(("cuda-core", "two wgmma kernels", "fused"), ys):
        assert torch.isfinite(y).all(), name
        assert _rel(y, ref) < 5e-6, name
    # the fused launch computes x1 with the out-projection GEMM's k-block order and LayerNorm, and the FFN as the
    # standalone fused kernel does: the same bits
    assert torch.equal(ys[2], ys[1])
    assert torch.equal(eng.debug_tail(att, X, *p, mode=2).cpu(), ys[2]), "repeated launch"


@pytest.mark.parametrize("M", [SMS * 128 * 2 + 20 * 128 - 3, 26 * 128 - 50])
def test_tail_split_off_matches(eng, M):
    """Without the hidden-dimension split of the leftover tiles both wgmma paths still agree bit for bit."""
    p = _params(M)
    att, X = _inputs(M, M + 1)
    eng.set_option("ffn_split", "0")
    try:
        y1 = eng.debug_tail(att, X, *p, mode=1).cpu()
        y2 = eng.debug_tail(att, X, *p, mode=2).cpu()
    finally:
        eng.set_option("ffn_split", "1")
    assert torch.equal(y2, y1)
    assert _rel(y2, _ref(att, X, *p)) < 5e-6


@pytest.mark.parametrize("M", [77, 128 * 3 + 5, 26 * 128 - 50])
def test_tail_leaves_padding_rows(eng, M):
    """The fused launch writes its output through TMA stores clipped at row M: rows past M keep their values."""
    p = _params(M)
    att, X = _inputs(M, M + 2)
    P = (M + 127) // 128 * 128 - M + 64
    pad = torch.full((P, D), 12345.0)
    pad[::3] = -3.0
    for mode in (1, 2):
        y = eng.debug_tail(att, X, *p, mode=mode, pad=pad).cpu()
        assert torch.equal(y[M:], pad), f"mode {mode}"
        assert _rel(y[:M], _ref(att, X, *p)) < 5e-6


@pytest.mark.parametrize("M", [1000, SMS * 128 * 2 + 20 * 128 - 3])
@pytest.mark.parametrize("which", ["att", "x"])
def test_tail_nan_stays_in_its_rows(eng, M, which):
    """A NaN in some rows of the attention output or of the layer input reaches no other row."""
    p = _params(M)
    att, X = _inputs(M, M + 3)
    clean = eng.debug_tail(att, X, *p, mode=2).cpu()
    for r0, r1 in [(0, 40), (M // 2 - 7, M // 2 + 70), (M - 50, M)]:
        a, x = att.clone(), X.clone()
        (a if which == "att" else x)[r0:r1] = float("nan")
        y = eng.debug_tail(a, x, *p, mode=2).cpu()
        assert torch.isnan(y[r0:r1]).all()
        keep = torch.ones(M, dtype=torch.bool)
        keep[r0:r1] = False
        assert torch.equal(y[keep], clean[keep]), (r0, r1)


def test_denoiser_encoder_layers_run_fused(built_lib):
    """At one prompt (2 m-tiles, where the fused launch is the faster one) the denoiser's encoder layers enqueue the
    fused tail, not the out-projection LayerNorm GEMM (which the MldVae decoder's layers still use)."""
    from mld_b200 import synth
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(vae="none"), 0)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.finalize()
    Bx = 2
    ctx, x = synth.text_context(Bx // 2, 77, seed=11).cuda(), synth.init_noise(Bx, seed=12).cuda()
    eng.kernel_stats(reset=True)
    y = eng.denoise(x, 501, ctx, [196, 100])
    torch.cuda.synchronize()
    st = eng.kernel_stats()
    assert torch.isfinite(y).all()
    assert st["gemm_ln_tc"] == 0 and st["ln_unfused"] == 0, st
    assert st["ffn_tc"] > 0, st
