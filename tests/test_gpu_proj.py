"""GPU tests of the K = 256 projection kernel k_proj_tc (pytest -m gpu), through the C ABI's debug hook with the
split16 output that the sampling path uses.  op_gemm sends a fast-epilogue GEMM with K = 256 from one A source and
N a multiple of 128 to k_proj_tc; the same product with K split over two A sources runs on k_gemm_tc with the same
per-element accumulation order, so the two must agree bit for bit."""
import pytest
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

K = 256
MS = (1, 127, 129, 200, 40448)                 # 40 448 = the benchmark's rows per encoder layer (2 x 256 x 79)
ACTS = {0: lambda x: x, 1: F.gelu, 4: lambda x: x * torch.sigmoid(1.702 * x),
        5: lambda x: torch.where(x > 0, x, 0.2 * x)}          # NONE, GELU, QUICKGELU, LEAKY


@pytest.fixture(scope="module")
def eng(built_lib):
    from mld_b200.engine import Engine, make_config
    return Engine(make_config(num_layers=0, vae="none"), 0)


def _tc_tol(K):
    return 5e-6 * max(1.0, K / 1024)


def _rel(a, b):
    return float((a.double() - b).abs().max() / b.abs().max())


def _kernels(fn):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("N", [128, 256, 512, 768, 1024])
def test_proj_accuracy_and_bit_identity(eng, N, act):
    g = torch.Generator().manual_seed(N * 10 + act)
    A = torch.randn(max(MS), K, generator=g).cuda()
    W = torch.randn(N, K, generator=g) / K ** 0.5
    b = 0.1 * torch.randn(N, generator=g)
    ref = ACTS[act](F.linear(A.double(), W.double().cuda(), b.double().cuda()))
    big = None
    for M in MS:
        y = eng.debug_gemm(A[:M], W, b, act=act, split_out=True)
        assert torch.isfinite(y).all()
        assert _rel(y, ref[:M]) < _tc_tol(K), M
        assert torch.equal(eng.debug_gemm(A[:M], W, b, act=act, split_out=True), y), M           # repeatable
        # k_gemm_tc: the same k-blocks from two A sources
        assert torch.equal(eng.debug_gemm(A[:M], W, b, K1=128, act=act, split_out=True), y), M
        if M == max(MS):
            big = y
    # a row's result does not depend on its m-tile, its place in the tile or the CTA range that computed it
    for r0, M in ((0, 129), (64, 129), (40000, 200), (12345, 1)):
        assert torch.equal(eng.debug_gemm(A[r0:r0 + M], W, b, act=act, split_out=True), big[r0:r0 + M]), (r0, M)


def test_proj_kernel_choice(eng):
    g = torch.Generator().manual_seed(7)
    A = torch.randn(200, 512, generator=g).cuda()
    W, b = torch.randn(768, 512, generator=g) / 16, torch.randn(768, generator=g)
    names = _kernels(lambda: eng.debug_gemm(A[:, :K], W[:, :K], b, split_out=True))
    assert any("k_proj_tc" in n for n in names) and not any("k_gemm_tc" in n for n in names), names
    for kw in (dict(A=A, W=W), dict(A=A[:, :K], W=W[:263, :K])):          # K = 512; N = 263 (not a multiple of 128)
        names = _kernels(lambda: eng.debug_gemm(kw["A"], kw["W"], b[:kw["W"].shape[0]], split_out=True))
        assert any("k_gemm_tc" in n for n in names) and not any("k_proj_tc" in n for n in names), (kw["W"].shape, names)
