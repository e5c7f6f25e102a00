"""GPU tests of the native UESTC action classifier (pytest -m gpu): the reference fixture, float64 accuracy over batch
and length (fp32 torch with TF32 off printed beside it), the predicted class, the CUDA-core path, weight scales,
isolation and bit-identity under permutation and chunking, the kernel counts, the drop-in called as
UESTCMetrics.update calls it, and the refusals."""
import pytest
import torch

from conftest import golden
from mld_b200 import _lib, synth
from mld_b200.engine import Engine, make_config
from mld_b200.evaluator import B200STGCN
from oracle import uestc_stgcn as O
from oracle.make_golden_uestc import CASES, WEIGHT_SEED, write_kintree

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
GATE, FIXTURE_GATE = 1e-4, 2e-4
PREFIX = "stgcn_classifier."
GRAPH = {"layout": "smpl", "strategy": "spatial"}


def _rel_rows(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float(((a - b).abs().max(1).values / b.abs().max(1).values).max())


def _engine(sd, simt=False):
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    if simt:
        eng.set_option("gemm", "simt")
    eng.stgcn_configure(_lib.default_stgcn_config())
    eng.load_state_dict(sd, PREFIX)
    eng.finalize()
    return eng


def _f64(sd, x):
    return O.classify({k: v.cuda() for k, v in sd.items()}, x.double())


@pytest.fixture(scope="module", autouse=True)
def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.fixture(scope="module")
def sd():
    return synth.stgcn_state_dict(WEIGHT_SEED)


@pytest.fixture(scope="module")
def eng(built_lib, sd):
    return _engine(sd)


@pytest.fixture(scope="module")
def torch_net(sd):
    net = O.TorchSTGCN().cuda().eval()
    net.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=True)
    return net


@pytest.mark.parametrize("B,T,seed", CASES)
def test_reference_fixture(eng, B, T, seed):
    g = golden("uestc_stgcn.npz")
    yhat, feats = eng.stgcn_classify(synth.uestc_motions(B, T, seed=seed).cuda())
    ey, ef = _rel_rows(yhat, torch.from_numpy(g[f"yhat_{B}x{T}"])), _rel_rows(feats, torch.from_numpy(g[f"features_{B}x{T}"]))
    print(f"uestc fixture B={B} T={T}: yhat {ey:.2e} features {ef:.2e}")
    assert ey < FIXTURE_GATE and ef < FIXTURE_GATE


@pytest.mark.parametrize("T", [1, 2, 7, 8, 9, 60, 61, 200])
@pytest.mark.parametrize("B", [1, 5, 32, 300])
def test_float64(eng, sd, torch_net, B, T):
    x = synth.uestc_motions(B, T, seed=B * 7 + T).cuda()
    yhat, feats = eng.stgcn_classify(x)
    ry, rf = _f64(sd, x)
    ty, tf = torch_net(x)
    ey, ef = _rel_rows(yhat, ry), _rel_rows(feats, rf)
    print(f"uestc B={B} T={T}: yhat {ey:.2e} features {ef:.2e} (fp32 torch {_rel_rows(ty, ry):.2e} {_rel_rows(tf, rf):.2e})")
    assert ey < GATE and ef < GATE
    # the predicted class, wherever the float64 top-2 margin is clear
    top = ry.cpu().topk(2, dim=1).values
    clear = (top[:, 0] - top[:, 1]) > 1e-3 * ry.cpu().abs().max(1).values
    assert torch.equal(yhat.cpu().argmax(1)[clear], ry.cpu().argmax(1)[clear])


@pytest.mark.parametrize("B,T", [(5, 60), (3, 9), (2, 61)])
def test_simt_path(built_lib, sd, B, T):
    eng = _engine(sd, simt=True)
    x = synth.uestc_motions(B, T, seed=3 + T).cuda()
    eng.kernel_stats(reset=True)
    yhat, feats = eng.stgcn_classify(x)
    st = eng.kernel_stats()
    assert st["gemm_tc"] == 0 and st["gemm_simt"] == 20 and st["misc"] == 31, st
    ry, rf = _f64(sd, x)
    ey, ef = _rel_rows(yhat, ry), _rel_rows(feats, rf)
    print(f"uestc gemm=simt B={B} T={T}: yhat {ey:.2e} features {ef:.2e}")
    assert ey < GATE and ef < GATE


def test_weight_scales(built_lib):
    """Packed weights at split16 exponents other than 14 and different from each other.  After the BatchNorms are
    folded in, these scales put block 0's gcn weight at exponent 9 and the temporal convolutions of blocks 1, 4 (with
    its residual segment) and 9 at 13, 10 and 11; the activations stay below 2^14."""
    sd = synth.stgcn_state_dict(77)
    scales = {"st_gcn_networks.0.gcn.conv.weight": 2.0 ** 4, "st_gcn_networks.1.tcn.2.weight": 2.0 ** 3,
              "st_gcn_networks.4.tcn.2.weight": 2.0 ** 4, "st_gcn_networks.4.residual.0.weight": 2.0 ** 4,
              "st_gcn_networks.9.tcn.2.weight": 2.0 ** 6, "fcn.weight": 2.0 ** 6}
    sd = {k: v * scales.get(k, 1.0) if v.is_floating_point() else v for k, v in sd.items()}
    eng = _engine(sd)
    x = synth.uestc_motions(16, 60, seed=5).cuda()
    yhat, feats = eng.stgcn_classify(x)
    ry, rf = _f64(sd, x)
    ey, ef = _rel_rows(yhat, ry), _rel_rows(feats, rf)
    print(f"uestc weight scales: yhat {ey:.2e} features {ef:.2e}")
    assert ey < GATE and ef < GATE


def test_isolation_and_bit_identity(eng):
    B, T = 40, 60
    x = synth.uestc_motions(B, T, seed=8).cuda()
    ref = eng.stgcn_classify(x)
    assert all(torch.equal(a, b) for a, b in zip(ref, eng.stgcn_classify(x)))
    # a NaN inside one sequence stays there (the gcn GEMM's ReLU epilogue flushes it to zero, so that sequence's
    # outputs change rather than turn NaN), and so does a huge value
    keep = (torch.arange(B) != 7).cuda()
    for bad in (float("nan"), 1e30):
        xn = x.clone()
        xn[7, 3, 1, 30] = bad
        out = eng.stgcn_classify(xn)
        for a, r in zip(out, ref):
            assert not torch.equal(a[7], r[7])
            assert torch.equal(a[keep], r[keep])
    # batch permutation, B = 1, and chunking
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(1)).cuda()
    assert all(torch.equal(a, r[perm]) for a, r in zip(eng.stgcn_classify(x[perm]), ref))
    for b in (0, 13, B - 1):
        assert all(torch.equal(a[0], r[b]) for a, r in zip(eng.stgcn_classify(x[b:b + 1]), ref))
    for chunk in ("1", "7", "0"):
        eng.set_option("stgcn_chunk", chunk)
        assert all(torch.equal(a, r) for a, r in zip(eng.stgcn_classify(x), ref))


def test_kernel_stats_and_chunks(built_lib, sd):
    eng = _engine(sd)
    x = synth.uestc_motions(20, 60, seed=2).cuda()
    eng.kernel_stats(reset=True)
    eng.stgcn_classify(x)
    st = eng.kernel_stats(reset=True)
    assert st["gemm_tc"] == 20 and st["misc"] == 11 and st["gemm_simt"] == 0, st
    assert sum(st.values()) == 31, st
    eng.set_option("stgcn_chunk", "7")
    eng.stgcn_classify(x)
    st = eng.kernel_stats(reset=True)
    assert st["gemm_tc"] == 20 * 3 and st["misc"] == 11 * 3 and st["gemm_simt"] == 0, st


@pytest.fixture(scope="module")
def dropin(sd, tmp_path_factory):
    p = str(tmp_path_factory.mktemp("smpl") / "kintree_table.pkl")
    write_kintree(p)
    m = B200STGCN(in_channels=6, kintree_path=p, num_class=40, graph_args=GRAPH, edge_importance_weighting=True)
    m.load_state_dict(sd, strict=True)
    return m.eval().cuda()


@pytest.mark.parametrize("B", [1, 6])
def test_dropin_as_uestc_metrics_calls_it(dropin, sd, B):
    """UESTCMetrics.update's input: m_rst [B, T, 150] viewed [B, T, 6, 25], permuted to [B, 25, 6, T], joints :-1."""
    T = 60
    x = synth.uestc_motions(B, T, seed=11 + B)                              # [B, 24, 6, T]
    m = torch.zeros(B, T, 6, 25)
    m[..., :24] = x.permute(0, 3, 2, 1)
    m_rst = m.reshape(B, T, 150).cuda()
    motion = m_rst.view(*m_rst.shape[:-1], 6, 25).permute(0, 3, 2, 1)[:, :-1]
    assert not motion.is_contiguous()
    out = dropin(motion)
    assert set(out) == {"output", "features", "yhat"} and out["output"] is motion
    assert tuple(out["yhat"].shape) == (B, 40)
    assert tuple(out["features"].shape) == ((256,) if B == 1 else (B, 256))
    ry, rf = _f64(sd, x.cuda())
    assert _rel_rows(out["yhat"], ry) < GATE and _rel_rows(out["features"].reshape(B, 256), rf) < GATE


def test_refusals(built_lib, eng, sd):
    with pytest.raises(ValueError):
        eng.stgcn_classify(torch.zeros(2, 24, 5, 10, device="cuda"))
    with pytest.raises(ValueError):
        eng.stgcn_classify(torch.zeros(2, 24, 6, 0, device="cuda"))
    bad = Engine(make_config(num_layers=0, vae="none"), 0)
    with pytest.raises(RuntimeError):
        bad.stgcn_classify(torch.zeros(1, 24, 6, 4, device="cuda"))
    bad.stgcn_configure(_lib.default_stgcn_config())
    with pytest.raises(RuntimeError, match="missing"):
        bad.load_state_dict({k: v for k, v in sd.items() if k != "st_gcn_networks.4.residual.1.running_var"}, PREFIX)
        bad.finalize()
    cfg = _lib.default_stgcn_config()
    cfg.num_class = 0
    with pytest.raises(RuntimeError):
        Engine(make_config(num_layers=0, vae="none"), 0).stgcn_configure(cfg)
