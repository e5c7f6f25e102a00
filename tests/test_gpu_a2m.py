"""GPU tests of the native HumanAct12 action classifier (pytest -m gpu): the reference fixture, float64 accuracy over
batch, length, depth and width (fp32 torch with TF32 off printed beside it), the predicted class, weight scales,
isolation and bit-identity, kernel selection (one k_gru_seq_tc launch per layer), the CUDA-core path, the drop-in
modules under the reference's RNG draw, and the refusals."""
import ctypes as C

import pytest
import torch

from conftest import golden
from mld_b200 import _lib, synth
from mld_b200.engine import Engine, make_config
from oracle import a2m_gru as O
from oracle.make_golden_a2m import EXPLICIT_LENS, RNG_SEED, SEEDED_LENS, WEIGHT_SEED, golden_inputs

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
GATE = 5e-5
PREFIX = "gru_classifier."


def _rel_rows(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float(((a - b).abs().max(1).values / b.abs().max(1).values).max())


def _engine(sd, simt=False, **dims):
    d = {**synth.A2M_DIMS, **dims}
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    if simt:
        eng.set_option("gemm", "simt")
    cfg = _lib.default_a2m_config()
    for k, v in d.items():
        setattr(cfg, k, v)
    eng.a2m_configure(cfg)
    eng.load_state_dict(sd, PREFIX)
    eng.finalize()
    return eng


def _ragged(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    ln = torch.randint(1, T + 1, (B,), generator=g)
    ln[0] = T
    if B > 1:
        ln[-1] = 1
    return ln


def _h0(L, B, H, seed):
    return torch.randn(L, B, H, generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.fixture(scope="module", autouse=True)
def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.fixture(scope="module")
def sd():
    return synth.a2m_state_dict(WEIGHT_SEED)


@pytest.fixture(scope="module")
def eng(built_lib, sd):
    return _engine(sd)


def test_reference_fixture(eng, sd):
    g = golden("a2m_gru.npz")
    x1, h0, x2 = golden_inputs()
    logits, feats = eng.a2m_classify(x1.cuda(), torch.tensor(EXPLICIT_LENS), h0.cuda())
    assert _rel_rows(logits, torch.as_tensor(g["logits_explicit"])) < 2e-4
    assert _rel_rows(feats, torch.as_tensor(g["features_explicit"])) < 2e-4
    from mld_b200.evaluator import B200MotionDiscriminator, B200MotionDiscriminatorForFID
    cls, fid = B200MotionDiscriminator(**synth.A2M_DIMS).cuda(), B200MotionDiscriminatorForFID(**synth.A2M_DIMS).cuda()
    cls.load_state_dict(sd, strict=True)
    fid.load_state_dict(sd, strict=True)
    torch.manual_seed(RNG_SEED)
    l2 = torch.tensor(SEEDED_LENS)
    logits2, feats2 = cls(x2.cuda(), lengths=l2), fid(x2.cuda(), lengths=l2)
    assert _rel_rows(logits2, torch.as_tensor(g["logits_seeded"])) < 2e-4
    assert _rel_rows(feats2, torch.as_tensor(g["features_seeded"])) < 2e-4


_ENGINES = {}


def _eng_for(H, L):
    if (H, L) not in _ENGINES:
        sd = synth.a2m_state_dict(100 + H + L, hidden_size=H, hidden_layer=L)
        _ENGINES[H, L] = (_engine(sd, hidden_size=H, hidden_layer=L), sd)
    return _ENGINES[H, L]


@pytest.mark.parametrize("H,L", [(128, 2), (128, 1), (128, 3), (64, 1), (64, 2), (64, 3)])
@pytest.mark.parametrize("T", [1, 2, 60, 200])
@pytest.mark.parametrize("B", [1, 5, 32, 300, 4096])
def test_float64(built_lib, B, T, H, L):
    eng, sd = _eng_for(H, L)
    x = synth.a2m_motions(B, T, seed=B * 7 + T).cuda()
    ln = torch.tensor([T]) if B == 1 else _ragged(B, T, B + T)
    h0 = _h0(L, B, H, B + 3 * T)
    logits, feats = eng.a2m_classify(x, ln, h0)
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    rl, rf = O.classify(sd64, x.double(), ln.tolist(), h0.double())
    tl, tf = O.TorchDiscriminator({k: v.cuda() for k, v in sd.items()}, 72, H, L, 12).cuda().both(x, ln, h0)
    el, ef = _rel_rows(logits, rl), _rel_rows(feats, rf)
    tel, tef = _rel_rows(tl, rl), _rel_rows(tf, rf)
    print(f"a2m B={B} T={T} H={H} L={L}: logits {el:.2e} features {ef:.2e} (fp32 torch {tel:.2e} {tef:.2e})")
    assert el < GATE and ef < GATE
    # the predicted class, wherever the float64 top-2 margin is clear
    top = rl.cpu().topk(2, dim=1).values
    clear = (top[:, 0] - top[:, 1]) > 1e-3 * rl.cpu().abs().max(1).values
    assert torch.equal(logits.cpu().argmax(1)[clear], rl.cpu().argmax(1)[clear])


def test_weight_scales(built_lib):
    """W_ih / W_hh of each layer at split16 exponents other than 14 and different from each other."""
    sd = synth.a2m_state_dict(77)
    scales = {"recurrent.weight_ih_l0": 2.0 ** 6, "recurrent.weight_hh_l0": 2.0 ** -5,
              "recurrent.weight_ih_l1": 2.0 ** -9, "recurrent.weight_hh_l1": 2.0 ** 2}
    sd = {k: v * scales.get(k, 1.0) for k, v in sd.items()}
    eng = _engine(sd)
    B, T = 64, 60
    x = synth.a2m_motions(B, T, seed=5).cuda() * 2.0 ** -6
    ln = _ragged(B, T, 9)
    h0 = _h0(2, B, 128, 4)
    logits, feats = eng.a2m_classify(x, ln, h0)
    rl, rf = O.classify({k: v.double().cuda() for k, v in sd.items()}, x.double(), ln.tolist(), h0.double())
    el, ef = _rel_rows(logits, rl), _rel_rows(feats, rf)
    print(f"a2m weight scales: logits {el:.2e} features {ef:.2e}")
    assert el < GATE and ef < GATE


def test_isolation_and_bit_identity(eng):
    B, T = 40, 60
    x = synth.a2m_motions(B, T, seed=8).cuda()
    ln = _ragged(B, T, 3)
    h0 = _h0(2, B, 128, 6)
    ref = eng.a2m_classify(x, ln, h0)
    again = eng.a2m_classify(x, ln, h0)
    assert all(torch.equal(a, b) for a, b in zip(ref, again))
    # garbage past each length changes no bit
    xg = x.clone()
    for b, n in enumerate(ln.tolist()):
        xg[b, ..., n:] = float("nan") if b % 2 else 1e30
    assert all(torch.equal(a, b) for a, b in zip(ref, eng.a2m_classify(xg, ln, h0)))
    # a NaN inside one sequence stays there
    xn = x.clone()
    xn[7, 3, 1, 0] = float("nan")
    out = eng.a2m_classify(xn, ln, h0)
    for a, r in zip(out, ref):
        assert torch.isnan(a[7]).all()
        keep = torch.arange(B) != 7
        assert torch.equal(a[keep], r[keep])
    # batch permutation and B = 1
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(1))
    out = eng.a2m_classify(x[perm.cuda()], ln[perm], h0[:, perm.cuda()])
    assert all(torch.equal(a, r[perm.cuda()]) for a, r in zip(out, ref))
    for b in (0, 13, B - 1):
        one = eng.a2m_classify(x[b:b + 1], ln[b:b + 1], h0[:, b:b + 1])
        assert all(torch.equal(a[0], r[b]) for a, r in zip(one, ref))


def test_kernel_stats_and_chunks(built_lib, sd):
    eng = _engine(sd)
    B, T = 200, 60
    x = synth.a2m_motions(B, T, seed=2).cuda()
    ln = _ragged(B, T, 2)
    h0 = _h0(2, B, 128, 2)
    eng.kernel_stats(reset=True)
    ref = eng.a2m_classify(x, ln, h0)
    st = eng.kernel_stats(reset=True)
    assert st["gru_tc"] == 2 and st["gemm_tc"] == 2 and st["gemm_simt"] == 0, st
    eng.set_option("a2m_chunk", "70")
    out = eng.a2m_classify(x, ln, h0)
    st = eng.kernel_stats(reset=True)
    assert st["gru_tc"] == 2 * 3 and st["gemm_simt"] == 0, st
    assert all(torch.equal(a, r) for a, r in zip(out, ref))


@pytest.mark.parametrize("H,L", [(128, 2), (64, 3)])
def test_simt_path(built_lib, H, L):
    sd = synth.a2m_state_dict(5 + H, hidden_size=H, hidden_layer=L)
    eng = _engine(sd, simt=True, hidden_size=H, hidden_layer=L)
    B, T = 37, 60
    x = synth.a2m_motions(B, T, seed=4).cuda()
    ln = _ragged(B, T, 4)
    h0 = _h0(L, B, H, 9)
    eng.kernel_stats(reset=True)
    logits, feats = eng.a2m_classify(x, ln, h0)
    st = eng.kernel_stats()
    assert st["gru_tc"] == 0 and st["gemm_tc"] == 0 and st["gemm_simt"] == L * (T + 1), st
    rl, rf = O.classify({k: v.double().cuda() for k, v in sd.items()}, x.double(), ln.tolist(), h0.double())
    el, ef = _rel_rows(logits, rl), _rel_rows(feats, rf)
    print(f"a2m gemm=simt H={H} L={L}: logits {el:.2e} features {ef:.2e}")
    assert el < GATE and ef < GATE


@pytest.fixture(scope="module")
def dropins(sd):
    from mld_b200.evaluator import B200MotionDiscriminator, B200MotionDiscriminatorForFID
    cls, fid = B200MotionDiscriminator(**synth.A2M_DIMS).cuda(), B200MotionDiscriminatorForFID(**synth.A2M_DIMS).cuda()
    cls.load_state_dict(sd, strict=True)
    fid.load_state_dict(sd, strict=True)
    return cls, fid, O.TorchDiscriminator({k: v.cuda() for k, v in sd.items()}, **synth.A2M_DIMS).cuda()


def test_dropins_draw_the_reference_rng(dropins):
    cls, fid, ref = dropins
    B, T = 32, 60
    x = synth.a2m_motions(B, T, seed=12).cuda()
    ln = torch.full((B,), T)
    torch.manual_seed(99)
    a, b = cls(x, lengths=ln), fid(x, lengths=ln)
    st_a = torch.get_rng_state()
    torch.manual_seed(99)
    ra, rb = ref.both(x, ln)[0], ref.both(x, ln)[1]
    assert torch.equal(st_a, torch.get_rng_state())
    assert _rel_rows(a, ra) < GATE and _rel_rows(b, rb) < GATE


def test_humanact_update_sequence(dropins):
    """HUMANACTMetrics.update's four calls, restated: the same confusion matrices except on near-ties, and the
    same features within the gate."""
    cls, fid, ref = dropins
    B, T = 32, 60
    rec, gt = synth.a2m_motions(B, T, seed=40).cuda(), synth.a2m_motions(B, T, seed=41).cuda()
    labels = torch.randint(0, 12, (B,), generator=torch.Generator().manual_seed(3))
    ln = torch.full((B,), T)

    def update(c, f):
        torch.manual_seed(2024)
        p, gp = c(rec, ln), c(gt, ln)
        return p, gp, f(rec, ln), f(gt, ln)

    ours = update(cls, fid)
    theirs = update(lambda x, l: ref.both(x, l)[0], lambda x, l: ref.both(x, l)[1])
    for p, q in zip(ours[:2], theirs[:2]):
        top = q.cpu().topk(2, dim=1).values
        clear = (top[:, 0] - top[:, 1]) > 1e-3 * q.cpu().abs().max(1).values
        conf_a, conf_b = torch.zeros(12, 12, dtype=torch.long), torch.zeros(12, 12, dtype=torch.long)
        for lab, pa, pb in zip(labels[clear], p.cpu().argmax(1)[clear], q.cpu().argmax(1)[clear]):
            conf_a[lab][pa] += 1
            conf_b[lab][pb] += 1
        assert torch.equal(conf_a, conf_b)
    for p, q in zip(ours[2:], theirs[2:]):
        assert _rel_rows(p, q) < GATE


def test_explicit_hidden_unit_is_honoured(dropins, eng):
    cls, fid, _ = dropins
    B, T = 6, 60
    x = synth.a2m_motions(B, T, seed=50).cuda()
    ln = torch.tensor([60, 1, 30, 60, 2, 59])
    h0 = _h0(2, B, 128, 51)
    logits, feats = eng.a2m_classify(x, ln, h0)
    assert torch.equal(cls(x, lengths=ln, hidden_unit=h0), logits)
    assert torch.equal(fid(x, lengths=ln, hidden_unit=h0), feats)
    assert not torch.equal(cls(x, lengths=ln, hidden_unit=h0 * 0.5), logits)


def test_refusals(built_lib, eng, sd):
    x = synth.a2m_motions(3, 10, seed=1).cuda()
    h0 = _h0(2, 3, 128, 1)
    with pytest.raises(ValueError, match=r"\[1, 10\]"):
        eng.a2m_classify(x, [10, 0, 3], h0)
    with pytest.raises(ValueError, match="h0"):
        eng.a2m_classify(x, [10, 3, 3], h0[:, :2])
    lib = _lib.lib()
    xd = x.reshape(3, 72, 10).contiguous()
    out = torch.empty(3, 12, device="cuda")
    for bad in ([10, 11, 3], [0, 3, 3]):
        ln = torch.tensor(bad, dtype=torch.int32, device="cuda")
        rc = lib.mldb_a2m_classify(eng._h, C.c_void_p(xd.data_ptr()), C.c_void_p(ln.data_ptr()),
                                   C.c_void_p(h0.data_ptr()), 3, 10, C.c_void_p(out.data_ptr()), None, None)
        assert rc != 0 and b"lengths[" in lib.mldb_last_error()
    rc = lib.mldb_a2m_classify(eng._h, C.c_void_p(xd.data_ptr()), C.c_void_p(ln.data_ptr()), C.c_void_p(h0.data_ptr()),
                               0, 10, C.c_void_p(out.data_ptr()), None, None)
    assert rc != 0 and b"B=0" in lib.mldb_last_error()
    e = Engine(make_config(num_layers=0, vae="none"), 0)
    cfg = _lib.default_a2m_config()
    cfg.hidden_size = 256
    with pytest.raises(RuntimeError, match="64 or 128"):
        e.a2m_configure(cfg)
    cfg.hidden_size = 128
    e.a2m_configure(cfg)
    e.a2m_cfg = cfg
    with pytest.raises(RuntimeError, match="finalize"):
        e.a2m_classify(x, [10, 3, 3], h0)
    e2 = Engine(make_config(num_layers=0, vae="none"), 0)
    with pytest.raises(RuntimeError, match="not configured"):
        e2.a2m_classify(x, [10, 3, 3], h0)
