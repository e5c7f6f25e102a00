"""GPU tests of the native SMPL layer (pytest -m gpu): the reference glue's fixture, float64 parity over batch, length
and vertex count for both joint types and both vertstrans values, posedirs at other split16 exponents, isolation and
bit-identity, the kernel counts, and the drop-in called exactly as MLD's two lambdas call it."""
import pytest
import torch

from conftest import golden
from mld_b200 import _lib, synth
from mld_b200.engine import Engine, make_config
from mld_b200.smpl import B200Rotation2xyz
from oracle import smpl as O
from oracle.make_golden_smpl import CASES, MODEL_SEED, V as FIXTURE_V, case_inputs
from weight_scales import engine_exponent

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
GATE = 1e-5                       # of each frame's largest absolute coordinate
KIND = {"smpl": _lib.SMPL_JOINTS, "vertices": _lib.SMPL_VERTICES}
_worst = {}


def _engine(m):
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    cfg = _lib.default_smpl_config()
    cfg.num_vertices = m["v_template"].shape[0]
    eng.smpl_configure(cfg)
    eng.load_state_dict(m, "smpl.")
    eng.finalize()
    return eng


def _f64(m, x, mask, jt, vt):
    B, T = x.shape[:2]
    md = {k: v.cuda() for k, v in m.items()}
    xx = x.cuda().double().view(B, T, 6, 25).permute(0, 3, 2, 1)
    return O.rotation2xyz(md, xx, None if mask is None else mask.cuda(), jt, vt)


def _rel_frames(a, ref):
    """max over frames of |a - ref| / the frame's largest |ref| coordinate ([B, n, 3, T])."""
    a, ref = a.double(), ref.to(a.device).double()
    err = (a - ref).abs().amax(dim=(1, 2))
    scale = ref.abs().amax(dim=(1, 2)).clamp_min(1e-30)
    return float((err / scale).max())


def _rel_chunked(out, m, x, mask, jt, vt, elems=1 << 25):
    """_rel_frames against the float64 oracle, a few sequences at a time (the oracle skins every vertex for either
    joint type, and its [frames, V, 4, 4] transforms would not fit at once)."""
    B, T = x.shape[:2]
    cb = max(1, elems // (T * m["v_template"].shape[0] * 16))
    return max(_rel_frames(out[b:b + cb], _f64(m, x[b:b + cb], None if mask is None else mask[b:b + cb], jt, vt))
               for b in range(0, B, cb))


@pytest.fixture(scope="module")
def models():
    return {V: synth.smpl_model(7 + V, V) for V in (333, 6890)}


@pytest.fixture(scope="module")
def engines(built_lib, models):
    return {V: _engine(m) for V, m in models.items()}


@pytest.mark.parametrize("name,B,T,seed", CASES)
def test_reference_fixture(built_lib, name, B, T, seed):
    g = golden("smpl.npz")
    eng = _engine(synth.smpl_model(MODEL_SEED, FIXTURE_V))
    x, mask = case_inputs(name, B, T, seed)
    for jt in ("smpl", "vertices"):
        for vt in (0, 1):
            ref = torch.from_numpy(g[f"{name}_{jt}_{vt}"])
            out = eng.smpl_forward(x.cuda(), None if mask is None else mask.cuda(), KIND[jt], bool(vt))
            assert torch.isfinite(out).all()
            e = _rel_frames(out, ref)
            print(f"smpl fixture {name} {jt} vertstrans={vt}: {e:.2e}")
            assert e < GATE


@pytest.mark.parametrize("V", [333, 6890])
@pytest.mark.parametrize("T", [1, 7, 60, 61, 200])
@pytest.mark.parametrize("B", [1, 5, 32, 300])
def test_float64(engines, models, B, T, V):
    x = synth.smpl_feats(B, T, seed=B * 13 + T)
    g = torch.Generator().manual_seed(B + T)
    mask = torch.rand(B, T, generator=g) > 0.2
    mask[:, 0] = True
    for jt in ("smpl", "vertices"):
        for vt in (False, True):
            out = engines[V].smpl_forward(x.cuda(), mask.cuda(), KIND[jt], vt)
            e = _rel_chunked(out, models[V], x, mask, jt, vt)
            del out
            key = (jt, V)
            _worst[key] = max(_worst.get(key, 0.0), e)
            print(f"smpl B={B} T={T} V={V} {jt} vertstrans={vt}: {e:.2e} (worst so far {_worst[key]:.2e})")
            assert e < GATE


@pytest.mark.parametrize("s", [13, 9, 4])
def test_posedirs_weight_scales(built_lib, s):
    """posedirs packed at split16 exponent s rather than 14 (the pose offsets scaled up to match)."""
    m = synth.smpl_model(21, 333)
    pd = m["posedirs"]
    m["posedirs"] = pd * (1.5 * 2.0 ** (13 - s) / float(pd.abs().max()))
    assert engine_exponent(m["posedirs"]) == s
    eng = _engine(m)
    x = synth.smpl_feats(6, 60, seed=3)
    out = eng.smpl_forward(x.cuda(), None, _lib.SMPL_VERTICES, True)
    e = _rel_frames(out, _f64(m, x, None, "vertices", True))
    print(f"smpl posedirs at exponent {s}: {e:.2e}")
    assert e < GATE


def test_isolation_and_bit_identity(engines):
    eng = engines[333]
    B, T = 6, 61
    x = synth.smpl_feats(B, T, seed=9).cuda()
    mask = torch.ones(B, T, dtype=torch.bool, device="cuda")
    mask[2, 40:] = False
    mask[4, ::3] = False
    for kind in (_lib.SMPL_JOINTS, _lib.SMPL_VERTICES):
        for vt in (False, True):
            ref = eng.smpl_forward(x, mask, kind, vt)
            assert torch.equal(ref, eng.smpl_forward(x, mask, kind, vt))
            # one sequence changed: every other sequence bit-identical
            x1 = x.clone()
            x1[3] = x1[3].flip(0)
            o = eng.smpl_forward(x1, mask, kind, vt)
            keep = torch.arange(B, device="cuda") != 3
            assert torch.equal(o[keep], ref[keep]) and not torch.equal(o[3], ref[3])
            # garbage in masked-out frames' rotations reaches no output
            for bad in (float("nan"), float("inf"), 1e30):
                x2 = x.clone().view(B, T, 6, 25)
                x2[2, 45, :, :24] = bad
                x2[4, 3, :, :24] = bad
                assert torch.equal(eng.smpl_forward(x2.view(B, T, 150), mask, kind, vt), ref)
            # a sequence alone, or in another batch, gives the same bits
            assert torch.equal(eng.smpl_forward(x[4:5], mask[4:5], kind, vt)[0], ref[4])


def test_chunks(built_lib, models):
    """Sequences split over chunks (option smpl_chunk) give the bits of one chunk, the translation included."""
    B, T = 20, 61
    x = synth.smpl_feats(B, T, seed=23).cuda()
    mask = (torch.rand(B, T, generator=torch.Generator().manual_seed(4)) > 0.3).cuda()
    mask[5] = False
    for V in (333, 6890):
        eng = _engine(models[V])
        for kind, n in ((_lib.SMPL_JOINTS, 24), (_lib.SMPL_VERTICES, V)):
            for vt in (False, True):
                ref = eng.smpl_forward(x, mask, kind, vt)
                eng.set_option("smpl_chunk", "7")
                eng.kernel_stats(reset=True)
                out = eng.smpl_forward(x, mask, kind, vt)
                st = eng.kernel_stats(reset=True)
                eng.set_option("smpl_chunk", "0")
                assert st["misc"] == 3 and st["gemm_tc"] == (3 if kind == _lib.SMPL_VERTICES else 0), st
                assert torch.equal(out, ref)
                if V == 333:
                    assert _rel_frames(out, _f64(models[V], x.cpu(), mask.cpu(), "smpl" if n == 24 else "vertices",
                                                 vt)) < GATE


def test_kernel_stats(engines):
    eng = engines[6890]
    x = synth.smpl_feats(32, 60, seed=4).cuda()
    eng.kernel_stats(reset=True)
    eng.smpl_forward(x, None, _lib.SMPL_VERTICES, False)
    st = eng.kernel_stats(reset=True)
    assert st["gemm_tc"] == 1 and st["misc"] == 1 and sum(st.values()) == 2, st
    eng.smpl_forward(x, None, _lib.SMPL_JOINTS, True)
    st = eng.kernel_stats(reset=True)
    assert st["misc"] == 1 and sum(st.values()) == 1, st


def test_refusals(built_lib, engines, models):
    eng = engines[333]
    x = synth.smpl_feats(2, 5).cuda()
    with pytest.raises(ValueError):
        eng.smpl_forward(x[..., :149], None, _lib.SMPL_JOINTS, False)
    with pytest.raises(ValueError):
        eng.smpl_forward(x, torch.ones(2, 4, dtype=torch.bool, device="cuda"), _lib.SMPL_JOINTS, False)
    with pytest.raises(ValueError):
        eng.smpl_forward(x, None, 2, False)
    bad = Engine(make_config(num_layers=0, vae="none"), 0)
    with pytest.raises(RuntimeError):
        bad.smpl_forward(x, None, _lib.SMPL_JOINTS, False)
    cfg = _lib.default_smpl_config()
    cfg.num_vertices = 333
    bad.smpl_configure(cfg)
    m = models[333]
    with pytest.raises(RuntimeError, match="smpl.lbs_weights"):
        bad.load_state_dict({k: v for k, v in m.items() if k != "lbs_weights"}, "smpl.")
        bad.finalize()
    with pytest.raises(RuntimeError, match="smpl.posedirs"):
        bad.load_state_dict({"posedirs": m["posedirs"][:, :-3]}, "smpl.")
    unordered = Engine(make_config(num_layers=0, vae="none"), 0)
    unordered.smpl_configure(cfg)
    p = m["parents"].clone()
    p[5] = 9
    with pytest.raises(RuntimeError, match="smpl.parents"):
        unordered.load_state_dict({**m, "parents": p}, "smpl.")
        unordered.finalize()


@pytest.fixture(scope="module")
def dropin(tmp_path_factory, models):
    d = tmp_path_factory.mktemp("smpl")
    synth.write_smpl_pkl(str(d / "SMPL_NEUTRAL.pkl"), models[6890])
    return B200Rotation2xyz(smpl_path=str(d)).cuda(), str(d)


def test_dropin_as_mld_calls_it(dropin):
    """MLD's feats2joints_eval ('smpl', vertstrans=True) and feats2joints ('vertices', vertstrans=False) lambdas
    (mld.py:119-143) on a [B, T, 150] sample and a length mask, at the HumanAct12 test batch."""
    r2x, d = dropin
    B, T = 32, 60
    sample = synth.smpl_feats(B, T, seed=17).cuda()
    lengths = torch.randint(20, T + 1, (B,), generator=torch.Generator().manual_seed(2))
    mask = (torch.arange(T)[None] < lengths[:, None]).cuda()
    feats2joints_eval = lambda sample, mask: r2x(
        sample.view(*sample.shape[:-1], 6, 25).permute(0, 3, 2, 1), mask=mask, pose_rep='rot6d', glob=True,
        translation=True, jointstype='smpl', vertstrans=True, betas=None, beta=0, glob_rot=None,
        get_rotations_back=False)
    feats2joints = lambda sample, mask: r2x(
        sample.view(*sample.shape[:-1], 6, 25).permute(0, 3, 2, 1), mask=mask, pose_rep='rot6d', glob=True,
        translation=True, jointstype='vertices', vertstrans=False, betas=None, beta=0, glob_rot=None,
        get_rotations_back=False)
    j = feats2joints_eval(sample, mask)
    v = feats2joints(sample, mask)
    assert j.dtype == v.dtype == torch.float32 and j.device == v.device == sample.device
    assert tuple(j.shape) == (B, 24, 3, T) and tuple(v.shape) == (B, 6890, 3, T)
    m = O.load_model(d)
    ej = _rel_frames(j, _f64(m, sample.cpu(), mask.cpu(), "smpl", True))
    # a strict load through the parent (as test.py loads a checkpoint) rebuilds the engine with the loaded model
    parent = torch.nn.Module()
    parent.rot2xyz = r2x
    sd = parent.state_dict()
    m2 = synth.smpl_model(77, 6890)
    for k in ("v_template", "posedirs", "J_regressor", "lbs_weights"):
        sd[f"rot2xyz.smpl_model.{k}"] = m2[k]
    parent.load_state_dict(sd, strict=True)
    v2 = feats2joints(sample, mask)
    e2 = _rel_frames(v2, _f64(m2, sample.cpu(), mask.cpu(), "vertices", False))
    assert e2 < GATE and not torch.equal(v2, v)
    ev = _rel_frames(v, _f64(m, sample.cpu(), mask.cpu(), "vertices", False))
    print(f"smpl drop-in: joints {ej:.2e} vertices {ev:.2e}")
    assert ej < GATE and ev < GATE
