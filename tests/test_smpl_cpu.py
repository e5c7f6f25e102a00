"""CPU tests of the SMPL layer: the float64 oracle against the reference glue's fixture, the pickle loader (sparse
J_regressor, chumpy-like arrays) and the drop-in's refusals, which all happen before any GPU work."""
import os

import numpy as np
import pytest
import torch

from conftest import golden
from mld_b200 import synth
from mld_b200.smpl import B200Rotation2xyz, load_smpl
from oracle import smpl as O
from oracle.make_golden_smpl import CASES, MODEL_SEED, V, case_inputs


class _ArrayOnly:
    """Exposes only __array__, as a chumpy Ch does to numpy."""

    def __init__(self, a):
        self._a = a

    def __array__(self, dtype=None, copy=None):
        return self._a if dtype is None else self._a.astype(dtype)


@pytest.fixture(scope="module")
def model_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("smpl")
    synth.write_smpl_pkl(str(d / "SMPL_NEUTRAL.pkl"), synth.smpl_model(MODEL_SEED, V))
    return str(d)


@pytest.mark.parametrize("name,B,T,seed", CASES)
def test_oracle_matches_reference_glue(model_dir, name, B, T, seed):
    g = golden("smpl.npz")
    m = O.load_model(model_dir)
    x, mask = case_inputs(name, B, T, seed)
    xx = x.double().view(B, T, 6, 25).permute(0, 3, 2, 1)
    for jt in ("smpl", "vertices"):
        for vt in (0, 1):
            ref = torch.from_numpy(g[f"{name}_{jt}_{vt}"])
            out = O.rotation2xyz(m, xx, mask, jt, bool(vt))
            assert out.shape == ref.shape
            assert torch.isfinite(out).all() and torch.isfinite(ref).all()
            assert torch.allclose(out, ref, rtol=0, atol=1e-12), (jt, vt, float((out - ref).abs().max()))


def test_fixture_pins_the_glue():
    """What the fixture holds: masked frames are zero before the translation, which every frame then gets."""
    g = golden("smpl.npz")
    name, B, T, seed = CASES[0]
    x, mask = case_inputs(name, B, T, seed)
    trans = x.double().view(B, T, 6, 25)[:, :, :3, 24].permute(0, 2, 1)        # [B, 3, T]
    off = (trans - trans[:, :, [0]])[:, None]
    for jt in ("smpl", "vertices"):
        a, b = torch.from_numpy(g[f"{name}_{jt}_0"]), torch.from_numpy(g[f"{name}_{jt}_1"])
        assert (a[~mask[:, None, None, :].expand_as(a)] == 0).all()
        assert torch.allclose(b - a, off.expand_as(a), atol=1e-12)
    assert (torch.from_numpy(g[f"{name}_smpl_0"])[:, 0] == 0).all()           # the root subtracted per frame


@pytest.mark.parametrize("wrap", [None, _ArrayOnly])
def test_load_smpl(tmp_path, wrap):
    m = synth.smpl_model(5, 70)
    path = str(tmp_path / "SMPL_NEUTRAL.pkl")
    synth.write_smpl_pkl(path, m, array=wrap)
    for p in (path, str(tmp_path)):
        got = load_smpl(p)
        assert got["parents"].dtype == torch.int64 and got["parents"].tolist() == list(synth.SMPL_PARENTS)
        for k in ("v_template", "posedirs", "J_regressor", "lbs_weights"):
            assert got[k].dtype == torch.float32 and torch.equal(got[k], m[k].float()), k
        o = O.load_model(p)
        for k in ("v_template", "posedirs", "J_regressor", "lbs_weights"):
            assert torch.equal(o[k], m[k].double()), k


def test_load_smpl_refuses_unordered_parents(tmp_path):
    m = synth.smpl_model(5, 40)
    m["parents"] = m["parents"].clone()
    m["parents"][3] = 7
    synth.write_smpl_pkl(str(tmp_path / "SMPL_NEUTRAL.pkl"), m)
    with pytest.raises(ValueError, match="parents"):
        load_smpl(str(tmp_path))


# The persistent buffers of the reference's SMPL (mld/transforms/smpl.py: smplx 0.1.28's SMPLLayer, which has no
# parameters, plus J_regressor_extra), i.e. the rot2xyz.smpl_model.* keys of every action-model checkpoint:
# name -> (shape for SMPL's V = 6890 and 13776 faces, dtype)
REFERENCE_SMPL_KEYS = {
    "faces_tensor": ((13776, 3), torch.int64), "shapedirs": ((6890, 3, 10), torch.float32),
    "v_template": ((6890, 3), torch.float32), "J_regressor": ((24, 6890), torch.float32),
    "posedirs": ((207, 20670), torch.float32), "parents": ((24,), torch.int64),
    "lbs_weights": ((6890, 24), torch.float32), "vertex_joint_selector.extra_joints_idxs": ((21,), torch.int64),
    "J_regressor_extra": ((9, 6890), torch.float32),
}


def _reference_state(seed):
    """A state dict with the reference SMPL's key set, shapes and dtypes (a synthetic model in its five used keys)."""
    m = synth.smpl_model(seed, 6890)
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, (shape, dt) in REFERENCE_SMPL_KEYS.items():
        sd[k] = m[k] if k in m else (torch.randint(0, 6890, shape, generator=g) if dt == torch.int64
                                     else torch.rand(shape, generator=g))
    return sd


@pytest.mark.parametrize("with_extra", [True, False])
def test_dropin_strict_loads_reference_checkpoint(built_lib, tmp_path, with_extra):
    """The drop-in as MLD holds it (self.rot2xyz) takes an action checkpoint's rot2xyz.smpl_model.* keys under a strict
    load through the parent, whether or not J_regressor_extra.npy was beside the pickle, and the load marks its engine
    for a rebuild."""
    synth.write_smpl_pkl(str(tmp_path / "SMPL_NEUTRAL.pkl"), synth.smpl_model(3, 6890))
    if with_extra:
        np.save(str(tmp_path / "J_regressor_extra.npy"), np.full((9, 6890), 1 / 6890, dtype=np.float64))

    class MLDLike(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.rot2xyz = B200Rotation2xyz(smpl_path=str(tmp_path))
            self.head = torch.nn.Linear(2, 2)

    model = MLDLike()
    mine = {k[len("rot2xyz.smpl_model."):]: v for k, v in model.state_dict().items() if k.startswith("rot2xyz.")}
    assert set(mine) == set(REFERENCE_SMPL_KEYS)
    if with_extra:
        for k, (shape, dt) in REFERENCE_SMPL_KEYS.items():
            if k != "faces_tensor":                     # the synthetic pickle's faces are a placeholder
                assert tuple(mine[k].shape) == shape and mine[k].dtype == dt, k
    ref = _reference_state(11)
    sd = {f"rot2xyz.smpl_model.{k}": v for k, v in ref.items()}
    sd.update({f"head.{k}": v for k, v in model.head.state_dict().items()})
    r2x = model.rot2xyz
    before = r2x._weights_epoch
    model.load_state_dict(sd, strict=True)
    assert r2x._weights_epoch != before
    got = model.state_dict()
    for k, v in ref.items():
        assert torch.equal(got[f"rot2xyz.smpl_model.{k}"], v), k
    assert all(torch.equal(r2x._engine_state_dict()[k], ref[k]) for k in
               ("v_template", "posedirs", "J_regressor", "lbs_weights", "parents"))
    with pytest.raises(RuntimeError, match="Unexpected key"):
        model.load_state_dict({**sd, "rot2xyz.smpl_model.betas": torch.zeros(1, 10)}, strict=True)


def _call(r2x, x, **kw):
    args = dict(mask=None, pose_rep="rot6d", glob=True, translation=True, jointstype="smpl", vertstrans=True,
                betas=None, beta=0, glob_rot=None, get_rotations_back=False)
    args.update(kw)
    return r2x(x, **args)


def test_dropin_refusals(built_lib, model_dir):
    r2x = B200Rotation2xyz(smpl_path=model_dir)
    assert sorted(r2x.state_dict()) == sorted(f"smpl_model.{k}" for k in REFERENCE_SMPL_KEYS)
    x = synth.smpl_feats(2, 7).view(2, 7, 6, 25).permute(0, 3, 2, 1)
    assert _call(r2x, x, pose_rep="xyz") is x
    for kw, exc in ((dict(pose_rep="rotvec"), NotImplementedError), (dict(pose_rep="rotmat"), NotImplementedError),
                    (dict(glob=False), TypeError), (dict(glob=False, glob_rot=[0.0, 0.0, 0.0]), NotImplementedError),
                    (dict(translation=False), NotImplementedError), (dict(jointstype="a2m"), NotImplementedError),
                    (dict(jointstype="vibe"), NotImplementedError), (dict(jointstype="bogus"), NotImplementedError),
                    (dict(betas=torch.zeros(14, 10)), NotImplementedError), (dict(beta=1), NotImplementedError),
                    (dict(get_rotations_back=True), NotImplementedError),
                    (dict(mask=torch.ones(2, 6, dtype=torch.bool)), ValueError),
                    (dict(mask=torch.ones(2, 7)), ValueError)):
        with pytest.raises(exc):
            _call(r2x, x, **kw)
    for bad in (torch.zeros(2, 24, 6, 7), torch.zeros(2, 25, 3, 7), torch.zeros(2, 25, 6, 0)):
        with pytest.raises(ValueError):
            _call(r2x, bad)
    # everything above was refused before an engine was built (none can exist on a CPU-only machine)
    assert r2x._engine is None
