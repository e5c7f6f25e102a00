"""Generate tests/golden/smpl.npz with the reference's own Rotation2xyz glue (TEST INFRASTRUCTURE).

    python -m oracle.make_golden_smpl REFERENCE_ROOT      (or MLD_REFERENCE=REFERENCE_ROOT python -m ...)

smplx is not installed and no SMPL model is available offline, so a stand-in ``smplx`` package is put in
``sys.modules`` first: ``SMPLLayer`` (loads the pickle with ``oracle.smpl.load_model``, ``num_betas = 10``, forward =
``oracle.smpl.lbs`` in the input's dtype, joints = the 24 FK joints + 21 vertex picks as smplx's vertex joint
selector gives them) and ``lbs.vertices2joints``.  The reference's ``mld.transforms.rotation2xyz.Rotation2xyz`` and
its ``SMPL`` subclass are then imported unchanged and run in float64 on a synthetic model (``synth.smpl_model``,
written with ``synth.write_smpl_pkl`` beside a ``J_regressor_extra.npy``) for both joint types and both
``vertstrans`` values, as ``MLD``'s lambdas call it.  What this pins is the glue (mask, root, translation, layout)
and the loader; the LBS core is the restatement in ``oracle/smpl.py``, not smplx itself.
"""
from __future__ import annotations

import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "smpl.npz")
MODEL_SEED, V = 606, 45
# (name, B, T, feature seed): "mask" has a non-prefix mask, an all-false row and NaN in masked frames; "full" none
CASES = (("mask", 3, 9, 61), ("full", 2, 5, 62))
EXTRA_JOINTS = 9          # J_regressor_extra rows: the reference's JOINT_MAP reaches joint 53 = 45 + 9 - 1


def case_inputs(name, B, T, seed):
    """The features [B, T, 150] and mask [B, T] (bool or None) of a fixture case."""
    from mld_b200 import synth
    x = synth.smpl_feats(B, T, seed=seed)
    if name != "mask":
        return x, None
    mask = torch.ones(B, T, dtype=torch.bool)
    mask[0, [1, 4, 5, 8]] = False                     # not a length prefix
    mask[1] = False                                   # an all-false row
    mask[2, T - 3:] = False                           # a length prefix
    rot = x.view(B, T, 6, 25)
    rot[0, 4, :, 3] = float("nan")                    # NaN in masked frames' rotations
    rot[1, 2, :, :24] = float("nan")
    return x, mask


def _install_smplx():
    from oracle import smpl as O
    vertex_ids = list(range(0, 2 * 21, 2))           # 21 vertex picks (smplx: nose, eyes, ears, feet, fingertips)

    class SMPLLayer(torch.nn.Module):
        def __init__(self, model_path=None, **kwargs):
            super().__init__()
            self.m = O.load_model(model_path)
            self.num_betas = 10

        def forward(self, betas=None, body_pose=None, global_orient=None, **kwargs):
            assert betas is None or not bool(betas.abs().sum()), "the stand-in has zero betas only"
            pose = torch.cat([global_orient.reshape(-1, 1, 3, 3), body_pose.reshape(-1, 23, 3, 3)], 1)
            verts, joints = O.lbs(pose, self.m)
            joints = torch.cat([joints, verts[:, vertex_ids]], 1)
            return types.SimpleNamespace(vertices=verts, joints=joints)

    smplx = types.ModuleType("smplx")
    lbs = types.ModuleType("smplx.lbs")
    smplx.SMPLLayer, lbs.vertices2joints, smplx.lbs = SMPLLayer, O.vertices2joints, lbs
    sys.modules["smplx"], sys.modules["smplx.lbs"] = smplx, lbs


def main(ref_root: str = ""):
    ref_root = ref_root or os.environ.get("MLD_REFERENCE", "")
    if not ref_root:
        raise SystemExit("give the reference checkout (ChenFengYe/motion-latent-diffusion) as an argument or MLD_REFERENCE")
    sys.path.insert(0, ref_root)
    _install_smplx()
    from mld.transforms.rotation2xyz import Rotation2xyz
    from mld_b200 import synth
    model = synth.smpl_model(MODEL_SEED, V)
    out = {}
    with tempfile.TemporaryDirectory() as d:
        synth.write_smpl_pkl(os.path.join(d, "SMPL_NEUTRAL.pkl"), model)
        extra = np.random.default_rng(0).random((EXTRA_JOINTS, V))
        np.save(os.path.join(d, "J_regressor_extra.npy"), extra / extra.sum(1, keepdims=True))
        r2x = Rotation2xyz(smpl_path=d)
    for name, B, T, seed in CASES:
        x, mask = case_inputs(name, B, T, seed)
        xx = x.double().view(B, T, 6, 25).permute(0, 3, 2, 1)
        for jt, vt in (("smpl", True), ("smpl", False), ("vertices", False), ("vertices", True)):
            with torch.no_grad():
                o = r2x(xx, mask=mask, pose_rep="rot6d", glob=True, translation=True, jointstype=jt,
                        vertstrans=vt, betas=None, beta=0, glob_rot=None, get_rotations_back=False)
            out[f"{name}_{jt}_{int(vt)}"] = o.numpy()
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main(*sys.argv[1:])
