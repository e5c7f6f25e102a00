"""Generate tests/golden/ape_ave.npz with the reference's own ComputeMetrics.update (TEST INFRASTRUCTURE).

    python -m oracle.make_golden_ape_ave REFERENCE_ROOT      (or MLD_REFERENCE=REFERENCE_ROOT python -m ...)

torchmetrics is not installed, so a stand-in with a minimal ``Metric`` (``add_state`` only) goes into ``sys.modules``.
The reference's ``compute.py``, ``rifke.py``, ``joints2jfeats/tools.py`` and ``base.py`` (with the small modules they
import: ``mld/utils/joints.py``, ``geometry.py``, ``rotation_conversions.py``, ``models/tools/tools.py``, ``models/metrics/utils.py``) are loaded
by path under stand-in packages, so no package ``__init__`` that needs smplx is imported.  The metric then runs
``update`` once per case, in float64 (states created in float64) and in float32, and the states are stored as the
increments.  Cases: both joint types, ``force_in_meter`` True and False, B = 8 with lengths 2 and T among them,
padded frames that hold a different motion, and one valid frame whose ``across`` vector is zero.
"""
from __future__ import annotations

import importlib.util
import os
import sys
import types
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "ape_ave.npz")
T = 40
LENGTHS = (40, 2, 17, 33, 25, 40, 9, 31)
ZERO_ACROSS = ((2, 5),)             # (sequence, valid frame) with across == 0
SEEDS = {"humanml3d": (11, 12), "mmm": (21, 22)}


def case_inputs(jointstype):
    from oracle.ape_ave import synth_joints
    st, sr = SEEDS[jointstype]
    text = synth_joints(len(LENGTHS), T, jointstype, st, LENGTHS, ZERO_ACROSS)
    ref = synth_joints(len(LENGTHS), T, jointstype, sr, LENGTHS)
    return text, ref


def _install(ref_root):
    tm = types.ModuleType("torchmetrics")

    class Metric(torch.nn.Module):
        def __init__(self, dist_sync_on_step=False, **kwargs):
            super().__init__()

        def add_state(self, name, default, dist_reduce_fx=None):
            setattr(self, name, default.clone())

    tm.Metric = Metric
    sys.modules["torchmetrics"] = tm
    for pkg in ("mld", "mld.utils", "mld.models", "mld.models.tools", "mld.models.metrics", "mld.transforms",
                "mld.transforms.joints2jfeats"):
        m = types.ModuleType(pkg)
        m.__path__ = []
        sys.modules[pkg] = m

    def load(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(ref_root, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod

    load("mld.utils.joints", "mld/utils/joints.py")
    load("mld.utils.rotation_conversions", "mld/utils/rotation_conversions.py")
    load("mld.utils.geometry", "mld/utils/geometry.py")
    load("mld.models.tools.tools", "mld/models/tools/tools.py")
    load("mld.models.metrics.utils", "mld/models/metrics/utils.py")
    load("mld.transforms.joints2jfeats.base", "mld/transforms/joints2jfeats/base.py")
    tools = load("mld.transforms.joints2jfeats.tools", "mld/transforms/joints2jfeats/tools.py")
    rifke = load("mld.transforms.joints2jfeats.rifke", "mld/transforms/joints2jfeats/rifke.py")
    sys.modules["mld.transforms.joints2jfeats"].Rifke = rifke.Rifke
    compute = load("mld.models.metrics.compute", "mld/models/metrics/compute.py")
    return tools, compute.ComputeMetrics


def _check_floor(tools):
    """get_floor indexes its [B] result with a list of None (``floor[(ndim - 2) * [None]]``); torch still accepts it
    (with a deprecation warning in some versions).  The fixture is only valid if it still gives [B, 1, 1]."""
    x = torch.randn(3, 5, 22, 3, dtype=torch.float64)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        f = tools.get_floor(x, jointstype="humanml3d")
    h = x[..., (8, 11, 7, 10), 1].min(-1).values
    lo, hi = h.min(-1).values, h.max(-1).values
    assert f.shape == (3, 1, 1), f.shape
    assert torch.equal(f.reshape(3), lo - torch.log(0.5 + torch.exp(lo - hi)))
    print(f"[golden] get_floor's list-of-None indexing works ({len(w)} warning(s): "
          f"{[str(m.message)[:60] for m in w]})")


def main():
    ref_root = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("MLD_REFERENCE", "")
    assert ref_root and os.path.isdir(os.path.join(ref_root, "mld")), "pass the reference's root directory"
    tools, ComputeMetrics = _install(ref_root)
    _check_floor(tools)
    out = {"lengths": np.array(LENGTHS, dtype=np.int64), "zero_across": np.array(ZERO_ACROSS, dtype=np.int64)}
    for jt in ("humanml3d", "mmm"):
        text, ref = case_inputs(jt)
        out[f"{jt}/text"], out[f"{jt}/ref"] = text.numpy(), ref.numpy()
        J = text.shape[2]
        for fim in (True, False):
            for dtype in (torch.float64, torch.float32):
                prev = torch.get_default_dtype()
                torch.set_default_dtype(dtype)                     # the metric's states in the run's dtype
                try:
                    m = ComputeMetrics(njoints=J, jointstype=jt, force_in_meter=fim)
                finally:
                    torch.set_default_dtype(prev)
                m.update(text.to(dtype), ref.to(dtype), list(LENGTHS))
                for k in m.metrics:
                    v = getattr(m, k)
                    assert v.dtype == dtype and bool(torch.isfinite(v).all()), (k, v)
                    out[f"{jt}/{int(fim)}/{str(dtype)[6:]}/{k}"] = v.detach().numpy()
    np.savez_compressed(OUT, **out)
    print(f"[golden] wrote {OUT} ({len(out)} arrays)")


if __name__ == "__main__":
    main()
