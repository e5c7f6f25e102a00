"""Drop-in replacement for the action model's SMPL layer (``Rotation2xyz``, mld/transforms/rotation2xyz.py), as
``MLD.a2m_eval`` calls it through its two lambdas (mld/models/modeltype/mld.py:119-143):

    from mld_b200.smpl import B200Rotation2xyz as Rotation2xyz        (mld.py:3)

``jointstype='smpl'`` gives the 24 SMPL joints that ``HUMANACTMetrics`` classifies, ``jointstype='vertices'`` the
skinned mesh that ``test_step`` returns as ``joints_rst``.  The math (smplx 0.1.28's ``SMPLLayer`` with zero betas,
then Rotation2xyz's mask, root and translation handling) runs in ``libmldb200.so``.  Only what ``MLD`` calls is
implemented: ``pose_rep='rot6d'`` (``'xyz'`` returns ``x`` as the reference does), ``glob=True``,
``translation=True``, zero betas and no rotations back.  Anything else raises before any GPU work.
"""
from __future__ import annotations

import os
import pickle
from typing import Dict

import numpy as np
import torch

from . import _lib
from .engine import make_config
from .modules import _EngineModule, _register_tree

NUM_JOINTS = 24
_JOINTSTYPES = ("a2m", "a2mpl", "smpl", "vibe", "vertices")     # the reference's JOINTSTYPES
_KEYS = ("v_template", "posedirs", "J_regressor", "lbs_weights", "parents")


def _np(a) -> np.ndarray:
    """A pickled array as numpy: a scipy sparse matrix through ``toarray()``, anything else (numpy, or a chumpy
    ``Ch`` when chumpy is installed) through ``np.asarray``."""
    if hasattr(a, "toarray"):
        a = a.toarray()
    return np.asarray(a)


def _read_pkl(smpl_path: str):
    path = os.path.join(smpl_path, "SMPL_NEUTRAL.pkl") if os.path.isdir(smpl_path) else smpl_path
    with open(path, "rb") as f:
        return pickle.load(f, encoding="latin1")


def _model_of(data) -> Dict[str, torch.Tensor]:
    posedirs = _np(data["posedirs"])
    posedirs = np.reshape(posedirs, [-1, posedirs.shape[-1]]).T
    parents = _np(data["kintree_table"])[0].astype(np.int64)
    parents[0] = -1
    m = {"v_template": _np(data["v_template"]), "posedirs": posedirs, "J_regressor": _np(data["J_regressor"]),
         "lbs_weights": _np(data["weights"])}
    out = {k: torch.tensor(np.array(v, dtype=np.float32)) for k, v in m.items()}
    out["parents"] = torch.from_numpy(parents)
    check_model(out)
    return out


def load_smpl(smpl_path: str) -> Dict[str, torch.Tensor]:
    """The SMPL model the way smplx 0.1.28 reads ``SMPL_NEUTRAL.pkl`` (``smpl_path`` is its directory, as the
    reference's ``SMPL(smpl_path)`` takes it, or the file): ``pickle.load(..., encoding="latin1")``, posedirs
    ``[V, 3, 207]`` reshaped to ``[207, 3 V]``, ``parents = kintree_table[0]`` with ``parents[0] = -1``.  Returns
    float32 ``v_template [V, 3]``, ``posedirs [207, 3 V]``, ``J_regressor [24, V]``, ``lbs_weights [V, 24]`` and int64
    ``parents [24]``: what the layer computes with."""
    return _model_of(_read_pkl(smpl_path))


# smplx 0.1.28's VertexJointSelector for SMPL (vertex_ids["smplh"]): face, feet, then left and right fingertips
_EXTRA_JOINTS_IDXS = (332, 6260, 2800, 4071, 583, 3216, 3226, 3387, 6617, 6624, 6787,
                      2746, 2319, 2445, 2556, 2673, 6191, 5782, 5905, 6016, 6133)
# buffers the reference's SMPL holds that neither joint type MLD uses reads: kept so that a checkpoint of MLD (whose
# rot2xyz.smpl_model.* keys are these and _KEYS) loads strictly and a saved state dict keeps them
_CARRIED = ("shapedirs", "faces_tensor", "J_regressor_extra", "vertex_joint_selector.extra_joints_idxs")


def reference_buffers(smpl_path: str) -> Dict[str, torch.Tensor]:
    """Every persistent buffer of the reference's ``SMPL(smpl_path)`` (smplx 0.1.28's ``SMPLLayer`` plus
    ``J_regressor_extra``), under its names, as that module builds them: ``_KEYS`` from ``load_smpl``,
    ``shapedirs [V, 3, 10]`` (the pickle's first 10 betas), ``faces_tensor`` (the pickle's ``f``, int64),
    ``vertex_joint_selector.extra_joints_idxs [21]`` and ``J_regressor_extra`` from ``J_regressor_extra.npy`` beside
    the pickle ([0, V] when that file is absent; a checkpoint's own then replaces it)."""
    data = _read_pkl(smpl_path)
    out = _model_of(data)
    V = out["v_template"].shape[0]
    shapedirs = _np(data["shapedirs"]) if "shapedirs" in data else np.zeros((V, 3, 10))
    out["shapedirs"] = torch.tensor(np.array(shapedirs[:, :, :10], dtype=np.float32))
    out["faces_tensor"] = torch.tensor(np.array(_np(data["f"]), dtype=np.int64))
    out["vertex_joint_selector.extra_joints_idxs"] = torch.tensor(_EXTRA_JOINTS_IDXS, dtype=torch.int64)
    extra = os.path.join(smpl_path if os.path.isdir(smpl_path) else os.path.dirname(smpl_path), "J_regressor_extra.npy")
    out["J_regressor_extra"] = (torch.tensor(np.load(extra), dtype=torch.float32) if os.path.exists(extra)
                                else torch.zeros(0, V))
    return out


class _SmplBuffers(torch.nn.Module):
    """``smpl_model``: the reference SMPL's buffers.  A state dict's carried buffers (never read here) are taken in
    whatever shape it holds them, so a checkpoint loads even when ``J_regressor_extra.npy`` was absent at
    construction."""

    loads = 0                                          # state loads seen (B200Rotation2xyz rebuilds its engine on a change)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        self.loads += 1
        for name in ("shapedirs", "faces_tensor", "J_regressor_extra"):
            t = state_dict.get(prefix + name)
            if t is not None and t.shape != self._buffers[name].shape:
                self._buffers[name] = torch.empty_like(t, device=self._buffers[name].device)
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)


def check_model(m: Dict[str, torch.Tensor]):
    """The shapes the native layer takes, and a topologically ordered parent table (ValueError otherwise)."""
    V = m["v_template"].shape[0]
    want = {"v_template": (V, 3), "posedirs": (207, 3 * V), "J_regressor": (NUM_JOINTS, V),
            "lbs_weights": (V, NUM_JOINTS), "parents": (NUM_JOINTS,)}
    for k, s in want.items():
        if tuple(m[k].shape) != s:
            raise ValueError(f"SMPL {k} must be {list(s)}, got {list(m[k].shape)}")
    p = [int(x) for x in m["parents"]]
    if p[0] != -1 or any(not 0 <= p[j] < j for j in range(1, NUM_JOINTS)):
        raise ValueError(f"SMPL parents must have parents[0] = -1 and 0 <= parents[j] < j, got {p}")


class B200Rotation2xyz(_EngineModule):
    """``Rotation2xyz(smpl_path)`` (mld/transforms/rotation2xyz.py:10-111) on the native SMPL layer.  The model is
    held as buffers of ``smpl_model`` under the reference SMPL's names, all of them (``reference_buffers``), so an
    action checkpoint's ``rot2xyz.smpl_model.*`` keys load strictly and ``.to(device)`` moves the model.  The five
    that the layer computes with are uploaded to a per-device engine on first use, and again after any load of the
    module's state (its own ``load_state_dict`` or a parent's).
    ``__call__`` takes ``x`` as ``MLD`` passes it, ``sample.view(B, T, 6, 25).permute(0, 3, 2, 1)``, and reads the
    features through that view without a copy (any other layout is made contiguous once).  It returns float32 on
    ``x.device``: ``[B, 24, 3, T]`` for ``'smpl'``, ``[B, V, 3, T]`` for ``'vertices'``."""
    _prefix = "smpl."

    def __init__(self, smpl_path: str):
        super().__init__()
        m = reference_buffers(smpl_path)
        self.smpl_model = _SmplBuffers()
        _register_tree(self.smpl_model, m, buffers=_KEYS + tuple(k.rsplit(".", 1)[-1] for k in _CARRIED))
        cfg = _lib.default_smpl_config()
        cfg.num_vertices = m["v_template"].shape[0]
        self._smpl_cfg = cfg

    def _make_config(self):
        return make_config(num_layers=0, vae="none")

    def _configure_engine(self, eng):
        eng.smpl_configure(self._smpl_cfg)

    def _engine_state_dict(self):
        return {k: getattr(self.smpl_model, k) for k in _KEYS}

    def engine(self):
        if self.smpl_model.loads != getattr(self, "_loads_seen", 0):  # smpl_model's state was loaded on its own
            self._loads_seen = self.smpl_model.loads
            self._weights_epoch += 1
        return super().engine()

    def __call__(self, x, mask, pose_rep, translation, glob, jointstype, vertstrans, betas=None, beta=0,
                 glob_rot=None, get_rotations_back=False, **kwargs):
        if pose_rep == "xyz":
            return x
        if pose_rep != "rot6d":
            raise NotImplementedError(f"pose_rep {pose_rep!r} is not implemented natively (only 'rot6d')")
        if not glob:
            if glob_rot is None:
                raise TypeError("You must specify global rotation if glob is False")
            raise NotImplementedError("glob=False is not implemented natively")
        if jointstype not in _JOINTSTYPES:
            raise NotImplementedError("This jointstype is not implemented.")
        if jointstype not in ("smpl", "vertices"):
            raise NotImplementedError(f"jointstype {jointstype!r} is not implemented natively ('smpl', 'vertices')")
        if not translation:
            raise NotImplementedError("translation=False is not implemented natively")
        if betas is not None or beta != 0:
            raise NotImplementedError("only zero betas are implemented natively")
        if get_rotations_back:
            raise NotImplementedError("get_rotations_back=True is not implemented natively")
        if x.dim() != 4 or x.shape[1] != 25 or x.shape[2] != 6 or x.shape[0] < 1 or x.shape[3] < 1:
            raise ValueError(f"x must be [B >= 1, 25, 6, T >= 1] (rot6d of 24 joints + the translation), "
                             f"got {tuple(x.shape)}")
        B, T = x.shape[0], x.shape[3]
        if mask is not None and (tuple(mask.shape) != (B, T) or mask.dtype != torch.bool):
            raise ValueError(f"mask must be a bool [{B}, {T}] tensor, got {mask.dtype} {tuple(mask.shape)}")
        feats = x.permute(0, 3, 2, 1)                   # [B, T, 6, 25]: MLD's view, contiguous when x is its permute
        if not feats.is_contiguous() or feats.dtype != torch.float32:
            feats = feats.float().contiguous()
        eng = self.engine()
        kind = _lib.SMPL_JOINTS if jointstype == "smpl" else _lib.SMPL_VERTICES
        out = eng.smpl_forward(feats.reshape(B, T, 150), mask, kind, vertstrans)
        return out if out.device == x.device else out.to(x.device)

    forward = __call__
