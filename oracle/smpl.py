"""Float64 restatement of the action model's SMPL layer (TEST INFRASTRUCTURE): smplx 0.1.28's loader, ``lbs`` with
``pose2rot=False``, ``batch_rigid_transform`` and ``vertices2joints``, restated from their definitions for zero betas,
and the glue of the reference's ``Rotation2xyz`` for ``pose_rep='rot6d'``, ``glob=True``, ``translation=True``.

The LBS core here is a restatement of smplx, checked against the reference's own ``Rotation2xyz`` glue through
``tests/golden/smpl.npz`` (``oracle/make_golden_smpl.py`` runs that glue on a stand-in ``smplx`` built from this
file).  It has not been checked against smplx itself, which is not available offline.

``TorchSMPL`` is the fp32 yardstick of ``scripts/bench_smpl.py``: the same computation in plain torch ops.
"""
from __future__ import annotations

import os
import pickle
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def load_model(smpl_path: str, dtype=torch.float64) -> Dict[str, Tensor]:
    """smplx 0.1.28's reading of SMPL_NEUTRAL.pkl (``smpl_path``: the file or its directory), for zero betas."""
    path = os.path.join(smpl_path, "SMPL_NEUTRAL.pkl") if os.path.isdir(smpl_path) else smpl_path
    with open(path, "rb") as f:
        data = pickle.load(f, encoding="latin1")

    def to_np(a):
        if "scipy.sparse" in str(type(a)):
            a = a.todense()
        return np.array(a, dtype=np.float64)
    posedirs = to_np(data["posedirs"])
    posedirs = np.reshape(posedirs, [-1, posedirs.shape[-1]]).T
    parents = torch.tensor(np.array(data["kintree_table"][0])).long()
    parents[0] = -1
    return {"v_template": torch.tensor(to_np(data["v_template"]), dtype=dtype),
            "posedirs": torch.tensor(posedirs, dtype=dtype),
            "J_regressor": torch.tensor(to_np(data["J_regressor"]), dtype=dtype),
            "lbs_weights": torch.tensor(to_np(data["weights"]), dtype=dtype), "parents": parents}


def vertices2joints(J_regressor: Tensor, vertices: Tensor) -> Tensor:
    return torch.einsum("bik,ji->bjk", vertices, J_regressor.to(vertices.dtype))


def batch_rigid_transform(rot_mats: Tensor, joints: Tensor, parents: Tensor):
    """rot_mats [n, J, 3, 3], joints [n, J, 3] -> posed joints [n, J, 3], relative transforms A [n, J, 4, 4]."""
    joints = joints.unsqueeze(-1)
    rel = joints.clone()
    rel[:, 1:] -= joints[:, parents[1:]]
    n, J = rot_mats.shape[:2]
    T = torch.zeros(n, J, 4, 4, dtype=rot_mats.dtype, device=rot_mats.device)
    T[:, :, :3, :3] = rot_mats
    T[:, :, :3, 3:] = rel
    T[:, :, 3, 3] = 1
    chain = [T[:, 0]]
    for i in range(1, J):
        chain.append(chain[int(parents[i])] @ T[:, i])
    transforms = torch.stack(chain, 1)
    posed = transforms[:, :, :3, 3]
    jh = F.pad(joints, [0, 0, 0, 1])
    rel_t = transforms - F.pad(transforms @ jh, [3, 0, 0, 0, 0, 0, 0, 0])
    return posed, rel_t


def lbs(rot_mats: Tensor, m: Dict[str, Tensor]):
    """lbs(zero betas, pose = rot_mats [n, 24, 3, 3], pose2rot=False) -> (vertices [n, V, 3], joints [n, 24, 3])."""
    n = rot_mats.shape[0]
    dt = rot_mats.dtype
    vt = m["v_template"].to(dt)
    J = vertices2joints(m["J_regressor"], vt[None]).expand(n, -1, -1)
    ident = torch.eye(3, dtype=dt, device=rot_mats.device)
    pose_feature = (rot_mats[:, 1:] - ident).reshape(n, -1)
    v_posed = vt + (pose_feature @ m["posedirs"].to(dt)).view(n, -1, 3)
    posed, A = batch_rigid_transform(rot_mats, J, m["parents"])
    W = m["lbs_weights"].to(dt)
    T = (W @ A.reshape(n, A.shape[1], 16)).view(n, -1, 4, 4)
    verts = (T[:, :, :3, :3] @ v_posed.unsqueeze(-1))[..., 0] + T[:, :, :3, 3]
    return verts, posed


def rotation_6d_to_matrix(d6: Tensor) -> Tensor:
    a1, a2 = d6[..., :3], d6[..., 3:]
    b1 = F.normalize(a1, dim=-1)
    b2 = a2 - (b1 * a2).sum(-1, keepdim=True) * b1
    b2 = F.normalize(b2, dim=-1)
    b3 = torch.cross(b1, b2, dim=-1)
    return torch.stack((b1, b2, b3), dim=-2)


def rotation2xyz(m: Dict[str, Tensor], x: Tensor, mask: Optional[Tensor], jointstype: str, vertstrans: bool) -> Tensor:
    """Rotation2xyz(x [B, 25, 6, T], mask, pose_rep='rot6d', translation=True, glob=True, jointstype, vertstrans) in
    x's dtype: [B, 24, 3, T] ('smpl') or [B, V, 3, T] ('vertices')."""
    B, T = x.shape[0], x.shape[-1]
    if mask is None:
        mask = torch.ones(B, T, dtype=torch.bool, device=x.device)
    trans = x[:, -1, :3]
    rots = x[:, :-1].permute(0, 3, 1, 2)
    R = rotation_6d_to_matrix(rots[mask])
    verts, joints = lbs(R, m)
    sel = joints if jointstype == "smpl" else verts
    out = torch.zeros(B, T, sel.shape[1], 3, dtype=x.dtype, device=x.device)
    out[mask] = sel
    out = out.permute(0, 2, 3, 1).contiguous()
    if jointstype == "smpl":
        out = out - out[:, [0]]
    if vertstrans:
        out = out + (trans - trans[:, :, [0]])[:, None]
    return out


class TorchSMPL(torch.nn.Module):
    """The same layer in fp32 eager torch (the benchmark's yardstick): model tensors as buffers."""

    def __init__(self, m: Dict[str, Tensor]):
        super().__init__()
        for k, v in m.items():
            self.register_buffer(k, v.clone() if k == "parents" else v.float().clone())

    def forward(self, x: Tensor, mask: Optional[Tensor], jointstype: str, vertstrans: bool) -> Tensor:
        m = {k: getattr(self, k) for k in ("v_template", "posedirs", "J_regressor", "lbs_weights", "parents")}
        return rotation2xyz(m, x.float(), mask, jointstype, vertstrans)
