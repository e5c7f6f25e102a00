"""Torch restatement of ``ComputeMetrics.update`` (mld/models/metrics/compute.py) with the Rifke feature round trip
(mld/transforms/joints2jfeats/rifke.py, tools.py), in a chosen dtype.  Float64 is the accuracy yardstick of
``mldb_ape_ave``; float32 on CUDA is the eager baseline it is timed against.

It keeps the reference's order of operations where that matters: the floor over every frame of the padded tensor,
the forward direction from the root-removed joints with the full table's indices, ``F.normalize``'s clamp (a zero
``across`` gives forward (0, 0)), the angle through diff / cumsum / minus the first value, the trajectory through
rotate / cumsum / minus the first value, and a per-sequence loop with the variance divided by ``length - 1``.
"""
from __future__ import annotations

from typing import Dict, Sequence

import torch

HUMANML3D = dict(J=22, feet=(8, 11, 7, 10), shoulders=(17, 16), hips=(2, 1), factor=1000.0 * 0.75 / 480.0)
MMM = dict(J=21, feet=(14, 15, 19, 20), shoulders=(5, 8), hips=(11, 16), factor=1000.0)
TABLES = {"humanml3d": HUMANML3D, "mmm": MMM}
NAMES = ("APE_root", "APE_traj", "APE_pose", "APE_joints", "AVE_root", "AVE_traj", "AVE_pose", "AVE_joints")


def _rot(v: torch.Tensor, c: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """Row vectors [..., 2] times [[c, -s], [s, c]]."""
    return torch.stack((v[..., 0] * c + v[..., 1] * s, -v[..., 0] * s + v[..., 1] * c), -1)


def round_trip(joints: torch.Tensor, tab: dict):
    """Rifke forward then the inverse of ``ComputeMetrics.transform``: (joints, local poses, root, trajectory) of
    every frame, before the meter factor and before the padding is removed."""
    x = joints.clone()
    h = x[..., list(tab["feet"]), 1].min(-1).values                      # [B, T]
    lo, hi = h.min(-1).values, h.max(-1).values
    floor = lo - torch.log(0.5 + torch.exp(lo - hi))                     # softmin(h, softness=0.5)
    x[..., 1] = x[..., 1] - floor[:, None, None]
    root = x[..., 0, :].clone()
    root_y, traj = root[..., 1], root[..., [0, 2]]
    p = x[..., 1:, :].clone()
    p[..., [0, 2]] = p[..., [0, 2]] - traj[..., None, :]
    step = torch.diff(traj, dim=-2)
    step = torch.cat((torch.zeros_like(step[..., :1, :]), step), -2)
    (ls, rs), (lh, rh) = tab["shoulders"], tab["hips"]
    across = p[..., rh, :] - p[..., lh, :] + p[..., rs, :] - p[..., ls, :]   # root-removed array, unshifted indices
    fwd = torch.nn.functional.normalize(torch.stack((-across[..., 2], across[..., 0]), -1), dim=-1)
    sn, cs = fwd[..., 0], fwd[..., 1]
    ang = torch.atan2(sn, cs)
    dang = torch.diff(ang, dim=-1)
    rel = torch.cumsum(torch.cat((torch.zeros_like(dang[..., :1]), dang), -1), -1)
    rel = rel - rel[..., :1]
    local_xz = _rot(p[..., [0, 2]], cs[..., None], -sn[..., None])      # inverse rotation
    local = torch.stack((local_xz[..., 0], p[..., 1], local_xz[..., 1]), -1)
    step_local = _rot(step, cs, -sn)
    C, S = torch.cos(rel), torch.sin(rel)
    xz = _rot(local[..., [0, 2]], C[..., None], S[..., None])
    traj_r = torch.cumsum(_rot(step_local, C, S), -2)
    traj_r = traj_r - traj_r[..., :1, :]
    jts = torch.cat((torch.zeros_like(local[..., :1, :]),
                     torch.stack((xz[..., 0], local[..., 1], xz[..., 1]), -1)), -2)
    jts[..., 0, 1] = root_y
    jts[..., [0, 2]] = jts[..., [0, 2]] + traj_r[..., None, :]
    root_r = torch.stack((traj_r[..., 0], root_y, traj_r[..., 1]), -1)
    return jts, local, root_r, traj_r


def _var(x: torch.Tensor, n: int) -> torch.Tensor:
    return ((x - x.mean(0)) ** 2).sum(0) / (n - 1)


def ape_ave_update(jts_text: torch.Tensor, jts_ref: torch.Tensor, lengths: Sequence[int], jointstype: str = "humanml3d",
                   force_in_meter: bool = True, dtype: torch.dtype = torch.float64) -> Dict[str, torch.Tensor]:
    """The eight increments of ``ComputeMetrics.update``, computed in ``dtype`` on the inputs' device."""
    tab = TABLES[jointstype]
    J = tab["J"]
    f = tab["factor"] if force_in_meter else 1.0
    a = [t / f for t in round_trip(jts_text.to(dtype), tab)]
    r = [t / f for t in round_trip(jts_ref.to(dtype), tab)]
    z = lambda *s: torch.zeros(s, dtype=dtype, device=jts_text.device)   # noqa: E731
    out = {"APE_root": z(), "APE_traj": z(), "APE_pose": z(J - 1), "APE_joints": z(J),
           "AVE_root": z(), "AVE_traj": z(), "AVE_pose": z(J - 1), "AVE_joints": z(J)}
    dist = lambda u, v, dim: torch.linalg.vector_norm(u - v, ord=2, dim=dim)   # noqa: E731
    for i, n in enumerate(int(v) for v in lengths):
        (ja, pa, ra, ta), (jr, pr, rr, tr) = ([t[i, :n] for t in a]), ([t[i, :n] for t in r])
        out["APE_root"] += dist(ra, rr, 1).sum()
        out["APE_pose"] += dist(pa, pr, 2).sum(0)
        out["APE_traj"] += dist(ta, tr, 1).sum()
        out["APE_joints"] += dist(ja, jr, 2).sum(0)
        out["AVE_root"] += dist(_var(ra, n), _var(rr, n), 0)
        out["AVE_traj"] += dist(_var(ta, n), _var(tr, n), 0)
        out["AVE_pose"] += dist(_var(pa, n), _var(pr, n), 1)
        out["AVE_joints"] += dist(_var(ja, n), _var(jr, n), 1)
    return out


def synth_joints(B: int, T: int, jointstype: str = "humanml3d", seed: int = 0, lengths: Sequence[int] = (),
                 zero_across: Sequence[tuple] = ()):
    """Seeded smooth test motions [B, T, J, 3] float32 in meters: a skeleton that walks, turns and bobs, each joint
    swinging a little.  Frames at and past ``lengths[b]`` hold a different motion (lower, shaking), so that they
    move the floor.  ``zero_across`` lists (b, t) frames whose shoulders and hips are put on top of each other, so
    that their ``across`` vector is exactly zero."""
    tab = TABLES[jointstype]
    J = tab["J"]
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(s, generator=g, dtype=torch.float64)   # noqa: E731
    off = (rnd(B, 1, J, 3) - 0.5) * torch.tensor([0.8, 1.6, 0.5], dtype=torch.float64)
    off[..., 0, :] = 0.0
    off[..., list(tab["feet"]), 1] = -0.85 - 0.1 * rnd(B, 1, 4)
    t = torch.arange(T, dtype=torch.float64)[None, :]
    turn = 3.0 * (rnd(B, 1) - 0.5) / T
    head = 2 * torch.pi * rnd(B, 1) + turn * t + 0.2 * torch.sin(t / 7.0 + rnd(B, 1) * 6)
    speed = 0.02 + 0.03 * rnd(B, 1)
    pos_x = torch.cumsum(speed * torch.sin(head), 1)
    pos_z = torch.cumsum(speed * torch.cos(head), 1)
    bob = 0.9 + 0.04 * torch.sin(t / 3.0 + rnd(B, 1) * 6)
    wob = 0.05 * torch.sin(t[..., None, None] / (2.0 + 3 * rnd(B, 1, J, 3)) + 6 * rnd(B, 1, J, 3))
    loc = off + wob
    c, s = torch.cos(head)[..., None], torch.sin(head)[..., None]
    x = torch.stack((c * loc[..., 0] + s * loc[..., 2], loc[..., 1], -s * loc[..., 0] + c * loc[..., 2]), -1)
    x = x + torch.stack((pos_x, bob, pos_z), -1)[..., None, :]
    for b, n in enumerate(lengths):
        pad = x[b, n:]
        pad[..., 1] -= 0.3 + 0.2 * torch.rand(pad.shape[:-1], generator=g, dtype=torch.float64)
        pad[..., [0, 2]] += 0.5 * torch.rand(pad.shape[:-1] + (2,), generator=g, dtype=torch.float64)
    x = x.float()
    (ls, rs), (lh, rh) = tab["shoulders"], tab["hips"]
    for b, f in zero_across:                                  # the array the reference reads has the root removed
        x[b, f, rh + 1] = x[b, f, lh + 1]
        x[b, f, rs + 1] = x[b, f, ls + 1]
    return x
