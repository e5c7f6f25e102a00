"""APE and AVE of the text-to-motion test: the per-batch work of ``TemosMetric`` (``ComputeMetrics.update``,
mld/models/metrics/compute.py), which ``MLD.allsplit_step`` calls on every test batch of a HumanML3D or KIT config.

``ape_ave_update`` returns the eight increments that ``update`` adds to the metric's states; the Rifke feature
round trip of both joint tensors and the per-sequence norms and variances run as two kernels in ``libmldb200.so``
(``mldb_ape_ave``).  The ``count`` bookkeeping, the torchmetrics states and ``compute()`` stay in the reference.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import _lib
from .engine import Engine, make_config

JOINTSTYPES = {"humanml3d": (_lib.JOINTS_HUMANML3D, 22), "mmm": (_lib.JOINTS_MMM, 21)}
NAMES = ("APE_root", "APE_traj", "APE_pose", "APE_joints", "AVE_root", "AVE_traj", "AVE_pose", "AVE_joints")

_engines: Dict[int, Engine] = {}


def _engine(device: torch.device) -> Engine:
    """One weightless handle per device: the metric needs no weights."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    eng = _engines.get(idx)
    if eng is None:
        eng = _engines[idx] = Engine(make_config(num_layers=0, vae="none"), idx)
    return eng


def _host_lengths(lengths, B: int, T: int) -> torch.Tensor:
    ln = torch.as_tensor(lengths).reshape(-1)
    if ln.is_floating_point() or ln.dtype == torch.bool:
        raise ValueError(f"lengths must be integers, got {ln.dtype}")
    ln = ln.cpu()          # a CUDA tensor costs one copy to the host here; a list or a CPU tensor none
    if ln.numel() != B:
        raise ValueError(f"expected {B} lengths, got {ln.numel()}")
    if int(ln.min()) < 2 or int(ln.max()) > T:
        raise ValueError(f"every length must lie in [2, {T}] (the variance divides by length - 1), "
                         f"got {ln.tolist()}")
    return ln.to(torch.int32)


def ape_ave_update(jts_text: torch.Tensor, jts_ref: torch.Tensor, lengths, *, jointstype: str = "humanml3d",
                   force_in_meter: bool = True) -> Dict[str, torch.Tensor]:
    """The increments of ``ComputeMetrics.update(jts_text, jts_ref, lengths)``: ``APE_root``, ``APE_traj`` (0-dim),
    ``APE_pose`` [J - 1], ``APE_joints`` [J] and the same four ``AVE_*``, float32 on the joints' device.

    ``jts_*`` are [B, T, J, 3] float32 CUDA tensors padded to T (padded frames enter the floor, as in the reference);
    ``lengths`` is a list or tensor of B ints in [2, T].  Anything else raises before any GPU work.  Enqueued on the
    current stream without a host synchronisation."""
    if jointstype not in JOINTSTYPES:
        raise NotImplementedError(f"This jointstype is not implemented: {jointstype!r} (humanml3d or mmm)")
    kind, J = JOINTSTYPES[jointstype]
    for name, t in (("jts_text", jts_text), ("jts_ref", jts_ref)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
            raise ValueError(f"{name} must be a float32 CUDA tensor")
    if jts_text.shape != jts_ref.shape or jts_text.device != jts_ref.device:
        raise ValueError(f"jts_text {tuple(jts_text.shape)} and jts_ref {tuple(jts_ref.shape)} must have the same "
                         "shape and device")
    if jts_text.dim() != 4 or jts_text.shape[0] < 1 or jts_text.shape[3] != 3:
        raise ValueError(f"joints must be [B, T, J, 3], got {tuple(jts_text.shape)}")
    B, T, Jin = jts_text.shape[:3]
    if Jin != J:
        raise ValueError(f"jointstype {jointstype!r} has {J} joints, got J={Jin}")
    ln = _host_lengths(lengths, B, T)
    eng = _engine(jts_text.device)
    ln_dev = ln.pin_memory().to(eng.device, non_blocking=True)
    out = eng.ape_ave(jts_text.contiguous(), jts_ref.contiguous(), ln_dev, kind, force_in_meter)
    sizes = (1, 1, J - 1, J) * 2
    parts = torch.split(out, sizes)
    return {k: (p[0] if n == 1 else p) for k, p, n in zip(NAMES, parts, sizes)}
