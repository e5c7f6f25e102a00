"""Batch-sharded sampling across the GPUs of one box (SURVEY.md section 8e).

Every motion is independent (attention is per sequence, LayerNorm per token, classifier-free
guidance pairs rows i and i+B of the same motion), so the path shards with no per-step
communication: each rank samples a contiguous slice of the batch with replicated weights and
ONE all-gather of the finished motions closes the step.  ``torch.distributed`` (NCCL over
NVLink on GPUs, gloo in the CPU tests) is the plumbing.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous slice [lo, hi) of ``total`` items owned by ``rank`` (first ranks get the extras)."""
    base, extra = divmod(total, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_cfg_condition(cond: torch.Tensor, B: int, lo: int, hi: int, cfg_on: bool) -> torch.Tensor:
    """Slice a [2B, ...] uncond-first condition tensor so that both CFG halves of each motion
    stay on the same rank (mld.py:225-230,340)."""
    if not cfg_on:
        return cond[lo:hi]
    return torch.cat([cond[lo:hi], cond[B + lo:B + hi]], 0)


def sample_sharded(run_local: Callable[[torch.Tensor, torch.Tensor, Sequence[int]], torch.Tensor],
                   cond: torch.Tensor, init_noise: torch.Tensor, lengths: Sequence[int], cfg_on: bool = True,
                   group=None, step_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Run ``run_local(cond_slice, noise_slice, lengths_slice) -> [b_local, T_local, ...]`` on this
    rank's slice of the GLOBAL batch and all-gather the padded results into ``[B, T_max, ...]``.
    With ``step_noise`` (the GLOBAL per-step draws [n_steps, B, ...] of a stochastic scheduler) ``run_local``
    gets this rank's slice ``step_noise[:, lo:hi]`` as a fourth argument.
    The gathered tensor is identical to a single-rank run on the whole batch."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    B = init_noise.shape[0]
    T_max = int(max(lengths))
    lo, hi = shard_range(B, rank, world)
    args = (shard_cfg_condition(cond, B, lo, hi, cfg_on), init_noise[lo:hi], list(lengths[lo:hi]))
    if step_noise is not None:
        args += (step_noise[:, lo:hi],)
    local = run_local(*args)
    if local.shape[1] < T_max:                      # reference pads to max(lengths) per batch
        pad = torch.zeros((local.shape[0], T_max - local.shape[1], *local.shape[2:]), dtype=local.dtype,
                          device=local.device)
        local = torch.cat([local, pad], 1)
    if world == 1:
        return local
    counts = [shard_range(B, r, world) for r in range(world)]
    cmax = max(c[1] - c[0] for c in counts)
    if local.shape[0] < cmax:                       # uneven split: pad to the largest shard
        pad = torch.zeros((cmax - local.shape[0], *local.shape[1:]), dtype=local.dtype, device=local.device)
        local = torch.cat([local, pad], 0)
    out = torch.empty((world * cmax, *local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous(), group=group)          # the one collective
    if world * cmax == B:
        return out
    return torch.cat([out[r * cmax: r * cmax + (c[1] - c[0])] for r, c in enumerate(counts)], 0)


def sample_sharded_engine(engine, cond: torch.Tensor, init_noise: torch.Tensor, lengths: Sequence[int],
                          group=None, step_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The product multi-GPU path: this rank's contiguous shard of the GLOBAL batch through
    ``Engine.sample_gather`` (C ABI: k_feats2joints writes into this rank's slot of the gathered buffer, one
    in-place ncclAllGather on a side stream).  The engine must have a communicator (``engine.comm_init``).
    ``step_noise`` is the GLOBAL per-step draw [n_steps, B, n_lat, d] of a stochastic scheduler (every rank
    passes the same tensor); each rank feeds its own columns ``[:, lo:hi]``.
    Returns joints ``[B, T_max, J, 3]`` identical on every rank and bit-identical to a single-GPU run on the
    whole batch.  The batch must split evenly (the reference's loaders drop the last partial batch)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    B = init_noise.shape[0]
    if B % world:
        raise ValueError(f"batch {B} does not split evenly over {world} ranks; use sample_sharded for ragged splits")
    lo, hi = shard_range(B, rank, world)
    return engine.sample_gather(shard_cfg_condition(cond, B, lo, hi, engine.cfg_on), init_noise[lo:hi],
                                list(lengths[lo:hi]), T=int(max(lengths)),
                                step_noise=None if step_noise is None else step_noise[:, lo:hi])
