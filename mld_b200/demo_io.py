"""The output contract of the reference's ``demo.py`` (demo.py:161-218), so that the CLI stays a drop-in:

* per sample ``{task}_{length}_batch{id}_{i}.npy`` holding the joints ``(nframe, 22, 3)`` float32 and a
  sibling ``.txt`` with the prompt (demo.py:186-193);
* with ``DEMO.OUTALL`` one ``{task}_{length}_all.npy`` of shape ``[n_samples, n_rep, nframes, 22, 3]`` (all
  lengths equal, else the reference raises) and a ``.txt`` with every prompt of every replication, one per line
  (demo.py:195-214).

What is H100-native here is how the joints reach the host: :class:`PinnedJointsReader` copies each finished batch
device -> pinned host memory on a side stream and hands the file writing to the caller while the NEXT
replication is already sampling, instead of the reference's synchronous ``.cpu()`` per motion.
"""
from __future__ import annotations

import os
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch


def sample_paths(output_dir: str, task: str, lengths: Sequence[int], batch_id: int = 0) -> List[str]:
    """demo.py:186-187 - note the reference keeps ``id = 0`` for every replication (files are overwritten)."""
    return [os.path.join(str(output_dir), f"{task}_{lengths[i]}_batch{batch_id}_{i}.npy") for i in range(len(lengths))]


def write_samples(output_dir: str, task: str, texts: Sequence[str], lengths: Sequence[int],
                  joints: Sequence[torch.Tensor], batch_id: int = 0) -> List[str]:
    """One ``.npy`` (``(nframe, 22, 3)``) + one ``.txt`` per sample (demo.py:185-193)."""
    paths = sample_paths(output_dir, task, lengths, batch_id)
    for i, npypath in enumerate(paths):
        with open(npypath.replace(".npy", ".txt"), "w") as text_file:
            text_file.write(texts[i])
        j = joints[i]
        np.save(npypath, j.detach().cpu().numpy() if torch.is_tensor(j) else np.asarray(j))
    return paths


def write_allinone(output_dir: str, task: str, lengths: Sequence[int], rep_lst: Sequence[Sequence[torch.Tensor]],
                   texts_lst: Sequence[Sequence[str]]) -> str:
    """``[n_samples, n_rep, nframes, 22, 3]`` (demo.py:199-214).  Raises ``ValueError`` like the reference when the
    motions have different lengths."""
    nsample = len(rep_lst[0])
    try:
        grouped = [torch.cat([torch.as_tensor(r[n])[None] for r in rep_lst], dim=0)[None] for n in range(nsample)]
        combined = torch.cat(grouped, dim=0)
    except RuntimeError as e:
        raise ValueError("Lengths of motions are different, so we cannot save all motions in one file.") from e
    # the reference names the file after the LAST sample's length (its loop variable leaks: demo.py:203)
    npypath = os.path.join(str(output_dir), f"{task}_{lengths[nsample - 1]}_all.npy")
    np.save(npypath, combined.detach().cpu().numpy())
    with open(npypath.replace("npy", "txt"), "w") as text_file:
        for texts in texts_lst:
            for text in texts:
                text_file.write(text)
                text_file.write("\n")
    return npypath


class PinnedJointsReader:
    """Asynchronous device -> host path for finished joints: ``fetch`` enqueues the copy of a ``[B, T, J, 3]``
    device tensor into pinned memory on a side stream (after the producing stream's work) and returns a
    handle; ``handle()`` waits for THAT copy only and returns per-sample views ``[len_i, J, 3]``
    (``remove_padding``, temos_utils.py:24-28).  Two pinned buffers alternate, so one batch can be written to
    disk while the next one is copied / sampled."""

    def __init__(self, device: torch.device, nbuf: int = 2):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device)
        self._bufs: List[Optional[torch.Tensor]] = [None] * nbuf
        self._events = [torch.cuda.Event() for _ in range(nbuf)]
        self._busy = [False] * nbuf
        self._k = 0

    def fetch(self, joints: torch.Tensor, lengths: Sequence[int]) -> Callable[[], List[torch.Tensor]]:
        k = self._k % len(self._bufs)
        self._k += 1
        if self._busy[k]:
            self._events[k].synchronize()                      # the buffer's previous copy (two fetches ago)
        if self._bufs[k] is None or self._bufs[k].shape != joints.shape:
            self._bufs[k] = torch.empty(joints.shape, dtype=joints.dtype).pin_memory()
        host = self._bufs[k]
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            host.copy_(joints, non_blocking=True)
            joints.record_stream(self.stream)
            self._events[k].record(self.stream)
        self._busy[k] = True
        lens = list(lengths)

        def result() -> List[torch.Tensor]:
            self._events[k].synchronize()
            return [host[i, :n] for i, n in enumerate(lens)]
        return result


def run_demo(sample_joints: Callable[[int], torch.Tensor], texts: Sequence[str], lengths: Sequence[int],
             output_dir: str, task: str = "Example", replication: int = 1, outall: bool = False,
             device: Optional[torch.device] = None) -> List[str]:
    """The sampling loop of demo.py:161-214 around any ``sample_joints(rep) -> [B, T, J, 3]`` DEVICE tensor
    (e.g. ``lambda rep: engine.sample(ctx, noise[rep], lengths)["joints"]``): replication ``r + 1`` is enqueued
    before the files of replication ``r`` are written, the joints travel through pinned memory on a side
    stream.  Returns the written ``.npy`` paths."""
    os.makedirs(str(output_dir), exist_ok=True)
    written: List[str] = []
    rep_lst, texts_lst = [], []
    reader = None
    pending = None
    for rep in range(replication):
        joints_dev = sample_joints(rep)
        if reader is None:
            reader = PinnedJointsReader(joints_dev.device if device is None else device)
        nxt = reader.fetch(joints_dev, lengths)
        if pending is not None:
            written += _flush(pending, output_dir, task, texts, lengths, rep_lst, texts_lst, outall)
        pending = nxt
    if pending is not None:
        written += _flush(pending, output_dir, task, texts, lengths, rep_lst, texts_lst, outall)
    if outall and rep_lst:
        written.append(write_allinone(output_dir, task, lengths, rep_lst, texts_lst))
    return written


def _flush(pending, output_dir, task, texts, lengths, rep_lst, texts_lst, outall):
    joints = pending()
    paths = write_samples(output_dir, task, texts, lengths, joints)
    if outall:
        rep_lst.append([j.clone() for j in joints])       # the pinned buffer is reused two fetches later
        texts_lst.append(list(texts))
    return paths
