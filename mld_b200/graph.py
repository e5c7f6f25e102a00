"""The SMPL skeleton graph of the UESTC action classifier (``Graph(layout="smpl", strategy="spatial")``,
mld/models/architectures/uestc_stgcn.py): the three-partition adjacency ``A [3, 24, 24]`` of ST-GCN's spatial
configuration strategy (Yan et al., 2018, https://arxiv.org/abs/1801.07455), with max_hop = dilation = 1.

The graph is the SMPL kinematic tree plus a self link per joint; the centre is joint 0 (the pelvis).  Hop distances
are only resolved up to max_hop, so every joint more than one hop from the centre is at distance inf, and two such
joints compare equal: this module keeps that convention, because the partition depends on it.
"""
from __future__ import annotations

import pickle

import numpy as np
import torch

NUM_JOINTS = 24
CENTER = 0
# SMPL's kinematic tree: the parent of each joint (joint 0 is the root); the first row of kintree_table.pkl
SMPL_PARENTS = (-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21)


def parents_from_kintree(path: str) -> list:
    """(parent, child) pairs of ``kintree_table.pkl``: a 2 x 24 table of parents (row 0) and joint ids (row 1)."""
    with open(path, "rb") as f:
        kt = pickle.load(f)
    if len(kt) != 2 or len(kt[0]) != NUM_JOINTS or len(kt[1]) != NUM_JOINTS:
        raise ValueError(f"{path}: expected a 2 x {NUM_JOINTS} kintree table (SMPL's 24 joints)")
    return [(int(k), int(kt[1][i + 1])) for i, k in enumerate(kt[0][1:])]


def smpl_edges(parents=SMPL_PARENTS) -> list:
    return [(int(p), j) for j, p in enumerate(parents) if j > 0]


def spatial_adjacency(edges, num_node: int = NUM_JOINTS, center: int = CENTER) -> np.ndarray:
    """float64 ``[3, V, V]``: root (same distance to the centre), centripetal + root at hop 1, centrifugal."""
    adj = np.eye(num_node)
    for i, j in edges:
        adj[i, j] = adj[j, i] = 1.0
    hop = np.full((num_node, num_node), np.inf)
    hop[adj > 0] = 1.0
    hop[np.eye(num_node, dtype=bool)] = 0.0
    deg = adj.sum(0)
    norm = adj / np.where(deg > 0, deg, 1.0)[None, :]          # column-normalised: norm[j, i] = adj[j, i] / deg[i]
    out = []
    for h in (0.0, 1.0):
        root, close, further = (np.zeros((num_node, num_node)) for _ in range(3))
        for i in range(num_node):
            for j in range(num_node):
                if hop[j, i] != h:
                    continue
                dj, di = hop[j, center], hop[i, center]
                if dj == di:
                    root[j, i] = norm[j, i]
                elif dj > di:
                    close[j, i] = norm[j, i]
                else:
                    further[j, i] = norm[j, i]
        if h == 0.0:
            out.append(root)
        else:
            out += [root + close, further]
    return np.stack(out)


def smpl_adjacency(kintree_path: str | None = None) -> torch.Tensor:
    """The classifier's ``A`` buffer (fp32), from ``kintree_table.pkl`` or, without a path, SMPL's parent table."""
    edges = parents_from_kintree(kintree_path) if kintree_path else smpl_edges()
    return torch.tensor(spatial_adjacency(edges), dtype=torch.float32)
