"""Generate tests/golden/uestc_stgcn.npz with the reference's own UESTC classifier (TEST INFRASTRUCTURE).

    python -m oracle.make_golden_uestc REFERENCE_ROOT      (or MLD_REFERENCE=REFERENCE_ROOT python -m ...)

``STGCN`` (mld/models/architectures/uestc_stgcn.py; torch, numpy and pickle only) is imported from the reference
tree and built the way ``UESTCMetrics`` builds it (metrics/stgcn.py:32-40), with a temporary ``kintree_table.pkl``
that holds SMPL's parent table.  It loads the seeded ``mld_b200.synth.stgcn_state_dict`` under ``strict=True`` and
runs in fp32 on the CPU on ``synth.uestc_motions`` for each (B, T) in CASES.  Stored: yhat and features per case,
the reference's ``A`` and the key/shape list; weights and inputs are rebuilt from the seeds by the tests.
"""
from __future__ import annotations

import os
import pickle
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "uestc_stgcn.npz")
WEIGHT_SEED = 2025
CASES = ((3, 60, 41), (2, 61, 42), (1, 1, 43))             # (B, T, motion seed)


def key_list(sd):
    return np.array(sorted(f"{k}:{'x'.join(map(str, v.shape))}" for k, v in sd.items()))


def write_kintree(path: str):
    """kintree_table.pkl as the reference's Graph reads it: row 0 the parents (the root's is unused), row 1 the ids."""
    from mld_b200.graph import SMPL_PARENTS
    kt = np.array([[4294967295] + list(SMPL_PARENTS[1:]), list(range(24))], dtype=np.int64)
    with open(path, "wb") as f:
        pickle.dump(kt, f)


def main(ref_root: str = ""):
    ref_root = ref_root or os.environ.get("MLD_REFERENCE", "")
    if not ref_root:
        raise SystemExit("give the reference checkout (ChenFengYe/motion-latent-diffusion) as an argument or MLD_REFERENCE")
    sys.path.insert(0, ref_root)
    from mld.models.architectures import uestc_stgcn
    from mld_b200 import synth
    sd = synth.stgcn_state_dict(WEIGHT_SEED)
    with tempfile.TemporaryDirectory() as d:
        kp = os.path.join(d, "kintree_table.pkl")
        write_kintree(kp)
        net = uestc_stgcn.STGCN(in_channels=6, kintree_path=kp, num_class=40,
                                graph_args={"layout": "smpl", "strategy": "spatial"}, edge_importance_weighting=True)
    A = net.A.clone()
    net.load_state_dict(sd, strict=True)
    net.eval()
    out = {"keys": key_list(net.state_dict()), "A": A.numpy()}
    with torch.no_grad():
        for B, T, seed in CASES:
            o = net(synth.uestc_motions(B, T, seed=seed))
            out[f"yhat_{B}x{T}"] = o["yhat"].numpy()
            out[f"features_{B}x{T}"] = o["features"].reshape(B, -1).numpy()
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main(*sys.argv[1:])
