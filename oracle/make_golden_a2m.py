"""Generate tests/golden/a2m_gru.npz with the reference's own HumanAct12 classifier modules (TEST INFRASTRUCTURE).

    python -m oracle.make_golden_a2m REFERENCE_ROOT      (or MLD_REFERENCE=REFERENCE_ROOT python -m ...)

``MotionDiscriminator`` and ``MotionDiscriminatorForFID`` (mld/models/architectures/humanact12_gru.py; torch only) are
imported from the reference tree, loaded with the seeded ``mld_b200.synth.a2m_state_dict`` under ``strict=True`` and
run in fp32 on the CPU, the way ``HUMANACTMetrics.update`` calls them.  Two cases:
  - ``explicit``: ragged lengths including 1 and T with an explicit ``hidden_unit``;
  - ``seeded``: no ``hidden_unit`` after ``torch.manual_seed(RNG_SEED)``, logits then features (two draws), which pins
    the initial-state draw.
Only outputs and the key/shape list are stored; weights and inputs are rebuilt from the seeds by the tests.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "a2m_gru.npz")
WEIGHT_SEED, RNG_SEED = 1357, 4321
T = 60
EXPLICIT_LENS = (60, 1, 37, 60, 2, 59)
SEEDED_LENS = (60, 60, 60, 45)


def golden_inputs():
    """(x_explicit, h0_explicit, x_seeded), rebuilt from seeds."""
    from mld_b200 import synth
    x1 = synth.a2m_motions(len(EXPLICIT_LENS), T, seed=31)
    h0 = torch.randn(synth.A2M_DIMS["hidden_layer"], len(EXPLICIT_LENS), synth.A2M_DIMS["hidden_size"],
                     generator=torch.Generator().manual_seed(32))
    x2 = synth.a2m_motions(len(SEEDED_LENS), T, seed=33)
    return x1, h0, x2


def key_list(sd):
    return np.array(sorted(f"{k}:{'x'.join(map(str, v.shape))}" for k, v in sd.items()))


def main(ref_root: str = ""):
    ref_root = ref_root or os.environ.get("MLD_REFERENCE", "")
    if not ref_root:
        raise SystemExit("give the reference checkout (ChenFengYe/motion-latent-diffusion) as an argument or MLD_REFERENCE")
    sys.path.insert(0, ref_root)
    from mld.models.architectures import humanact12_gru
    from mld_b200 import synth
    sd = synth.a2m_state_dict(WEIGHT_SEED)
    cls = humanact12_gru.MotionDiscriminator(**synth.A2M_DIMS)
    fid = humanact12_gru.MotionDiscriminatorForFID(**synth.A2M_DIMS)
    for m in (cls, fid):
        m.load_state_dict(sd, strict=True)
        m.eval()
    x1, h0, x2 = golden_inputs()
    with torch.no_grad():
        l1 = torch.tensor(EXPLICIT_LENS)
        logits1, feats1 = cls(x1, lengths=l1, hidden_unit=h0), fid(x1, lengths=l1, hidden_unit=h0)
        l2 = torch.tensor(SEEDED_LENS)
        torch.manual_seed(RNG_SEED)
        logits2, feats2 = cls(x2, lengths=l2), fid(x2, lengths=l2)
    np.savez_compressed(OUT, keys=key_list(sd), logits_explicit=logits1.numpy(), features_explicit=feats1.numpy(),
                        logits_seeded=logits2.numpy(), features_seeded=feats2.numpy())
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main(*sys.argv[1:])
