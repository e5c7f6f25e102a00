"""Generate tests/golden/vae_actor_encode.npz with the reference's own ActorVae (TEST INFRASTRUCTURE).

    python -m oracle.make_golden_actor_encode      (MLD_REFERENCE=<reference checkout>, default /root/reference)

The seeded ``mld_b200.synth.actor_vae_state_dict(777)`` is loaded into the reference ``ActorVae``
(mld/models/architectures/actor_vae.py) with ``strict=True`` and ``ActorVae.encode`` is run in fp32/eval/no_grad on
the two cases of ``CASES``.  Only the distribution's ``loc`` and ``scale`` are stored; weights and motions are
rebuilt from the seeds by the tests.  Case a has 62 keys per sequence, case b has 152 keys and a one-frame sequence.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

REF = os.environ.get("MLD_REFERENCE", "/root/reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "vae_actor_encode.npz")
WEIGHT_SEED = 777
NFEATS, NUM_LAYERS = 150, 6
# tag: (motion seed, T, lengths)
CASES = {"a": (42, 60, (60, 40, 12)), "b": (43, 150, (150, 97, 1))}


def case_motion(tag: str) -> torch.Tensor:
    seed, T, lengths = CASES[tag]
    return torch.randn(len(lengths), T, NFEATS, generator=torch.Generator().manual_seed(seed))


def main():
    from mld_b200 import synth
    from oracle import mld_oracle as O
    from oracle.actor_encode import actor_encode
    from oracle.make_golden import abl
    sys.path.insert(0, REF)
    from mld.models.architectures.actor_vae import ActorVae
    torch.set_grad_enabled(False)
    sd = synth.actor_vae_state_dict(seed=WEIGHT_SEED)
    vae = ActorVae(ablation=abl(), nfeats=NFEATS, latent_dim=[1, 256], ff_size=1024, num_layers=NUM_LAYERS,
                   num_heads=4, dropout=0.1, is_vae=True, activation="gelu", position_embedding="learned")
    vae.load_state_dict(sd, strict=True)
    vae.eval()
    cfg = O.VaeCfg(kind="actor", nfeats=NFEATS, num_layers=NUM_LAYERS)
    out = {}
    for tag, (_, _, lengths) in CASES.items():
        motion = case_motion(tag)
        _, dist = vae.encode(motion, list(lengths))
        mu, logvar = actor_encode(sd, cfg, motion, lengths)
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max())
        print(f"case {tag}: oracle vs reference, mu {rel(mu[0], dist.loc):.2e}, "
              f"std {rel(logvar[0].exp().pow(0.5), dist.scale):.2e} (relative to max)")
        out[f"{tag}_mu"], out[f"{tag}_std"] = dist.loc.numpy(), dist.scale.numpy()
    np.savez(OUT, **out)
    print("written", OUT)


if __name__ == "__main__":
    main()
