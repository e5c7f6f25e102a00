"""Generate tests/golden/t2m_eval.npz with the reference's own T2M evaluator modules (TEST INFRASTRUCTURE).

    python -m oracle.make_golden_t2m REFERENCE_ROOT      (or MLD_REFERENCE=REFERENCE_ROOT python -m ...)

``TextEncoderBiGRUCo``, ``MovementConvEncoder`` and ``MotionEncoderBiGRUCo`` (mld/models/architectures/
t2m_textenc.py, t2m_motionenc.py; torch only) are imported from the reference tree, loaded with the seeded
``mld_b200.synth.t2m_state_dicts`` under ``strict=True`` and run in fp32 on the CPU, in eval mode, the way
``MLD.t2m_eval`` calls them (mld.py:675-697).  Only outputs and the key/shape list are stored; weights and inputs
are rebuilt from the seeds by the tests.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "t2m_eval.npz")
WEIGHT_SEED = 2468
TEXT_B, TEXT_L, TEXT_LENS = 4, 22, (22, 15, 7, 1)
MOTION_T, MOTION_LENS = 196, (196, 120, 64, 16)     # sorted as t2m_eval sorts them (align_idx)
MOVE_HEAD = 4                                       # movement-encoder output steps stored per sequence


def key_list(sds):
    return np.array(sorted(f"{part}/{k}:{'x'.join(map(str, v.shape))}" for part, sd in sds.items() for k, v in sd.items()))


def golden_inputs():
    """The fixture's inputs, rebuilt from seeds: text word vectors / POS one-hots and the renormed motion feats."""
    from mld_b200 import synth
    word, pos = synth.t2m_text_inputs(TEXT_B, TEXT_L, seed=11)
    feats = synth.t2m_feats(len(MOTION_LENS), MOTION_T, list(MOTION_LENS), seed=12)
    mean, std = synth.mean_std()
    mean_eval, std_eval = synth.t2m_mean_std()
    return word, pos, synth.renorm4t2m(feats, mean, std, mean_eval, std_eval)


def main(ref_root: str = ""):
    ref_root = ref_root or os.environ.get("MLD_REFERENCE", "")
    if not ref_root:
        raise SystemExit("give the reference checkout (ChenFengYe/motion-latent-diffusion) as an argument or MLD_REFERENCE")
    sys.path.insert(0, ref_root)
    from mld.models.architectures import t2m_motionenc, t2m_textenc
    from mld_b200 import synth
    torch.backends.cudnn.allow_tf32 = False
    sds = synth.t2m_state_dicts(WEIGHT_SEED)
    d = synth.T2M_DIMS
    te = t2m_textenc.TextEncoderBiGRUCo(d["dim_word"], d["dim_pos_ohot"], d["dim_text_hidden"], d["dim_coemb_hidden"])
    mv = t2m_motionenc.MovementConvEncoder(d["dim_pose"], d["dim_move_hidden"], d["dim_move_latent"])
    mo = t2m_motionenc.MotionEncoderBiGRUCo(d["dim_move_latent"], d["dim_motion_hidden"], d["dim_motion_latent"])
    for m, k in ((te, "text_encoder"), (mv, "movement_encoder"), (mo, "motion_encoder")):
        m.load_state_dict(sds[k], strict=True)
        m.eval()
    word, pos, motions = golden_inputs()
    with torch.no_grad():
        text_emb = te(word, pos, torch.tensor(TEXT_LENS))
        mov = mv(motions[..., :-4])
        motion_emb = mo(mov, torch.div(torch.tensor(MOTION_LENS), 4, rounding_mode="floor"))
    np.savez_compressed(OUT, keys=key_list(sds), text_emb=text_emb.numpy(), movement_head=mov[:, :MOVE_HEAD].numpy(),
                        motion_emb=motion_emb.numpy())
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main(*sys.argv[1:])
