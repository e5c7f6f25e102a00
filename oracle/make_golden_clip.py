"""Generate tests/golden/clip_text.npz with transformers' CLIP text tower (TEST INFRASTRUCTURE).

    python -m oracle.make_golden_clip

``MldTextEncoder`` (mld/models/architectures/mld_clip.py) calls ``get_text_features`` / ``text_model`` of a
transformers CLIP model; ``CLIPTextModelWithProjection`` is the class behind both.  The seeded synthetic weights
of ``mld_b200.synth.clip_text_state_dict`` (full CLIP-L/14 shape) are loaded into it with ``strict=True`` and the
tower is run in fp32 on seeded ids.  Only outputs are stored: weights and ids are rebuilt from the seeds by the
tests; last_hidden_state is kept at the positions HIDDEN_POS only.  transformers 5.x ``get_text_features`` returns an output object, so the pooled output is computed as
``text_projection(text_model(ids).pooler_output)`` - what transformers 4.x ``get_text_features`` returned.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "clip_text.npz")
WEIGHT_SEED = 4242
# last_hidden_state is stored at these positions only (the fixture stays small): bos, every eos position of
# golden_ids() and the position after it, and the last position
HIDDEN_POS = (0, 1, 4, 5, 11, 12, 29, 30, 76)


def golden_ids() -> torch.Tensor:
    """Rows: "" (bos, eos, eos padding), prompts with eos at 4 / 11 / 29, a full 77-token row with eos at 76."""
    from mld_b200 import synth
    rows = [torch.tensor([49406] + [49407] * 76)]
    for k, e in enumerate((4, 11, 29)):
        rows.append(synth.clip_text_ids(1, 77, seed=100 + k, eos_lo=e, eos_hi=e)[0])
    full = synth.clip_text_ids(1, 77, seed=104, eos_lo=76, eos_hi=76)[0]
    rows.append(full)
    return torch.stack(rows)


def load_hf(sd, eos_token_id: int):
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, projection_dim=768,
                         num_hidden_layers=12, num_attention_heads=12, max_position_embeddings=77,
                         hidden_act="quick_gelu", layer_norm_eps=1e-5, bos_token_id=49406, pad_token_id=1,
                         eos_token_id=eos_token_id, attn_implementation="eager")
    m = CLIPTextModelWithProjection(cfg)
    m.load_state_dict({k[len("text_model."):]: v for k, v in sd.items()}, strict=True)
    return m.eval()


def main():
    from mld_b200 import synth
    torch.set_grad_enabled(False)
    sd = synth.clip_text_state_dict(WEIGHT_SEED)
    ids = golden_ids()
    out = {}
    for tag, eos in (("", 49407), ("_legacy", 2)):
        m = load_hf(sd, eos)
        o = m.text_model(input_ids=ids)
        if not tag:
            out["hidden"] = o.last_hidden_state[:, list(HIDDEN_POS)].numpy()
            out["hidden_pos"] = np.array(HIDDEN_POS, dtype=np.int64)
        out["pooled" + tag] = m.text_projection(o.pooler_output).numpy()
    from oracle.clip_text import ClipTextCfg, clip_text_forward
    ref = clip_text_forward(sd, ids, "clip_hidden", ClipTextCfg())[:, list(HIDDEN_POS)]
    print(f"oracle vs transformers, hidden: max abs {float((ref - torch.from_numpy(out['hidden'])).abs().max()):.3e}")
    np.savez(OUT, **out)
    print("written", OUT)


if __name__ == "__main__":
    main()
