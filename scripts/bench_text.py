"""Benchmark of the native CLIP text encoder on one GPU (synthetic CLIP ViT-L/14 weights).

    python scripts/bench_text.py [--out DIR] [--iters N] [--warmup W]

Times with CUDA events after warm-up:
  * the text tower alone on 2B = 512 prompts (B uncond "" rows + B prompts with eos at seeded positions 8..30),
    in both modes, through mldb_text_encode on all rows ("plain") and through B200TextEncoder.encode_ids with
    the two host-side savings (distinct rows once, clip mode truncated after the last eos) ("savings");
  * the same request through the fp32 eager torch restatement (oracle/clip_text.py) on the same GPU;
  * text ids -> joints at B = 256, 50 DDIM steps: encode_ids, then the sampling path (mldb_sample), for clip
    (S_ctx = 1) and clip_hidden (S_ctx = 77).
TFLOP/s are algorithmic: FLOPs of the full request (every row, all 77 positions, causal attention counted per
key actually attended) computed from shapes here, divided by the measured time.  Prints the GPU name, power
limit and SM clock of the same run, one JSON line, and writes it to DIR/bench_text.json.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [s.strip() for s in q.split(",")]
    except Exception as exc:                                            # not fatal: the numbers still stand
        info["nvidia_smi"] = f"unavailable ({exc})"
    return info


def tower_flops(n, L, c, pooled):
    """Forward FLOPs of the text tower on n rows of L tokens (2 per multiply-add)."""
    d, ff = c.hidden, c.ff
    per_tok = 2 * d * 3 * d + 2 * d * d + 2 * 2 * d * ff             # qkv, out-projection, fc1 + fc2
    attn = 2 * 2 * d * (L * (L + 1) // 2)                              # QK^T and PV over the causal keys
    f = c.layers * (n * L * per_tok + n * attn)
    return f + (2 * d * c.projection_dim * n if pooled else 0)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters + 1)]
    ev[0].record()
    for i in range(iters):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ms = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(iters))
    return ms[len(ms) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="bench_text_out")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--B", type=int, default=256)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from mld_b200 import synth
    from mld_b200.pipeline import B200MLD
    from mld_b200.text import B200TextEncoder, ClipTextConfig, plan_ids
    from oracle.clip_text import ClipTextCfg, clip_text_forward
    torch.set_grad_enabled(False)
    torch.cuda.set_device(0)
    res = {"bench": "clip_text", **gpu_info()}
    B, L = args.B, 77
    c = ClipTextConfig()
    sd = synth.clip_text_state_dict(4242)
    ids = torch.cat([torch.tensor([[49406] + [49407] * 76] * B), synth.clip_text_ids(B, L, seed=11, eos_lo=8, eos_hi=30)])
    enc = B200TextEncoder.from_state_dict(sd).cuda()
    eng = enc.engine()
    d_ids = ids.cuda()
    from mld_b200 import _lib
    for name, pooled in (("clip", True), ("clip_hidden", False)):
        mode = _lib.TEXT_POOLED if pooled else _lib.TEXT_HIDDEN
        flops = tower_flops(2 * B, L, c, pooled)
        ms_plain = timed(lambda: eng.text_encode(d_ids, mode), args.iters, args.warmup)
        enc.name = name
        ms_sav = timed(lambda: enc.encode_ids(ids), args.iters, args.warmup)
        rows, _ = plan_ids(ids, pooled, c.eos_token_id)
        res[f"tower_{name}"] = {
            "rows": 2 * B, "L": L, "tflop": flops / 1e12,
            "plain_ms": ms_plain, "plain_tflops": flops / ms_plain / 1e9,
            "savings_ms": ms_sav, "savings_rows": int(rows.shape[0]), "savings_L": int(rows.shape[1]),
            "savings_effective_tflops": flops / ms_sav / 1e9,
            "savings_executed_tflops": tower_flops(rows.shape[0], rows.shape[1], c, pooled) / ms_sav / 1e9,
        }
    sd32 = {k: v.cuda() for k, v in sd.items()}
    torch.backends.cuda.matmul.allow_tf32 = False
    for name in ("clip", "clip_hidden"):
        ms = timed(lambda: clip_text_forward(sd32, d_ids, name, ClipTextCfg(), dtype=torch.float32), 3, 1)
        res[f"tower_{name}"]["torch_fp32_eager_ms"] = ms
        res[f"tower_{name}"]["torch_fp32_eager_tflops"] = res[f"tower_{name}"]["tflop"] / ms * 1e3
    del sd32
    # text ids -> joints at B, 50 DDIM steps
    dsd, vsd = synth.denoiser_state_dict(1234), synth.mld_vae_state_dict(4321)
    mean, std = synth.mean_std()
    mld = B200MLD(dsd, vsd, mean=mean, std=std, text_encoder=enc)
    noise = synth.init_noise(B, seed=2).cuda()
    lengths = [196] * B
    for name in ("clip", "clip_hidden"):
        enc.name = name

        def e2e():
            ctx = enc.encode_ids(ids)
            return mld.engine.sample(ctx, noise, lengths, want=("joints",))

        ms = timed(e2e, max(3, args.iters // 3), 1)
        ms_enc = timed(lambda: enc.encode_ids(ids), args.iters, 1)
        res[f"e2e_{name}"] = {"B": B, "steps": 50, "S_ctx": 1 if name == "clip" else L, "ms": ms,
                              "text_ms": ms_enc, "motions_per_s": B / ms * 1e3}
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_text.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
