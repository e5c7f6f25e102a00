"""Cost of stochastic DDIM (eta = 1) against the deterministic sampler (eta = 0) at the headline shape.

    python scripts/bench_stochastic.py [--rounds R] [--reps N] [--B 256] [--out DIR]

B = 256 motions, 77-token context, 50 DDIM steps (CFG 7.5), decode 196x263, joints; synthetic seeded weights.
Two legs per setting, alternated eta = 0 / eta = 1 in every round so that both see the same machine state:
  * ``pipeline``: ``B200MLD.forward`` on a precomputed context - for eta = 1 this includes torch's 1 + 50 draws
    of the initial and per-step noise, and the joints' copy to the host (the reference's call surface);
  * ``sample``: ``Engine.sample`` on device tensors with the noise drawn once beforehand (the library alone).
Times are host wall clock around calls that end in a device synchronise; the median of the rounds is reported
as motions/s.  Prints the GPU name and power limit of the same run and one JSON line (also written to
DIR/bench_stochastic.json with --out).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [s.strip() for s in q.split(",")]
    except Exception as exc:                                            # not fatal: the timings still stand
        info["nvidia_smi"] = f"unavailable ({exc})"
    return info


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--B", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from mld_b200 import synth
    from mld_b200.pipeline import B200MLD
    torch.set_grad_enabled(False)
    torch.cuda.set_device(0)
    B, S, steps = args.B, 77, 50
    dsd, vsd = synth.denoiser_state_dict(1234), synth.mld_vae_state_dict(4321)
    mean, std = synth.mean_std()
    models = {eta: B200MLD(dsd, vsd, mean=mean, std=std, eta=eta, num_inference_timesteps=steps) for eta in (0.0, 1.0)}
    ctx = synth.text_context(B, S, seed=1).cuda()
    lengths = [196] * B
    batch = {"length": lengths, "text_emb": ctx}
    noise = synth.init_noise(B, seed=2).cuda()
    step_noise = torch.randn(steps, B, 1, 256, generator=torch.Generator().manual_seed(3)).cuda()
    legs = {}
    for eta, m in models.items():
        sn = step_noise if eta > 0 else None
        legs[("pipeline", eta)] = lambda m=m: m(batch)
        legs[("sample", eta)] = lambda m=m, sn=sn: m.engine.sample(ctx, noise, lengths, want=("joints",), step_noise=sn)
    for fn in legs.values():                                            # capture the graphs, warm the allocator
        timed(fn, 2)
    times = {k: [] for k in legs}
    for _ in range(args.rounds):
        for leg in ("pipeline", "sample"):
            for eta in (0.0, 1.0):
                times[(leg, eta)].append(timed(legs[(leg, eta)], args.reps))
    res = {"bench": "stochastic_ddim", **gpu_info(), "B": B, "S_ctx": S, "steps": steps, "T": 196,
           "rounds": args.rounds, "reps": args.reps}
    for leg in ("pipeline", "sample"):
        mps = {eta: B / statistics.median(times[(leg, eta)]) for eta in (0.0, 1.0)}
        spread = {eta: [round(B / t, 1) for t in times[(leg, eta)]] for eta in (0.0, 1.0)}
        res[leg] = {"eta0_motions_per_s": mps[0.0], "eta1_motions_per_s": mps[1.0],
                    "eta1_over_eta0": mps[1.0] / mps[0.0], "eta0_rounds": spread[0.0], "eta1_rounds": spread[1.0]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_stochastic.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
