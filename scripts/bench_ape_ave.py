"""Time one APE / AVE update (TemosMetric, ComputeMetrics.update) natively and as the eager float32 loop.

    python scripts/bench_ape_ave.py [--sizes 32,1024] [--rounds 7] [--out FILE.json]

For each batch size B (T = 196, ragged lengths 40..196 as in a HumanML3D eval batch) one round times the native
``ape_ave_update`` and the float32 restatement of the reference's update loop (oracle/ape_ave.py, the same per-sequence
loop in torch) on the same inputs, one after the other; the JSON line reports the medians over rounds of CUDA-event
times.  To put the metric in context it also times ``Engine.sample`` (B = 32, 50 DDIM steps, synthetic weights: the
sampling of one test batch), and reports each path's worst error against float64 relative to each output's largest
element, with the card name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mld_b200 import metrics as M, synth  # noqa: E402
from mld_b200.engine import Engine, make_config  # noqa: E402
from oracle import ape_ave as O  # noqa: E402

T = 196


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except Exception:
        power = "unknown"
    return name, power


def _time(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def _rel(out, ref):
    return max(float((out[k].double() - ref[k]).abs().max() / ref[k].abs().max()) for k in O.NAMES)


def _sampler():
    eng = Engine(make_config(), 0)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
    eng.finalize()
    eng.set_mean_std(*synth.mean_std())
    eng.set_timesteps(50)
    return eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32,1024")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    torch.set_grad_enabled(False)
    card, power = _card()
    res = {"card": card, "power_limit": power, "T": T, "rounds": a.rounds, "sizes": {}}
    for B in [int(s) for s in a.sizes.split(",")]:
        g = torch.Generator().manual_seed(B)
        lengths = torch.randint(40, T + 1, (B,), generator=g).tolist()
        lengths[0] = T
        text = O.synth_joints(B, T, "humanml3d", 1, lengths).cuda()
        ref = O.synth_joints(B, T, "humanml3d", 2, lengths).cuda()
        native = lambda: M.ape_ave_update(text, ref, lengths)                          # noqa: E731
        eager = lambda: O.ape_ave_update(text, ref, lengths, dtype=torch.float32)      # noqa: E731
        f64 = O.ape_ave_update(text, ref, lengths)
        acc = {"native": _rel(native(), f64), "eager_fp32": _rel(eager(), f64)}
        n_reps, e_reps = 50, max(1, 96 // B)
        native(), eager()                                                              # warm-up
        times = {"native": [], "eager_fp32": []}
        for _ in range(a.rounds):
            times["native"].append(_time(native, n_reps))
            times["eager_fp32"].append(_time(eager, e_reps))
        med = {k: statistics.median(v) for k, v in times.items()}
        res["sizes"][str(B)] = {"ms_median": med, "ms_all": times, "speedup": med["eager_fp32"] / med["native"],
                                "rel_err_vs_f64": acc}
    eng = _sampler()
    Bs = 32
    ctx, noise = synth.text_context(Bs, 77, seed=1), synth.init_noise(Bs, seed=2)
    ctx, noise = ctx.cuda(), noise.cuda()
    lens = [T] * Bs
    sample = lambda: eng.sample(ctx, noise, lens, want=("joints",))                   # noqa: E731
    sample()
    res["sample_ms_B32_50steps"] = statistics.median(_time(sample, 3) for _ in range(a.rounds))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
