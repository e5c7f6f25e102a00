"""Time the four classifier calls of one HUMANACTMetrics.update (logits on generated and ground-truth joints, then
features on both) at T = 60: the native drop-ins against the reference modules' math in fp32 eager torch on the same
GPU (nn.GRU through cuDNN), with TF32 off and with torch's defaults.  Median of alternating rounds; the card's name
and power limit are read in the same run.  Optionally writes a torch.profiler kernel table of each side.

    python scripts/bench_a2m.py [--batches 32 4096] [--rounds 7] [--iters 20] [--profile DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def flops(B, T, In=72, H=128, L=2, out=12):
    """Algorithmic FLOPs of one call: input GEMMs, recurrent GEMMs, the head (gates not counted)."""
    per = sum(2 * T * 3 * H * (In if k == 0 else H) + 2 * T * 3 * H * H for k in range(L))
    return B * (per + 2 * H * 30 + 2 * 30 * out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 4096])
    ap.add_argument("--T", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--profile", default="")
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    from mld_b200 import synth
    from mld_b200.evaluator import B200MotionDiscriminator, B200MotionDiscriminatorForFID
    from oracle.a2m_gru import TorchDiscriminator
    sd = synth.a2m_state_dict(1357)
    cls, fid = B200MotionDiscriminator(**synth.A2M_DIMS).cuda(), B200MotionDiscriminatorForFID(**synth.A2M_DIMS).cuda()
    cls.load_state_dict(sd)
    fid.load_state_dict(sd)
    ref = TorchDiscriminator({k: v.cuda() for k, v in sd.items()}, **synth.A2M_DIMS).cuda()
    info = gpu_info()
    res = {"gpu": info, "T": a.T, "results": []}
    for B in a.batches:
        rec, gt = synth.a2m_motions(B, a.T, seed=1).cuda(), synth.a2m_motions(B, a.T, seed=2).cuda()
        ln = torch.full((B,), a.T)

        def native():
            cls(rec, ln); cls(gt, ln); fid(rec, ln); fid(gt, ln)

        def torch_side():
            ref.both(rec, ln)[0]; ref.both(gt, ln)[0]; ref.both(rec, ln)[1]; ref.both(gt, ln)[1]

        def tf32(on):
            torch.backends.cudnn.allow_tf32 = on
            torch.backends.cuda.matmul.allow_tf32 = on

        sides = {"native": (native, False), "torch_fp32": (torch_side, False), "torch_default": (torch_side, True)}
        times = {k: [] for k in sides}
        for fn, on in sides.values():
            tf32(on)
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k, (fn, on) in sides.items():
                tf32(on)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(a.iters):
                    fn()
                e.record()
                e.synchronize()
                times[k].append(s.elapsed_time(e) / a.iters)
        f = 4 * flops(B, a.T)
        row = {"B": B}
        for k, v in times.items():
            med = statistics.median(v)
            row[k] = {"ms": round(med, 4), "spread_ms": [round(min(v), 4), round(max(v), 4)],
                      "tflops": round(f / med / 1e9, 3)}
        res["results"].append(row)
        print(json.dumps(row), flush=True)
        if a.profile:
            os.makedirs(a.profile, exist_ok=True)
            from torch.profiler import ProfilerActivity, profile
            for k, (fn, on) in sides.items():
                tf32(on)
                with profile(activities=[ProfilerActivity.CUDA]) as p:
                    fn()
                    torch.cuda.synchronize()
                with open(os.path.join(a.profile, f"a2m_{k}_B{B}.txt"), "w") as fh:
                    fh.write(p.key_averages().table(sort_by="cuda_time_total", row_limit=25))
        tf32(False)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
