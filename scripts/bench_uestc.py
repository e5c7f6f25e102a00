"""Time the two classifier calls of one UESTCMetrics.update (yhat and features on generated and ground-truth motions)
at T = 60: the native drop-in against the same network built from torch.nn layers in fp32 eager on the same GPU
(cuDNN convolutions), with TF32 off and with torch's defaults.  Median of alternating rounds; the card's name and
power limit are read in the same run.  Optionally writes a torch.profiler kernel table of each side.

    python scripts/bench_uestc.py [--batches 32 1024] [--rounds 7] [--iters 20] [--profile DIR]
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

CHANNELS = (64, 64, 64, 64, 128, 128, 128, 256, 256, 256)
STRIDES = (1, 1, 1, 1, 2, 1, 1, 2, 1, 1)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def flops(T, cin=6, ncls=40, V=24, K=3):
    """Algorithmic FLOPs of one sequence, by part: the graph mix (dense 24 x 24 per partition), the gcn 1 x 1
    convolutions, the temporal convolutions (with the residual convolutions of blocks 4 and 7), the pool and head."""
    parts = {"mix": 0, "gcn": 0, "tconv": 0, "head": 0}
    Ti, ci = T, cin
    for i, (co, s) in enumerate(zip(CHANNELS, STRIDES)):
        To = (Ti - 1) // s + 1
        parts["mix"] += 2 * Ti * V * V * K * ci
        parts["gcn"] += 2 * Ti * V * K * ci * co
        parts["tconv"] += 2 * To * V * 9 * co * co + (2 * To * V * ci * co if i > 0 and (ci != co or s != 1) else 0)
        Ti, ci = To, co
    parts["head"] = Ti * V * 256 + 2 * 256 * ncls
    return parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 1024])
    ap.add_argument("--T", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--profile", default="")
    a = ap.parse_args()
    parts = flops(a.T)
    per_seq = sum(parts.values())
    print(json.dumps({"T": a.T, "gflop_per_sequence": round(per_seq / 1e9, 4),
                      "share": {k: round(v / per_seq, 4) for k, v in parts.items()}}), flush=True)
    if not torch.cuda.is_available():
        raise SystemExit("bench_uestc.py times the GPU: no CUDA device")
    torch.set_grad_enabled(False)
    import tempfile
    from mld_b200 import synth
    from mld_b200.evaluator import B200STGCN
    from oracle.make_golden_uestc import write_kintree
    from oracle.uestc_stgcn import TorchSTGCN
    sd = synth.stgcn_state_dict(2025)
    with tempfile.TemporaryDirectory() as d:
        kp = os.path.join(d, "kintree_table.pkl")
        write_kintree(kp)
        net = B200STGCN(in_channels=6, kintree_path=kp, num_class=40,
                        graph_args={"layout": "smpl", "strategy": "spatial"}, edge_importance_weighting=True)
    net.load_state_dict(sd, strict=True)
    net = net.cuda().eval()
    ref = TorchSTGCN().cuda().eval()
    ref.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=True)
    res = {"gpu": gpu_info(), "T": a.T, "gflop_per_sequence": per_seq / 1e9, "results": []}
    for B in a.batches:
        # UESTCMetrics.update's inputs: [B, T, 150] features viewed and permuted to [B, 24, 6, T]
        def metric_view(x):
            m = torch.zeros(B, a.T, 6, 25)
            m[..., :24] = x.permute(0, 3, 2, 1)
            m = m.reshape(B, a.T, 150).cuda()
            return m.view(B, a.T, 6, 25).permute(0, 3, 2, 1)[:, :-1]
        rec, gt = metric_view(synth.uestc_motions(B, a.T, seed=1)), metric_view(synth.uestc_motions(B, a.T, seed=2))

        def native():
            net(rec); net(gt)

        def torch_side():
            ref(rec.contiguous()); ref(gt.contiguous())

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
        f = 2 * B * per_seq
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
                with open(os.path.join(a.profile, f"uestc_{k}_B{B}.txt"), "w") as fh:
                    fh.write(p.key_averages().table(sort_by="cuda_time_total", row_limit=25))
        tf32(False)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
