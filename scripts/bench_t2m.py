"""Benchmark of the native T2M evaluator on one GPU (synthetic finest.tar-shaped weights).

    python scripts/bench_t2m.py [--out DIR] [--rounds R] [--batches 32,4096]

Per batch size B, times with CUDA events:
  * the motion side: MovementConvEncoder + MotionEncoderBiGRUCo on renorm4t2m'd feats [B, 196, 263] with synthetic
    ragged lengths (m_lens = length // 4, the GRU runs up to 49 steps);
  * the text side: TextEncoderBiGRUCo on word vectors / POS one-hots [B, 22, *] with ragged caption lengths;
through the native engine ("native"), and through the same networks built from torch.nn layers in fp32 eager on
the same GPU (oracle.t2m_eval.TorchNets) with cuDNN TF32 off ("torch_fp32") and with torch's defaults
("torch_default": cuDNN may use TF32).  The three alternate inside every round; the median of the rounds is
reported.  TFLOP/s are algorithmic: FLOPs from the shapes and the actual lengths (the GRU counted for the valid
steps of each sequence), over the measured time.  Prints the GPU name, power limit and max SM clock of the same
run, one JSON line, and writes it to DIR/bench_t2m.json.
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
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [s.strip() for s in q.split(",")]
    except Exception as exc:                                            # not fatal: the numbers still stand
        info["nvidia_smi"] = f"unavailable ({exc})"
    return info


def motion_flops(T, m_lens, d):
    """movement encoder over all T frames of every sequence + motion encoder (input_emb over all L rows, the GRU
    over each sequence's m_len steps in both directions, the head)."""
    T1, T2 = T // 2, T // 2 // 2
    pose, mh, ml, H, out = d["dim_pose"], d["dim_move_hidden"], d["dim_move_latent"], d["dim_motion_hidden"], d["dim_motion_latent"]
    per_seq = 2 * T1 * 4 * pose * mh + 2 * T2 * 4 * mh * ml + 2 * T2 * ml * ml + 2 * T2 * ml * H
    per_seq += 2 * 2 * H * H + 2 * H * out
    gru = sum(2 * int(n) * 2 * (3 * H * H + 3 * H * H) for n in m_lens)
    return len(m_lens) * per_seq + gru


def text_flops(L, lens, d):
    W, P, H, out = d["dim_word"], d["dim_pos_ohot"], d["dim_text_hidden"], d["dim_coemb_hidden"]
    per_seq = 2 * L * P * W + 2 * L * W * H + 2 * 2 * H * H + 2 * H * out
    gru = sum(2 * int(n) * 2 * (3 * H * H + 3 * H * H) for n in lens)
    return len(lens) * per_seq + gru


def time_ms(fn, reps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="bench_t2m_out")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batches", default="32,4096")
    args = ap.parse_args()
    import __graft_entry__ as G
    G.build()
    from mld_b200 import _lib, synth
    from mld_b200.engine import Engine, make_config
    from oracle.t2m_eval import TorchNets
    torch.set_grad_enabled(False)
    torch.cuda.set_device(0)
    sds = synth.t2m_state_dicts(2468)
    d = synth.T2M_DIMS
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    eng.t2m_configure(_lib.default_t2m_config())
    for k, p in (("text_encoder", "t2m_textencoder."), ("movement_encoder", "t2m_moveencoder."),
                 ("motion_encoder", "t2m_motionencoder.")):
        eng.load_state_dict(sds[k], p)
    eng.finalize()
    nets = TorchNets(sds, "cuda")
    mean, std = synth.mean_std()
    mean_e, std_e = synth.t2m_mean_std()
    info = gpu_info()
    print(f"[bench_t2m] {info}", flush=True)
    res = {"gpu": info, "rounds": args.rounds, "results": []}
    T, Lt = 196, 22
    for B in [int(b) for b in args.batches.split(",")]:
        lengths = torch.tensor(synth.ragged_lengths(B, seed=3))
        feats = synth.renorm4t2m(synth.t2m_feats(B, T, lengths.tolist(), seed=4), mean, std, mean_e, std_e).cuda()
        m_lens = lengths // 4
        word, pos = synth.t2m_text_inputs(B, Lt, seed=5)
        word, pos = word.cuda(), pos.cuda()
        t_lens = torch.randint(3, Lt + 1, (B,), generator=torch.Generator().manual_seed(6))
        reps = 20 if B <= 256 else 1

        def nat_motion():
            return eng.t2m_motion(eng.t2m_movement(feats[..., :-4]), m_lens)

        def nat_text():
            return eng.t2m_text(word, pos, t_lens)

        def tor_motion():
            return nets.motion(nets.movement(feats[..., :-4]), m_lens)

        def tor_text():
            return nets.text(word, pos, t_lens)

        def with_tf32(fn, on):
            def run():
                torch.backends.cudnn.allow_tf32 = on
                return fn()
            return run

        legs = {("motion", "native"): nat_motion, ("motion", "torch_fp32"): with_tf32(tor_motion, False),
                ("motion", "torch_default"): with_tf32(tor_motion, True), ("text", "native"): nat_text,
                ("text", "torch_fp32"): with_tf32(tor_text, False), ("text", "torch_default"): with_tf32(tor_text, True)}
        for fn in legs.values():                                        # warm-up: modules, workspaces, cuDNN plans
            fn(); fn()
        times = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, fn in legs.items():
                times[k].append(time_ms(fn, reps))
        torch.backends.cudnn.allow_tf32 = True
        flops = {"motion": motion_flops(T, m_lens.tolist(), d), "text": text_flops(Lt, t_lens.tolist(), d)}
        for (side, impl), ts in times.items():
            ms = statistics.median(ts)
            row = {"B": B, "side": side, "impl": impl, "ms": round(ms, 4), "spread_ms": [round(min(ts), 4), round(max(ts), 4)],
                   "seq_per_s": round(B / ms * 1e3, 1), "tflops": round(flops[side] / ms / 1e9, 2)}
            res["results"].append(row)
            print(f"[bench_t2m] B={B:5d} {side:6s} {impl:13s} {ms:9.3f} ms  {row['seq_per_s']:10.1f} seq/s  "
                  f"{row['tflops']:6.2f} TFLOP/s", flush=True)
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_t2m.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
