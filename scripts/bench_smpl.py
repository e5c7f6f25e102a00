"""Time the SMPL layer as one ``MLD.a2m_eval`` uses it: four Rotation2xyz calls per test batch (``feats2joints``
('vertices', vertstrans=False) and ``feats2joints_eval`` ('smpl', vertstrans=True) on the generated and the reference
features), with V = 6890 and a length mask.

    python scripts/bench_smpl.py [--sizes 32x60,1024x60] [--rounds 7] [--out FILE.json]

Compared against ``oracle.smpl.TorchSMPL`` (the same layer in fp32 eager torch, as smplx computes it) on the same GPU,
once with TF32 off and once with torch's defaults.  The three are alternated within every round; each result is the
median over the rounds of CUDA-event time around the four calls.  TorchSMPL runs the vertex calls in chunks of at
most 16384 frames (its [frames, V, 4, 4] skinning transforms of a whole B = 1024 batch take 27 GB each).  Accuracy
at the timed sizes: the worst per-frame error against the float64 oracle, relative to the frame's largest coordinate.
Per call it also times the joints call (``k_smpl_fk`` alone), the vertex call, and the vertex call of the same model
with every skinning weight zero, which skips the skinning sums (every tile's joint mask is empty): the difference is
what the sums on CUDA cores cost.  Prints one JSON line with the card name and power limit.
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

from mld_b200 import _lib, synth  # noqa: E402
from mld_b200.engine import Engine, make_config  # noqa: E402
from oracle import smpl as O  # noqa: E402

V = 6890
CHUNK_FRAMES = 16384


def _engine(model):
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    cfg = _lib.default_smpl_config()
    cfg.num_vertices = V
    eng.smpl_configure(cfg)
    eng.load_state_dict(model, "smpl.")
    eng.finalize()
    return eng


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except Exception:
        power = "unknown"
    return name, power


def _inputs(B, T, seed):
    rst, ref = synth.smpl_feats(B, T, seed=seed).cuda(), synth.smpl_feats(B, T, seed=seed + 1).cuda()
    lengths = torch.randint(max(1, T // 3), T + 1, (B,), generator=torch.Generator().manual_seed(seed))
    mask = (torch.arange(T)[None] < lengths[:, None]).cuda()
    return rst, ref, mask


def native_calls(eng, rst, ref, mask):
    return [eng.smpl_forward(f, mask, kind, vt) for f in (rst, ref)
            for kind, vt in ((_lib.SMPL_VERTICES, False), (_lib.SMPL_JOINTS, True))]


def torch_calls(net, rst, ref, mask):
    out = []
    for f in (rst, ref):
        B, T = f.shape[:2]
        x = f.view(B, T, 6, 25).permute(0, 3, 2, 1)
        cb = max(1, CHUNK_FRAMES // T)
        out.append(torch.cat([net(x[b:b + cb], mask[b:b + cb], "vertices", False) for b in range(0, B, cb)]))
        out.append(net(x, mask, "smpl", True))
    return out


def _time(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def _accuracy(model, outs, rst, ref, mask):
    """worst per-frame relative error of the four outputs against float64, a few sequences at a time"""
    md = {k: v.cuda() for k, v in model.items()}
    worst = 0.0
    for i, (f, jt, vt) in enumerate(((rst, "vertices", False), (rst, "smpl", True), (ref, "vertices", False),
                                     (ref, "smpl", True))):
        B, T = f.shape[:2]
        cb = max(1, (1 << 25) // (T * V * 16))       # the oracle skins every vertex for either joint type
        for b in range(0, B, cb):
            x = f[b:b + cb].double().view(-1, T, 6, 25).permute(0, 3, 2, 1)
            r = O.rotation2xyz(md, x, mask[b:b + cb], jt, vt)
            a = outs[i][b:b + cb].double()
            err = (a - r).abs().amax(dim=(1, 2)) / r.abs().amax(dim=(1, 2)).clamp_min(1e-30)
            worst = max(worst, float(err.max()))
    return worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32x60,1024x60")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_smpl needs a GPU")
    torch.set_grad_enabled(False)
    import __graft_entry__ as G
    G.build()
    model = synth.smpl_model(1, V)
    eng = _engine(model)
    # the same model with every skinning weight zero: each vertex tile's joint mask is empty, so its vertex call runs
    # the GEMM, v_posed, the staging and the stores without the skinning sums (its output is not the layer's)
    no_skin = _engine({**model, "lbs_weights": torch.zeros_like(model["lbs_weights"])})
    net = O.TorchSMPL(model).cuda()
    card, power = _card()
    res = {"card": card, "power_limit": power, "V": V, "rounds": a.rounds, "sizes": {}}
    for size in a.sizes.split(","):
        B, T = map(int, size.split("x"))
        rst, ref, mask = _inputs(B, T, seed=B + T)
        reps = 20 if B * T <= 4096 else 3

        def run_native():
            native_calls(eng, rst, ref, mask)

        def run_torch(tf32):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            torch.backends.cudnn.allow_tf32 = tf32
            torch_calls(net, rst, ref, mask)
        default_tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
        legs = {"native": run_native, "torch_fp32": lambda: run_torch(False),
                "torch_default": lambda: run_torch(default_tf32[0])}
        for fn in legs.values():                          # warm-up of every shape
            fn()
        times = {k: [] for k in legs}
        for _ in range(a.rounds):
            for k, fn in legs.items():
                times[k].append(_time(fn, reps))
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = default_tf32
        outs = native_calls(eng, rst, ref, mask)
        acc = {"native": _accuracy(model, outs, rst, ref, mask)}
        del outs
        for leg, tf32 in (("torch_fp32", False), ("torch_default", default_tf32[0])):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            outs = torch_calls(net, rst, ref, mask)
            acc[leg] = _accuracy(model, outs, rst, ref, mask)
            del outs
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = default_tf32
        # one call of each kind: 'smpl' is k_smpl_fk alone, 'vertices' is k_smpl_fk + k_smpl_lbs
        split = {"joints_call": statistics.median(_time(lambda: eng.smpl_forward(rst, mask, _lib.SMPL_JOINTS, True), reps)
                                                  for _ in range(a.rounds)),
                 "vertices_call": statistics.median(_time(lambda: eng.smpl_forward(rst, mask, _lib.SMPL_VERTICES, False),
                                                          reps) for _ in range(a.rounds)),
                 "vertices_call_without_skinning_sums": statistics.median(
                     _time(lambda: no_skin.smpl_forward(rst, mask, _lib.SMPL_VERTICES, False), reps)
                     for _ in range(a.rounds))}
        res["sizes"][f"{B}x{T}"] = {"ms_median": {k: statistics.median(v) for k, v in times.items()},
                                    "ms_all": times, "native_ms_per_call": split, "rel_err_vs_f64": acc}
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
