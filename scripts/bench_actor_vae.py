"""Benchmark of the ActorVae encoder on one GPU (synthetic weights of the HumanAct12 action model's VAE).

    python scripts/bench_actor_vae.py [--out DIR] [--rounds R] [--batches 512,32] [--T 60]

Per batch size B (every motion T = 60 frames, the action512 shape), times with CUDA events:
  * "encode": ``ActorVae.encode`` up to the distribution (mu, std);
  * "encode_decode": encode -> rsample -> decode, the reconstruction ``MLD.a2m_eval`` runs at its stage "vae";
through the native drop-in ``B200ActorVae`` ("native"), and through the same ActorVae built from torch.nn layers
(nn.TransformerEncoder / nn.TransformerDecoder, sine PE) in fp32 eager on the same GPU, with TF32 off for matmuls
and cuDNN ("torch_fp32") and with torch's defaults ("torch_default").  All legs alternate inside every round after
every shape has been warmed up; the median of the rounds is reported.  FLOP counts are algorithmic, from the shapes
(the encoder counted with its last layer trimmed to the two distribution rows, as the reference's output only
reads those; the decoder counted as the reference's layers state it).  Worst errors, relative to the max, are
taken against the float64 oracle on the B = 32 batch.  Prints the GPU name, power limit and max SM clock of the
same run, one JSON line, and writes it to DIR/bench_actor_vae.json.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NFEATS, D, FF, LAYERS, HEADS = 150, 256, 1024, 6, 4


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [s.strip() for s in q.split(",")]
    except Exception as exc:                                            # not fatal: the numbers still stand
        info["nvidia_smi"] = f"unavailable ({exc})"
    return info


def encode_flops(T, d=D, ff=FF, layers=LAYERS, nfeats=NFEATS):
    """Per motion: the skel embedding over T frames, layers - 1 full layers over L = T + 2 tokens, and the last
    layer with k | v over all L tokens but queries, out-projection and FFN on the 2 distribution rows."""
    L = T + 2
    full = 2 * L * d * 3 * d + 2 * 2 * L * L * d + 2 * L * d * d + 2 * 2 * L * d * ff
    last = 2 * L * d * 2 * d + 2 * 2 * d * d + 2 * 2 * 2 * L * d + 2 * 2 * d * d + 2 * 2 * 2 * d * ff
    return 2 * T * nfeats * d + (layers - 1) * full + last


def decode_flops(T, d=D, ff=FF, layers=LAYERS, nfeats=NFEATS):
    """Per motion: T queries, self-attention over T keys, cross-attention to the 1 latent token, FFN, final layer."""
    self_attn = 2 * T * d * 3 * d + 2 * 2 * T * T * d + 2 * T * d * d
    cross = 2 * T * d * d + 2 * d * 2 * d + 2 * 2 * T * d + 2 * T * d * d
    return layers * (self_attn + cross + 2 * 2 * T * d * ff) + 2 * T * d * nfeats


class TorchActorVae(nn.Module):
    """ActorVae's math from torch.nn layers, with the reference's state-dict names (the yardstick)."""

    def __init__(self):
        super().__init__()
        enc, dec = nn.Module(), nn.Module()
        enc.skel_embedding = nn.Linear(NFEATS, D)
        enc.mu_token, enc.logvar_token = nn.Parameter(torch.zeros(D)), nn.Parameter(torch.zeros(D))
        enc.seqTransEncoder = nn.TransformerEncoder(nn.TransformerEncoderLayer(D, HEADS, FF, 0.1, "gelu"), LAYERS)
        dec.seqTransDecoder = nn.TransformerDecoder(nn.TransformerDecoderLayer(D, HEADS, FF, 0.1, "gelu"), LAYERS)
        dec.final_layer = nn.Linear(D, NFEATS)
        for m in (enc, dec):
            m.sequence_pos_encoding = nn.Module()
            m.sequence_pos_encoding.register_buffer("pe", torch.zeros(5000, 1, D))
        self.encoder, self.decoder = enc, dec

    def encode(self, x, lengths):
        B, T, _ = x.shape
        e = self.encoder
        valid = torch.arange(T, device=x.device)[None] < lengths[:, None]
        tokens = torch.stack((e.mu_token, e.logvar_token))[:, None].expand(2, B, D)
        xseq = torch.cat((tokens, e.skel_embedding(x).permute(1, 0, 2)), 0) + e.sequence_pos_encoding.pe[:T + 2]
        keep = torch.cat((torch.ones(B, 2, dtype=torch.bool, device=x.device), valid), 1)
        final = e.seqTransEncoder(xseq, src_key_padding_mask=~keep)
        return torch.distributions.Normal(final[0], final[1].exp().pow(0.5))

    def decode(self, z, lengths, T):
        dec = self.decoder
        valid = torch.arange(T, device=z.device)[None] < lengths[:, None]
        queries = torch.zeros(T, z.shape[1], D, device=z.device) + dec.sequence_pos_encoding.pe[:T]
        out = dec.final_layer(dec.seqTransDecoder(tgt=queries, memory=z, tgt_key_padding_mask=~valid))
        out[~valid.T] = 0
        return out.permute(1, 0, 2)


def rsample(dist):
    return (dist.loc + 1.0 * (dist.rsample() - dist.loc)).unsqueeze(0)


def time_ms(fn, reps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="bench_actor_out")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batches", default="512,32")
    ap.add_argument("--T", type=int, default=60)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_actor_vae.py measures on a GPU and found none")
    import __graft_entry__ as G
    G.build()
    from types import SimpleNamespace
    from mld_b200 import synth
    from mld_b200.modules import B200ActorVae
    from oracle import mld_oracle as O
    from oracle.actor_encode import actor_encode
    torch.set_grad_enabled(False)
    torch.cuda.set_device(0)
    sd = synth.actor_vae_state_dict(seed=777)
    native = B200ActorVae(ablation=SimpleNamespace(), nfeats=NFEATS, latent_dim=[1, D], ff_size=FF,
                          num_layers=LAYERS, num_heads=HEADS)
    native.load_state_dict(sd, strict=True)
    native = native.cuda()
    yard = TorchActorVae()
    yard.load_state_dict(sd, strict=True)
    yard = yard.cuda().eval()
    default_tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)

    def precision(fp32):
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = (False, False) if fp32 else default_tf32

    info = gpu_info()
    print(f"[bench_actor_vae] {info}", flush=True)
    res = {"gpu": info, "rounds": args.rounds, "T": args.T, "torch_default_tf32": {"matmul": default_tf32[0],
           "cudnn": default_tf32[1]}, "flop_per_motion": {"encode": encode_flops(args.T)}, "results": [], "errors": {}}
    res["flop_per_motion"]["encode_decode"] = encode_flops(args.T) + decode_flops(args.T)
    print(f"[bench_actor_vae] FLOP per motion: encode {res['flop_per_motion']['encode'] / 1e9:.3f} G, "
          f"encode+decode {res['flop_per_motion']['encode_decode'] / 1e9:.3f} G", flush=True)
    T = args.T
    for B in [int(b) for b in args.batches.split(",")]:
        x = torch.randn(B, T, NFEATS, generator=torch.Generator().manual_seed(B)).cuda()
        lengths = [T] * B
        len_d = torch.full((B,), T, device="cuda")

        def legs_for(impl):
            if impl == "native":
                return {"encode": lambda: native.encode(x, lengths),
                        "encode_decode": lambda: native.decode(native.encode(x, lengths)[0], lengths)}
            fp32 = impl == "torch_fp32"

            def enc():
                precision(fp32)
                return yard.encode(x, len_d)

            def enc_dec():
                precision(fp32)
                return yard.decode(rsample(yard.encode(x, len_d)), len_d, T)
            return {"encode": enc, "encode_decode": enc_dec}

        legs = {(case, impl): fn for impl in ("native", "torch_fp32", "torch_default") for case, fn in legs_for(impl).items()}
        for fn in legs.values():                                      # warm-up: modules, workspaces, plans
            fn(); fn()
        times = {k: [] for k in legs}
        for _ in range(args.rounds):
            for k, fn in legs.items():
                times[k].append(time_ms(fn, 20))
        precision(False)
        for (case, impl), ts in times.items():
            ms = statistics.median(ts)
            row = {"B": B, "case": case, "impl": impl, "ms": round(ms, 4), "spread_ms": [round(min(ts), 4), round(max(ts), 4)],
                   "motions_per_s": round(B / ms * 1e3, 1),
                   "tflops": round(res["flop_per_motion"][case] * B / ms / 1e9, 2)}
            res["results"].append(row)
            print(f"[bench_actor_vae] B={B:4d} {case:13s} {impl:13s} {ms:9.3f} ms  {row['motions_per_s']:10.1f} motions/s  "
                  f"{row['tflops']:6.2f} TFLOP/s", flush=True)
        if B == 32:                                                   # accuracy against float64
            sd64 = {k: v.double() for k, v in sd.items()}
            cfg = O.VaeCfg(kind="actor", nfeats=NFEATS, num_layers=LAYERS)
            mu64, logvar64 = actor_encode(sd64, cfg, x.cpu().double(), lengths)
            prev = torch.get_default_dtype()
            torch.set_default_dtype(torch.float64)                    # the oracle's decoder queries
            try:
                rec64 = O.vae_decode(sd64, cfg, mu64, lengths)
            finally:
                torch.set_default_dtype(prev)
            for impl in ("native", "torch_fp32", "torch_default"):
                if impl == "native":
                    dist = native.encode(x, lengths)[1]
                    rec = native.decode(dist.loc[None], lengths)
                else:
                    precision(impl == "torch_fp32")
                    dist = yard.encode(x, len_d)
                    rec = yard.decode(dist.loc[None], len_d, T)
                res["errors"][impl] = {"mu": rel(dist.loc, mu64[0]), "std": rel(dist.scale, logvar64[0].exp().pow(0.5)),
                                       "decode_of_mu": rel(rec, rec64)}
                print(f"[bench_actor_vae] vs float64, B=32 {impl:13s} " +
                      "  ".join(f"{k} {v:.2e}" for k, v in res["errors"][impl].items()), flush=True)
            precision(False)
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_actor_vae.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
