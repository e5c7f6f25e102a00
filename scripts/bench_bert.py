"""Benchmark of the native BERT text encoder on one GPU (synthetic distilbert-base-uncased weights).

    python scripts/bench_bert.py [--out DIR] [--iters N] [--warmup W]

Times with CUDA events after warm-up:
  * the DistilBERT tower alone on 2B = 512 rows as MLD sends them under classifier-free guidance: B "" rows
    ([CLS] [SEP]) + B prompts of seeded length 8..30 tokens, right-padded to the longest.  Through mldb_bert_encode on
    every row ("plain"), through B200TextEncoder.encode_ids with the distinct rows once ("savings"), and through
    transformers' DistilBertModel in fp32 (its default attention, TF32 off) on the same GPU;
  * token ids -> joints at B = 256, 50 DDIM steps: encode_ids, then the sampling path (mldb_sample) with the
    [2B, L, 768] context.
TFLOP/s are algorithmic: FLOPs of the full request (every row, every padded position, every key of the padded row)
computed from shapes here, divided by the measured time.  Prints the GPU name, power limit and SM clock of the same
run, one JSON line, and writes it to DIR/bench_bert.json.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_text import gpu_info, timed  # noqa: E402


def tower_flops(n, L, c):
    """Forward FLOPs of the BERT tower on n rows of L positions (2 per multiply-add)."""
    d, ff = c.hidden, c.ff
    per_tok = 2 * d * 3 * d + 2 * d * d + 2 * 2 * d * ff             # qkv, out-projection, lin1 + lin2
    return c.layers * (n * L * per_tok + n * 2 * 2 * d * L * L)       # + QK^T and PV over all L keys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="bench_bert_out")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--B", type=int, default=256)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from mld_b200 import synth
    from mld_b200.pipeline import B200MLD
    from mld_b200.text import B200TextEncoder, BertTextConfig, plan_bert_rows
    torch.set_grad_enabled(False)
    torch.cuda.set_device(0)
    res = {"bench": "bert_text", **gpu_info()}
    B = args.B
    c = BertTextConfig()
    sd = synth.bert_text_state_dict(5151)
    pids, plen = synth.bert_text_ids(B, 30, seed=11, len_lo=8, len_hi=30)
    L = int(plen.max())
    empty = torch.zeros(B, L, dtype=torch.long)
    empty[:, 0], empty[:, 1] = 101, 102
    ids = torch.cat([empty, pids[:, :L]])
    lengths = torch.cat([torch.full((B,), 2), plen])
    mask = (torch.arange(L)[None] < lengths[:, None]).long()
    enc = B200TextEncoder.from_state_dict(sd, config=c).cuda()
    eng = enc.engine()
    d_ids, d_len, d_mask = ids.cuda(), lengths.cuda(), mask.cuda()
    flops = tower_flops(2 * B, L, c)
    ms_plain = timed(lambda: eng.bert_encode(d_ids, d_len), args.iters, args.warmup)
    ms_sav = timed(lambda: enc.encode_ids(ids, mask), args.iters, args.warmup)
    rows, _, _ = plan_bert_rows(ids, lengths)
    tower = {"rows": 2 * B, "L": L, "tflop": flops / 1e12, "plain_ms": ms_plain,
             "plain_tflops": flops / ms_plain / 1e9, "savings_ms": ms_sav, "savings_rows": int(rows.shape[0]),
             "savings_effective_tflops": flops / ms_sav / 1e9}
    try:
        import transformers as T
        torch.backends.cuda.matmul.allow_tf32 = False
        m = T.DistilBertModel(T.DistilBertConfig())
        m.load_state_dict({k[len("text_model."):]: v for k, v in sd.items()}, strict=True)
        m = m.cuda().eval()
        ms = timed(lambda: m(input_ids=d_ids, attention_mask=d_mask).last_hidden_state, args.iters, args.warmup)
        tower.update(hf_fp32_ms=ms, hf_fp32_tflops=flops / ms / 1e9, hf_attn=m.config._attn_implementation)
        del m
    except ImportError as exc:
        tower["hf_fp32"] = f"not measured ({exc})"
    res["tower"] = tower
    # token ids -> joints at B, 50 DDIM steps
    dsd, vsd = synth.denoiser_state_dict(1234), synth.mld_vae_state_dict(4321)
    mean, std = synth.mean_std()
    mld = B200MLD(dsd, vsd, mean=mean, std=std, text_encoder=enc)
    noise = synth.init_noise(B, seed=2).cuda()
    frames = [196] * B

    def e2e():
        return mld.engine.sample(enc.encode_ids(ids, mask), noise, frames, want=("joints",))

    ms = timed(e2e, max(3, args.iters // 3), 1)
    res["e2e"] = {"B": B, "steps": 50, "S_ctx": L, "ms": ms, "text_ms": ms_sav, "motions_per_s": B / ms * 1e3}
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_bert.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
