"""Bring-up aid for the wgmma attention kernel: every shape in its own process (a device trap poisons the
context), with an error breakdown by head / query-row block / which key blocks seem to contribute.
usage: python scripts/dbg_attn.py            (all cases)      python scripts/dbg_attn.py one nseq Lq Lk hd masked"""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = [(3, 79, 79, 64, 0), (5, 79, 79, 64, 1), (2, 16, 16, 64, 0), (2, 64, 64, 64, 0), (2, 128, 128, 64, 0),
         (7, 3, 3, 64, 0), (300, 79, 79, 64, 0), (8, 196, 196, 64, 1), (6, 196, 196, 128, 0), (3, 79, 79, 128, 1),
         (300, 1, 79, 64, 0), (5, 196, 2, 128, 0), (2, 256, 256, 64, 0),
         (256, 196, 196, 64, 1), (100, 196, 196, 128, 0), (200, 198, 198, 64, 1), (400, 130, 130, 64, 1), (512, 3, 3, 64, 0)]


def one(nseq, Lq, Lk, hd, masked):
    import torch
    from mld_b200.engine import Engine, make_config
    heads, d = 4, 4 * hd
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    g = torch.Generator().manual_seed(nseq * 131 + Lq + hd)
    q = torch.randn(nseq * Lq, d, generator=g)
    kv = torch.randn(nseq * Lk, 2 * d, generator=g)
    lengths = [max(1, (7 * i + 5) % Lk) for i in range(nseq)] if masked else None
    qh = q.reshape(nseq, Lq, heads, hd).permute(0, 2, 1, 3).double()
    kh = kv[:, :d].reshape(nseq, Lk, heads, hd).permute(0, 2, 1, 3).double()
    vh = kv[:, d:].reshape(nseq, Lk, heads, hd).permute(0, 2, 1, 3).double()
    s = qh @ kh.transpose(-1, -2) / hd ** 0.5
    if lengths is not None:
        mask = torch.arange(Lk)[None, :] >= torch.as_tensor(lengths)[:, None]
        s = s.masked_fill(mask[:, None, None, :], float("-inf"))
    ref = (torch.softmax(s, -1) @ vh)                       # [nseq, heads, Lq, hd]
    if Lq == Lk:
        qkv = torch.cat([q, kv], 1)
        y = eng.debug_attention(qkv, nseq, Lq, heads, lengths, mode=2)
    else:
        y = eng.debug_attention(q, nseq, Lq, heads, lengths, mode=2, kv=kv, Lk=Lk)
    torch.cuda.synchronize()
    y = y.cpu().double().reshape(nseq, Lq, heads, hd).permute(0, 2, 1, 3)
    fin = bool(torch.isfinite(y).all())
    err = (y - ref).abs()
    rel = float(err.max() / ref.abs().max())
    print(f"case nseq={nseq} Lq={Lq} Lk={Lk} hd={hd} masked={masked}: finite={fin} rel={rel:.3e}", flush=True)
    if fin and rel < 5e-6:
        return
    print("  per head:", [f"{float(err[:, h].max()):.2e}" for h in range(heads)])
    print("  per row block of 32:", [f"{float(err[:, :, r:r + 32].max()):.2e}" for r in range(0, Lq, 32)])
    print("  per d block of 16:", [f"{float(err[..., c:c + 16].max()):.2e}" for c in range(0, hd, 16)])
    print("  per sequence (first 8):", [f"{float(err[i].max()):.2e}" for i in range(min(nseq, 8))])
    # which key range does the output look like it used?
    for k1 in range(16, Lk + 15, 16):
        s2 = s.clone()
        s2[..., min(k1, Lk):] = float("-inf")
        r2 = torch.softmax(s2, -1) @ vh
        e2 = float((y - r2).abs().max() / r2.abs().max())
        if e2 < 1e-4:
            print(f"  matches a softmax over the first {k1} keys only (rel {e2:.2e})")
    yn = torch.nan_to_num(y)
    print("  y[0,0,0,:8] =", [f"{float(v):.4f}" for v in yn[0, 0, 0, :8]], " ref =", [f"{float(v):.4f}" for v in ref[0, 0, 0, :8]])
    print("  ratio y/ref rows 0..3 col 0:", [f"{float(yn[0, 0, r, 0] / ref[0, 0, r, 0]):.4f}" for r in range(min(4, Lq))])


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "one":
        one(*map(int, sys.argv[2:7]))
    else:
        for c in CASES:
            r = subprocess.run([sys.executable, __file__, "one", *map(str, c)], capture_output=True, text=True, timeout=300)
            out = (r.stdout + r.stderr).strip().splitlines()
            keep = [l for l in out if not l.startswith("[build]")]
            print("\n".join(keep[-14:]) if r.returncode else "\n".join(keep), flush=True)
            if r.returncode:
                print(f"  -> exit code {r.returncode} for case {c}", flush=True)
