"""Weights at chosen split16 exponents, for the tests of every packed-weight path at s != 14 (not a test module).

The engine packs each weight matrix with its own power-of-two scale 2^s, s = floor(log2(2^14 / max|w|)) clamped to
[-14, 14] (``pack_linear``, mld_b200/csrc/engine.cu), and every kernel multiplies its accumulator by 2^-s.  Weights
of the usual 1/sqrt(K) size all sit at the clamp, s = 14, so a kernel that applied the wrong weight's scale, or a
hard-coded 2^-14, would still be right on them.  ``weight_at`` builds a weight at any exponent, and
``with_outliers`` gives a synthetic state dict a spread of exponents over its packs while the model stays the same
model; ``packed_exponents`` says which exponent each pack the engine builds gets."""
import itertools
import re

import torch

from split16_ref import weight_scale_log2

# magnitudes planted by with_outliers and the exponents they give (floor(log2(2^14 / m)))
OUTLIERS = {1.5: 13, 3.0: 12, 6.0: 11}
_PERMS = list(itertools.permutations(OUTLIERS))
_WEIGHT = re.compile(r"(weight|weight_[ih]h_l0(_reverse)?)$")
_TABLES = ("token_embedding.weight", "position_embedding.weight")
_LAYER = re.compile(r"^(.*?)(input_blocks\.\d+|middle_block|output_blocks\.\d+|layers\.\d+)\.$")
_BLOCK_ORDER = {"input_blocks": 0, "layers": 0, "middle_block": 1, "output_blocks": 2}


def engine_exponent(W: torch.Tensor) -> int:
    """The exponent the engine packs W with: the largest finite |w| sets it, an all-zero (or all non-finite)
    weight packs at s = 0."""
    finite = W[torch.isfinite(W)]
    return weight_scale_log2(finite) if finite.numel() else 0


def weight_at(N: int, K: int, s: int, gen: torch.Generator) -> torch.Tensor:
    """[N, K] fp32 randn rescaled so that max|w| = 1.5 * 2^(13 - s): the engine's exponent is exactly s, with no
    clamp involved, for every s in [-14, 14]."""
    assert -14 <= s <= 14
    W = torch.randn(N, K, generator=gen, dtype=torch.float64)
    W = (W * (1.5 * 2.0 ** (13 - s) / W.abs().max())).float()
    assert engine_exponent(W) == s
    return W


def is_packed(key: str, t: torch.Tensor) -> bool:
    """A weight matrix the engine packs (a GEMM operand), as opposed to a table it uploads as it is: token and
    position embeddings, PE tables, distribution tokens, action embeddings, LayerNorm parameters, biases."""
    return t.dim() >= 2 and bool(_WEIGHT.search(key)) and not key.endswith(_TABLES)


def _plant(W: torch.Tensor, rows: slice, mag: float, g: torch.Generator, n: int = 2):
    """Set n seeded elements of W[rows] to +-mag (W viewed as [N, K...])."""
    sub = W[rows].reshape(-1)
    idx = torch.randperm(sub.numel(), generator=g)[:n]
    sign = torch.randint(0, 2, (n,), generator=g).float() * 2 - 1
    sub[idx] = sign * mag
    W[rows] = sub.reshape(W[rows].shape)


def _perm(g: torch.Generator):
    return _PERMS[int(torch.randint(0, len(_PERMS), (1,), generator=g))]


def with_outliers(sd, seed: int = 0):
    """A copy of a synthetic state dict (any of mld_b200.synth's) in which a few elements of every packed weight are
    set to +-1.5, +-3 or +-6 (exponents 13, 12, 11).  The bulk of each weight, and so the model, stays as it was.

    - In every layer the attention out-projection and the two FFN weights (linear1 / linear2, CLIP's fc1 / fc2)
      get pairwise different exponents, from a per-layer permutation.
    - The q rows of every in_proj_weight get 1.5, its k rows 6 and its v rows 3: the q sub-packs (13) differ from
      the whole in_proj and the k | v sub-packs (11), and a decoder's v sub-pack (12) differs from both.  CLIP's
      q_proj / k_proj / v_proj get the same magnitudes.
    - A GRU's weight_ih_l0, weight_ih_l0_reverse and its W_hh (both directions are one pack) get three different
      exponents.
    - Every other packed weight gets a seeded one of the three.  Tables (see ``is_packed``) are left alone."""
    g = torch.Generator().manual_seed(seed)
    out = {k: v.clone() for k, v in sd.items()}
    done = set()
    for k in sorted(out):
        if k in done or not is_packed(k, out[k]):
            continue
        for ffn1, ffn2 in (("linear1.weight", "linear2.weight"), ("mlp.fc1.weight", "mlp.fc2.weight")):
            if k.endswith(ffn1):
                p = k[:-len(ffn1)]
                trio = (p + "self_attn.out_proj.weight", k, p + ffn2)
                for key, mag in zip(trio, _perm(g)):
                    _plant(out[key], slice(None), mag, g)
                    done.add(key)
    for k in sorted(out):
        if k in done or not is_packed(k, out[k]):
            continue
        t = out[k]
        if k.endswith("in_proj_weight"):
            d = t.shape[0] // 3
            for rows, mag in ((slice(0, d), 1.5), (slice(d, 2 * d), 6.0), (slice(2 * d, 3 * d), 3.0)):
                _plant(t, rows, mag, g)
        elif re.search(r"self_attn\.[qkv]_proj\.weight$", k):
            _plant(t, slice(None), {"q": 1.5, "k": 6.0, "v": 3.0}[k[-len("q_proj.weight")]], g)
        elif k.endswith("gru.weight_ih_l0"):
            p = k[:-len("weight_ih_l0")]
            perm = _perm(g)
            for key, mag in zip((p + "weight_ih_l0", p + "weight_ih_l0_reverse"), perm[:2]):
                _plant(out[key], slice(None), mag, g)
                done.add(key)
            for key in (p + "weight_hh_l0", p + "weight_hh_l0_reverse"):
                _plant(out[key], slice(None), perm[2], g)
                done.add(key)
        elif "gru.weight_" in k:
            continue                                    # planted with its weight_ih_l0 above
        else:
            _plant(t, slice(None), list(OUTLIERS)[int(torch.randint(0, 3, (1,), generator=g))], g)
        done.add(k)
    return out


def _last_encoder_layers(sd):
    """Prefixes of the last layer of each encoder stack: the engine packs that layer's q rows and k | v rows of
    in_proj as two more operands (pack_trimmed_qkv)."""
    last = {}
    for k in sd:
        if not k.endswith("self_attn.in_proj_weight"):
            continue
        p = k[:-len("self_attn.in_proj_weight")]
        m = _LAYER.match(p)
        if m is None or p + "multihead_attn.in_proj_weight" in sd:
            continue
        kind, _, i = m.group(2).partition(".")
        rank = (_BLOCK_ORDER[kind], int(i or 0))
        if m.group(1) not in last or rank > last[m.group(1)][0]:
            last[m.group(1)] = (rank, p)
    return {p for _, p in last.values()}


def packed_exponents(sd):
    """{pack: exponent} for every operand the engine packs from this state dict, named by its key, with
    ``[q]`` / ``[kv]`` / ``[v]`` for row sub-packs of an in_proj_weight, ``...self_attn.qkv`` for CLIP's concatenated
    q | k | v and ``...gru.weight_hh`` for a GRU's two W_hh.  The exponents are what ``engine_exponent`` gives the
    pack's rows, as ``pack_linear`` computes them (a conv weight's permutation and zero padding change no max)."""
    trimmed = _last_encoder_layers(sd)
    out = {}
    for k, t in sd.items():
        if not is_packed(k, t):
            continue
        if k.endswith("multihead_attn.in_proj_weight"):
            d = t.shape[0] // 3
            out[k + "[q]"] = engine_exponent(t[:d])
            out[k + "[kv]"] = engine_exponent(t[d:])
            out[k + "[v]"] = engine_exponent(t[2 * d:])
        elif k.endswith("self_attn.in_proj_weight"):
            out[k] = engine_exponent(t)
            if k[:-len("self_attn.in_proj_weight")] in trimmed:
                d = t.shape[0] // 3
                out[k + "[q]"] = engine_exponent(t[:d])
                out[k + "[kv]"] = engine_exponent(t[d:])
        elif re.search(r"self_attn\.[qkv]_proj\.weight$", k):
            p = k[:-len("q_proj.weight")]
            out[p + "qkv"] = engine_exponent(torch.cat([sd[p + n + "_proj.weight"] for n in "qkv"]))
        elif "gru.weight_hh_l0" in k:
            p = k[:k.index("weight_hh_l0")]
            out[p + "weight_hh"] = engine_exponent(torch.cat([sd[p + "weight_hh_l0"], sd[p + "weight_hh_l0_reverse"]]))
        else:
            out[k] = engine_exponent(t)
    return out
