"""Batch isolation (pytest -m gpu): a NaN, an inf or a value past split16's range (|x| >= 65520 stores hi = inf) in one
batch member must not change any other member's output.  In the reference every motion, prompt and sequence is
computed on its own, and non-finite values do reach the library in normal use: an out-of-range token id gives a NaN
row, and the caller supplies the context, the noise, the motion to encode and the per-step noise.

Each test runs a clean batch, then the same batch with the first, a middle or the last member poisoned, and demands
that every other member's output is bit-identical (``torch.equal``) to the clean run.  The batch is cut the same way
in both runs, so the rows are summed in the same order and bit equality is a fair demand.  The poisoned member itself
may come out non-finite.  The last member matters on its own: its tail is out of bounds for the TMA loads, which
zero-fill there, while every other member's tail is the next member's head."""
import ctypes as C

import pytest
import torch

from mld_b200 import synth
from test_gpu_kernels import CASES, CROSS_ATTN_CASES

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

POISONS = (float("nan"), float("inf"), 1e5)


def _positions(n):
    return sorted({0, n // 2, n - 1})


def _assert_isolated(clean, poisoned, members, p, what):
    """clean / poisoned: lists of tensors whose dim ``members[i]`` indexes the batch member."""
    for c, y, dim in zip(clean, poisoned, members):
        c, y = c.movedim(dim, 0), y.movedim(dim, 0)
        keep = [i for i in range(c.shape[0]) if i != p]
        assert torch.isfinite(c[keep]).all(), f"{what}: the clean run is not finite"
        bad = [i for i in keep if not torch.equal(c[i], y[i])]
        assert not bad, (f"{what}: poisoning member {p} changed members {bad} "
                         f"(non-finite in {[i for i in bad if not torch.isfinite(y[i]).all()]})")


@pytest.fixture(scope="module")
def eng(built_lib):
    from mld_b200.engine import Engine, make_config
    return Engine(make_config(num_layers=0, vae="none"), 0)


# ------------------------------------------------------------------ attention cores
# mode 0 CUDA-core, 1 mma.sync, 2 wgmma (product)
def _mma_ok(Lk, hd, causal):
    return not causal and Lk >= 8 and (hd == 64 or Lk <= 128)


SELF_CASES = [
    # L, causal, masked
    (3, False, False),       # action denoiser: 3 tokens, 13 padding rows in the only key block
    (60, False, True),       # ActorVae: 4 padding rows
    (77, True, False),       # CLIP text tower: 3 padding rows
    (79, False, False),      # denoiser: 1 padding row
    (130, False, True),
    (196, False, True),      # VAE decoder: 12 padding rows
    (198, False, True),      # VAE encoder: 10 padding rows
    (256, False, False),     # no padding at all
]


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("L,causal,masked", SELF_CASES)
def test_self_attention_isolation(eng, L, causal, masked, hd):
    nseq, heads = 5, 4
    d = heads * hd
    g = torch.Generator().manual_seed(L * 3 + hd)
    qkv = torch.randn(nseq * L, 3 * d, generator=g).cuda()
    lengths = [max(1, (7 * i + 5) % L) for i in range(nseq)] if masked else None
    for mode in (0, 1, 2):
        if mode == 1 and not _mma_ok(L, hd, causal):
            continue
        run = lambda x: eng.debug_attention(x, nseq, L, heads, lengths, mode=mode, causal=causal).view(nseq, L, d)
        clean = run(qkv).clone()
        for p in _positions(nseq):
            for v in POISONS:
                x = qkv.clone()
                x[p * L:(p + 1) * L] = v
                _assert_isolated([clean], [run(x)], [0], p, f"mode {mode}, poison {v}")


@pytest.mark.parametrize("hd_override", [None, 128])
@pytest.mark.parametrize("nseq,Lq,Lk,hd,prefix,masked", CROSS_ATTN_CASES)
def test_cross_attention_isolation(eng, nseq, Lq, Lk, hd, prefix, masked, hd_override):
    hd = hd_override or hd
    heads = 4
    d = heads * hd
    g = torch.Generator().manual_seed(nseq * 17 + Lq * 3 + Lk)
    q = torch.randn(nseq * Lq, d, generator=g).cuda()
    kv = torch.randn(nseq * Lk, 2 * d, generator=g).cuda()
    lengths = [max(1, (11 * i + 3) % (Lk - prefix)) for i in range(nseq)] if masked else None
    for mode in (0, 1, 2):
        if mode == 1 and not _mma_ok(Lk, hd, False):
            continue
        run = lambda a, b: eng.debug_attention(a, nseq, Lq, heads, lengths, mode=mode, kv=b, Lk=Lk,
                                               kv_prefix=prefix).view(nseq, Lq, d)
        clean = run(q, kv).clone()
        for p in _positions(nseq):
            for v in POISONS:
                a, b = q.clone(), kv.clone()
                a[p * Lq:(p + 1) * Lq] = v
                b[p * Lk:(p + 1) * Lk] = v
                _assert_isolated([clean], [run(a, b)], [0], p, f"mode {mode}, poison {v}")


# ------------------------------------------------------------------ GEMMs and the fused FFN
def _row_blocks(M, n=5):
    """Cut M rows into n members of nearly equal size: [(r0, r1)]."""
    cut = [M * i // n for i in range(n + 1)]
    return [(cut[i], cut[i + 1]) for i in range(n)]


def _by_member(y, blocks):
    # pad each member's rows to the same count so the members stack along dim 0
    n = max(r1 - r0 for r0, r1 in blocks)
    out = torch.zeros((len(blocks), n) + tuple(y.shape[1:]), dtype=y.dtype, device=y.device)
    for i, (r0, r1) in enumerate(blocks):
        out[i, :r1 - r0] = y[r0:r1]
    return out


@pytest.mark.parametrize("M,N,K,K1,act,ln", CASES)
def test_gemm_epilogue_isolation(eng, M, N, K, K1, act, ln):
    g = torch.Generator().manual_seed(M * 7 + N)
    A = torch.randn(M, K, generator=g).cuda()
    W = torch.randn(N, K, generator=g) * (1.0 / K ** 0.5)
    bias = torch.randn(N, generator=g) * 0.1
    R = torch.randn(M, N, generator=g).cuda()
    kw = dict(gamma=1 + 0.1 * torch.randn(N, generator=g), beta=0.1 * torch.randn(N, generator=g), R=R) if ln else {}
    blocks = _row_blocks(M)
    variants = [dict(use_tc=True), dict(use_tc=False)]
    if not ln and N % 8 == 0:
        variants.append(dict(use_tc=True, split_out=True))
    for var in variants:
        clean = eng.debug_gemm(A, W, bias, K1=K1, act=act, **kw, **var).clone()
        for p in _positions(len(blocks)):
            r0, r1 = blocks[p]
            for v in POISONS:
                x = A.clone()
                x[r0:r1] = v
                pk = dict(kw)
                if ln:
                    pk["R"] = R.clone()
                    pk["R"][r0:r1] = v
                y = eng.debug_gemm(x, W, bias, K1=K1, act=act, **pk, **var)
                _assert_isolated([_by_member(clean, blocks)], [_by_member(y, blocks)], [0], p, f"{var}, poison {v}")


@pytest.mark.parametrize("M,N,K", [(385, 768, 768), (333, 768, 3072)])
def test_residual_add_isolation(eng, M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    A, R = torch.randn(M, K, generator=g).cuda(), torch.randn(M, N, generator=g).cuda()
    W, b = torch.randn(N, K, generator=g) / K ** 0.5, 0.1 * torch.randn(N, generator=g)
    blocks = _row_blocks(M)
    for tc in (True, False):
        for in_place in (False, True):
            clean = eng.debug_gemm(A, W, b, R=R, use_tc=tc, in_place=in_place).clone()
            for p in _positions(len(blocks)):
                r0, r1 = blocks[p]
                for v in POISONS:
                    x, r = A.clone(), R.clone()
                    x[r0:r1] = v
                    r[r0:r1] = v
                    y = eng.debug_gemm(x, W, b, R=r, use_tc=tc, in_place=in_place)
                    _assert_isolated([_by_member(clean, blocks)], [_by_member(y, blocks)], [0], p,
                                     f"tc {tc}, in_place {in_place}, poison {v}")


@pytest.mark.parametrize("M,ff", [(1000, 1024), (148 * 128 + 20 * 128 - 3, 1024)])
def test_ffn_isolation(eng, M, ff):
    """Both sizes leave tile groups that the fused kernel cuts along the hidden dimension (ffn_split)."""
    d = 256
    g = torch.Generator().manual_seed(M + ff)
    X = torch.randn(M, d, generator=g).cuda()
    W1, b1 = torch.randn(ff, d, generator=g) / d ** 0.5, 0.1 * torch.randn(ff, generator=g)
    W2, b2 = torch.randn(d, ff, generator=g) / ff ** 0.5, 0.1 * torch.randn(d, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    blocks = _row_blocks(M)
    for mode in (0, 1, 2):
        clean = eng.debug_ffn(X, W1, b1, W2, b2, gamma, beta, mode=mode).clone()
        for p in _positions(len(blocks)):
            r0, r1 = blocks[p]
            for v in POISONS:
                x = X.clone()
                x[r0:r1] = v
                y = eng.debug_ffn(x, W1, b1, W2, b2, gamma, beta, mode=mode)
                _assert_isolated([_by_member(clean, blocks)], [_by_member(y, blocks)], [0], p,
                                 f"mode {mode}, poison {v}")


# ------------------------------------------------------------------ entry points
VOCAB, EOS, POISON_ID = 1000, 999, 777


@pytest.fixture(scope="module")
def tower(built_lib):
    """A two-layer CLIP-L/14-shaped text tower whose embedding row POISON_ID is 1e5."""
    from mld_b200 import _lib
    from mld_b200.engine import Engine, make_config
    tc = _lib.default_text_config()
    tc.vocab_size, tc.eos_token_id, tc.layers = VOCAB, EOS, 2
    e = Engine(make_config(num_layers=0, vae="none"), 0)
    e.text_configure(tc)
    sd = synth.clip_text_state_dict(99, vocab_size=VOCAB, max_positions=tc.max_positions, hidden=tc.hidden,
                                    layers=2, ff=tc.ff, projection_dim=tc.projection_dim)
    sd["text_model.text_model.embeddings.token_embedding.weight"][POISON_ID] = 1e5
    e.load_state_dict(sd, "text_encoder.")
    e.finalize()
    return e


def _text_encode_raw(e, ids, mode):
    """mldb_text_encode without the wrapper's id check: an id outside the vocabulary gives a NaN row."""
    from mld_b200 import _lib
    n, L = ids.shape
    tc = e.text_cfg
    out = torch.empty((n, L, tc.hidden) if mode == _lib.TEXT_HIDDEN else (n, tc.projection_dim),
                      dtype=torch.float32, device=e.device)
    d_ids = ids.to(device=e.device, dtype=torch.int64).contiguous()
    _lib.check(e.lib.mldb_text_encode(e._h, C.c_void_p(d_ids.data_ptr()), n, L, int(mode),
                                      C.c_void_p(out.data_ptr()), e._stream()), "mldb_text_encode")
    return out


@pytest.mark.parametrize("poison", ["out_of_range_id", "embedding_1e5"])
def test_text_tower_isolation(tower, poison):
    from mld_b200 import _lib
    n, L = 5, 77
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, VOCAB - 1, (n, L), generator=g)
    ids[ids == POISON_ID] = 1
    for i in range(n):
        ids[i, 5 + 9 * i] = EOS
    for mode in (_lib.TEXT_HIDDEN, _lib.TEXT_POOLED):
        clean = _text_encode_raw(tower, ids, mode).clone()
        for p in _positions(n):
            x = ids.clone()
            if poison == "out_of_range_id":
                x[p, 0] = VOCAB
            else:
                x[p, 0] = x[p, 3] = POISON_ID
            _assert_isolated([clean], [_text_encode_raw(tower, x, mode)], [0], p, f"text mode {mode}")


@pytest.fixture(scope="module")
def mld(built_lib):
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(), 0)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
    eng.finalize()
    eng.set_mean_std(*synth.mean_std())
    eng.set_timesteps(3)
    return eng


@pytest.mark.parametrize("S", [1, 77])
def test_denoise_isolation(mld, S):
    Bx = 6
    ctx, x = synth.text_context(Bx // 2, S, seed=11).cuda(), synth.init_noise(Bx, seed=12).cuda()   # [Bx, S, 768]
    lengths = [196, 100, 40, 196, 7, 150]
    clean = mld.denoise(x, 501, ctx, lengths).clone()
    for p in _positions(Bx):
        for v in POISONS:
            c, z = ctx.clone(), x.clone()
            c[p] = v
            z[p] = v
            _assert_isolated([clean], [mld.denoise(z, 501, c, lengths)], [0], p, f"poison {v}")


def test_vae_isolation(mld):
    B = 5
    lengths = [196, 120, 8, 60, 196]
    z = synth.init_noise(B, seed=41).permute(1, 0, 2).contiguous().cuda()
    clean = mld.vae_decode(z, lengths).clone()
    feats = torch.randn(B, 196, 263, generator=torch.Generator().manual_seed(42)).cuda()
    mu0, lv0 = (t.clone() for t in mld.vae_encode(feats, lengths))
    for p in _positions(B):
        for v in POISONS:
            zz = z.clone()
            zz[:, p] = v
            _assert_isolated([clean], [mld.vae_decode(zz, lengths)], [0], p, f"vae_decode, poison {v}")
            f = feats.clone()
            f[p, :lengths[p]] = v                      # inside the valid frames
            _assert_isolated([mu0, lv0], list(mld.vae_encode(f, lengths)), [1, 1], p, f"vae_encode, poison {v}")


@pytest.mark.parametrize("graph", ["1", "0"])
def test_sample_isolation(mld, graph):
    B = 5
    lengths = [196, 64, 120, 33, 196]
    ctx, noise = synth.text_context(B, 77, seed=15).cuda(), synth.init_noise(B, seed=16).cuda()     # ctx [2B, 77, 768]
    want = ("latents", "joints")
    mld.set_option("graph", graph)
    try:
        clean = [t.clone() for t in mld.sample(ctx, noise, lengths, want=want).values()]
        for p in _positions(B):
            for v in POISONS:
                c, z = ctx.clone(), noise.clone()
                c[p] = c[B + p] = v                    # both guidance halves of member p
                z[p] = v
                out = mld.sample(c, z, lengths, want=want)
                _assert_isolated(clean, [out["latents"], out["joints"]], [1, 0], p, f"graph {graph}, poison {v}")
    finally:
        mld.set_option("graph", "1")


def test_step_noise_isolation(built_lib):
    """DDIM at eta = 1: one sample's per-step noise stays in that sample."""
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(eta=1.0), 0)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
    eng.finalize()
    eng.set_mean_std(*synth.mean_std())
    n = len(eng.set_timesteps(4))
    B = 5
    lengths = [196, 64, 120, 33, 196]
    ctx, noise = synth.text_context(B, 77, seed=25).cuda(), synth.init_noise(B, seed=26).cuda()
    sn = torch.randn(n, B, 1, 256, generator=torch.Generator().manual_seed(27)).cuda()
    want = ("latents", "joints")
    clean = [t.clone() for t in eng.sample(ctx, noise, lengths, want=want, step_noise=sn).values()]
    for p in _positions(B):
        for v in POISONS:
            s = sn.clone()
            s[:, p] = v
            out = eng.sample(ctx, noise, lengths, want=want, step_noise=s)
            _assert_isolated(clean, [out["latents"], out["joints"]], [1, 0], p, f"poison {v}")


def test_novae_denoiser_isolation(built_lib):
    """The no-VAE trans_dec denoiser: d = 512 (head_dim 128), self-attention over the frames, cross-attention to the
    time and text tokens."""
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(arch="trans_dec", latent_dim=(1, 512), diffusion_only=True, vae="none"), 0)
    eng.load_state_dict(synth.denoiser_state_dict(seed=3456, arch="trans_dec", d=512, diffusion_only=True),
                        "denoiser.")
    eng.finalize()
    Bx, T = 6, 60
    lengths = [60, 44, 60, 12, 60, 31]
    x = torch.randn(Bx, T, 263, generator=torch.Generator().manual_seed(31)).cuda()
    ctx = synth.text_context(Bx // 2, 1, seed=32).cuda()
    clean = eng.denoise(x, 501, ctx, lengths).clone()
    for p in _positions(Bx):
        for v in POISONS:
            z, c = x.clone(), ctx.clone()
            z[p, :lengths[p]] = v
            c[p] = v
            _assert_isolated([clean], [eng.denoise(z, 501, c, lengths)], [0], p, f"poison {v}")


def test_action_denoiser_isolation(built_lib):
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(condition="action", num_layers=15, nclasses=12, nfeats=150, vae="none"), 0)
    eng.load_state_dict(synth.denoiser_state_dict(seed=2345, condition="action", num_layers=15, nclasses=12,
                                                  nfeats=150), "denoiser.")
    eng.finalize()
    Bx = 6
    cond = torch.tensor([[0], [0], [0], [3], [7], [11]])
    x = synth.init_noise(Bx, seed=22).cuda()
    clean = eng.denoise(x, 501, cond, [60] * Bx).clone()
    for p in _positions(Bx):
        for v in POISONS:
            z = x.clone()
            z[p] = v
            _assert_isolated([clean], [eng.denoise(z, 501, cond, [60] * Bx)], [0], p, f"poison {v}")
