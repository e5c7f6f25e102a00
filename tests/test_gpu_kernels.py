"""GPU kernel unit tests (pytest -m gpu): each GEMM epilogue of the wgmma kernel against a
float64 torch reference of the same op, and against the CUDA-core kernel, through the C ABI's
debug hook.  Tolerance 5e-6 relative-to-max: the split-fp16 3-product scheme keeps ~22 bits."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture(scope="module")
def eng(built_lib):
    from mld_b200.engine import Engine, make_config
    return Engine(make_config(num_layers=0, vae="none"), 0)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max())


CASES = [
    # M,    N,    K,    K1,  act, ln
    (200, 768, 256, 0, 0, False),       # QKV projection, ragged M tail
    (1000, 1024, 256, 0, 1, False),     # FFN up-projection + exact GELU
    (333, 256, 1024, 0, 0, True),       # FFN down-projection + residual + LayerNorm (fused epilogue)
    (640, 256, 256, 0, 0, True),        # attention out-projection + residual + LayerNorm
    (515, 256, 512, 256, 0, False),     # skip connection: cat([x, skip]) @ W^T as two A sources
    (392, 263, 256, 0, 0, False),       # final layer: N not a tile multiple (TMA zero fill)
    (129, 512, 256, 0, 2, False),       # kv projection, ReLU epilogue variant
    (4096, 1024, 256, 0, 3, False),     # many tiles, SiLU
    (1300, 256, 1024, 0, 0, True),      # 11 m-tiles: cluster groups with an out-of-range m-tile, LN epilogue
    (1100, 263, 512, 256, 0, False),    # clusters + ragged N + two A sources
]


@pytest.mark.parametrize("M,N,K,K1,act,ln", CASES)
def test_tc_gemm_epilogues(eng, M, N, K, K1, act, ln):
    g = torch.Generator().manual_seed(M * 7 + N)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) * (1.0 / K ** 0.5)
    bias = torch.randn(N, generator=g) * 0.1
    ref = F.linear(A.double(), W.double(), bias.double())
    kw = {}
    if ln:
        R = torch.randn(M, N, generator=g)
        gamma, beta = 1 + 0.1 * torch.randn(N, generator=g), 0.1 * torch.randn(N, generator=g)
        ref = F.layer_norm(ref + R.double(), (N,), gamma.double(), beta.double(), 1e-5)
        kw = dict(gamma=gamma, beta=beta, R=R)
    else:
        ref = {0: lambda x: x, 1: F.gelu, 2: F.relu, 3: F.silu}[act](ref)
    y_tc = eng.debug_gemm(A, W, bias, K1=K1, act=act, use_tc=True, **kw)
    y_cc = eng.debug_gemm(A, W, bias, K1=K1, act=act, use_tc=False, **kw)
    assert torch.isfinite(y_tc).all()
    assert _rel(y_cc, ref) < 5e-6, "CUDA-core kernel vs float64 reference"
    assert _rel(y_tc, ref) < 5e-6, "wgmma kernel vs float64 reference"
    if not ln and N % 8 == 0:
        # the production epilogue: split16 planes (TMA bulk stores on the CTA-pair kernels)
        y_sp = eng.debug_gemm(A, W, bias, K1=K1, act=act, use_tc=True, split_out=True)
        assert _rel(y_sp, ref) < 5e-6, "wgmma kernel, split16 output"


@pytest.mark.parametrize("M,ff", [(100, 1024), (128 * 3 + 5, 1024), (148 * 128 * 2 + 777, 1024), (1000, 512),
                                  (148 * 128 + 20 * 128 - 3, 1024), (148 * 128 + 36 * 128, 512)])
def test_fused_ffn_block(eng, M, ff):
    """k_ffn_tc (hidden activations kept on the SM) vs float64 and vs the unfused operators."""
    d = 256
    g = torch.Generator().manual_seed(M + ff)
    X = torch.randn(M, d, generator=g)
    W1, b1 = torch.randn(ff, d, generator=g) / d ** 0.5, 0.1 * torch.randn(ff, generator=g)
    W2, b2 = torch.randn(d, ff, generator=g) / ff ** 0.5, 0.1 * torch.randn(d, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)
    Xd = X.double()
    hid = F.gelu(F.linear(Xd, W1.double(), b1.double()))
    ref = F.layer_norm(Xd + F.linear(hid, W2.double(), b2.double()), (d,), gamma.double(), beta.double(), 1e-5)
    ys = [eng.debug_ffn(X, W1, b1, W2, b2, gamma, beta, mode=m).cpu().double() for m in (0, 1, 2)]
    for name, y in zip(("cuda-core", "tc unfused", "tc fused"), ys):
        assert torch.isfinite(y).all(), name
        assert _rel(y, ref) < 5e-6, name
    assert _rel(ys[2], ys[1]) < 4e-6
    # every size above leaves tile groups that do not fill a round of the persistent grid: the fused kernel cut
    # them along the hidden dimension (ffn_split, partial accumulators through scratch + flags).  Without the
    # split the same rows are summed in one piece; with it, repeated launches are bit-identical.
    eng.set_option("ffn_split", "0")
    y_whole = eng.debug_ffn(X, W1, b1, W2, b2, gamma, beta, mode=2).cpu().double()
    eng.set_option("ffn_split", "1")
    assert _rel(y_whole, ref) < 5e-6 and _rel(y_whole, ys[2]) < 4e-6
    assert torch.equal(eng.debug_ffn(X, W1, b1, W2, b2, gamma, beta, mode=2).cpu().double(), ys[2])


def test_whole_path_tc_equals_cuda_core_path(built_lib):
    """The same 6-step sample through both GEMM paths agrees to fp32 re-association noise."""
    from mld_b200 import synth
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(), 0)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
    eng.finalize()
    eng.set_mean_std(*synth.mean_std())
    eng.set_timesteps(6)
    ctx, noise = synth.text_context(3, 77, seed=5), synth.init_noise(3, seed=6)
    lengths = [196, 64, 120]
    a = eng.sample(ctx, noise, lengths, want=("latents", "joints"))
    l_tc = eng.launch_count
    eng.set_option("gemm", "simt")
    b = eng.sample(ctx, noise, lengths, want=("latents", "joints"))
    assert _rel(a["latents"], b["latents"]) < 1e-4
    assert _rel(a["joints"], b["joints"]) < 1e-4
    assert l_tc > 0


def test_scheduling_options_do_not_change_results(built_lib):
    """Engine scheduling options only reorder independent work: CUDA-graph replay vs eager launches must give
    bit-identical motions, and so must the number of concurrent sub-batch branches once the fused FFN's
    hidden-dimension split is off (with it, the rows of the tile groups that do not fill a round are summed
    piecewise, and which rows those are depends on how the batch is cut); the split itself, the unfused FFN
    (same math, the hidden activations round-trip HBM) and the other attention cores agree to fp32
    re-association noise.  Repeated runs are bit-identical in every configuration."""
    from mld_b200 import synth
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(), 0)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
    eng.finalize()
    eng.set_mean_std(*synth.mean_std())
    eng.set_timesteps(4)
    B = 300                                   # 600 sequences x 79 tokens = 371 m-tiles: > 2 waves + ragged tail
    ctx, noise = synth.text_context(B, 77, seed=15), synth.init_noise(B, seed=16)
    lengths = [196] * B
    base = eng.sample(ctx, noise, lengths, want=("latents",))["latents"].clone()
    assert torch.isfinite(base).all()
    eng.set_option("graph", "0")
    assert torch.equal(eng.sample(ctx, noise, lengths, want=("latents",))["latents"], base), "graph replay vs eager"
    eng.set_option("graph", "1")
    eng.set_option("ffn_split", "0")
    whole = eng.sample(ctx, noise, lengths, want=("latents",))["latents"].clone()
    assert _rel(whole, base) < 1e-5, "ffn_split"
    for value in ("1", "3"):
        eng.set_option("branches", value)
        out = eng.sample(ctx, noise, lengths, want=("latents",))["latents"]
        assert torch.equal(out, whole), f"branches={value} changed the result"
    eng.set_option("ffn_split", "1")
    for value in ("1", "3"):
        eng.set_option("branches", value)
        out = eng.sample(ctx, noise, lengths, want=("latents",))["latents"]
        assert _rel(out, base) < 1e-5, f"branches={value} with the split"
    eng.set_option("branches", "2")
    eng.set_option("ffn_fused", "0")
    out = eng.sample(ctx, noise, lengths, want=("latents",))["latents"]
    assert _rel(out, base) < 1e-5
    eng.set_option("ffn_fused", "1")
    for kind in ("mma", "simt"):
        eng.set_option("attn", kind)
        out = eng.sample(ctx, noise, lengths, want=("latents",))["latents"]
        assert _rel(out, base) < 1e-5, kind
    eng.set_option("attn", "tc")
    # repeated runs are bit-identical (no atomics anywhere on the path)
    assert torch.equal(eng.sample(ctx, noise, lengths, want=("latents",))["latents"], base)


def _attention_ref(q, k, v, nseq, Lq, Lk, heads, nk=None):
    """float64 reference: q [nseq*Lq, d], k / v [nseq*Lk, d]; nk[s] valid keys of sequence s."""
    d = q.shape[1]
    hd = d // heads
    qh = q.reshape(nseq, Lq, heads, hd).permute(0, 2, 1, 3).double()
    kh = k.reshape(nseq, Lk, heads, hd).permute(0, 2, 1, 3).double()
    vh = v.reshape(nseq, Lk, heads, hd).permute(0, 2, 1, 3).double()
    s = qh @ kh.transpose(-1, -2) / hd ** 0.5
    if nk is not None:
        mask = torch.arange(Lk)[None, :] >= torch.as_tensor(nk)[:, None]
        s = s.masked_fill(mask[:, None, None, :], float("-inf"))
    return (torch.softmax(s, -1) @ vh).permute(0, 2, 1, 3).reshape(nseq * Lq, d)


SELF_ATTN_CASES = [
    # nseq, L, hd, masked        (heads = 4)
    (3, 79, 64, False),          # denoiser sequence: 2 key blocks (64 + 16), two score buffers
    (5, 79, 64, True),
    (300, 79, 64, False),        # > 148 CTAs x several items: persistent loop, both softmax groups, ring wrap
    (7, 3, 64, False),           # action model / pooled context: 3 tokens
    (2, 128, 64, False),         # exactly one query tile, two full key blocks
    (4, 33, 64, True),
    (8, 196, 64, True),          # VAE decoder: two query tiles, 4 key blocks (208 keys), one score buffer
    (5, 198, 64, True),          # VAE encoder: 2 distribution tokens + 196 frames
    (3, 60, 64, True),           # ActorVae
    (6, 196, 128, False),        # no-VAE denoiser (d = 512): two 64-wide slices of the head, one Q buffer
    (3, 79, 128, True),
    (2, 256, 64, False),         # the largest key count the score row fits (the score row lives in registers)
    (256, 196, 64, True),        # VAE decode at the benchmark batch: many items per CTA on ONE score buffer
    (90, 196, 128, False),       # ... and with head_dim 128
    (400, 130, 64, True),        # three key blocks on two score buffers
]


@pytest.mark.parametrize("nseq,L,hd,masked", SELF_ATTN_CASES)
def test_self_attention_kernels(eng, nseq, L, hd, masked):
    """The attention cores in isolation on the packed q|k|v layout of the stacks, against float64: wgmma
    (product), mma.sync and CUDA cores.  5e-6 relative-to-max: the split-fp16 scheme keeps ~22 bits."""
    heads = 4
    d = heads * hd
    g = torch.Generator().manual_seed(nseq * 131 + L + hd)
    qkv = torch.randn(nseq * L, 3 * d, generator=g)
    lengths = [max(1, (7 * i + 5) % L) for i in range(nseq)] if masked else None
    ref = _attention_ref(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], nseq, L, L, heads, lengths)
    for mode, name in ((2, "wgmma"), (1, "mma.sync"), (0, "cuda-core")):
        if mode == 1 and (hd == 128 and L > 128 or L < 8):
            continue                       # outside the mma.sync kernel's shared-memory budget / tile shape
        y = eng.debug_attention(qkv, nseq, L, heads, lengths, mode=mode).cpu().double()
        assert torch.isfinite(y).all(), name
        assert _rel(y, ref) < 5e-6, name


CROSS_ATTN_CASES = [
    # nseq, Lq, Lk, hd, kv_prefix, masked
    (300, 1, 79, 64, 0, False),   # trimmed last denoiser layer: one query row per sequence
    (4, 2, 198, 64, 2, True),     # trimmed last VAE-encoder layer: 2 queries, 2 always-on tokens + masked frames
    (5, 196, 2, 128, 0, False),   # no-VAE denoiser cross-attention: 2 memory tokens (time, text)
    (3, 60, 1, 64, 0, False),     # one memory token
    (2, 130, 70, 64, 0, True),
]


@pytest.mark.parametrize("nseq,Lq,Lk,hd,prefix,masked", CROSS_ATTN_CASES)
def test_cross_attention_kernels(eng, nseq, Lq, Lk, hd, prefix, masked):
    heads = 4
    d = heads * hd
    g = torch.Generator().manual_seed(nseq * 17 + Lq * 3 + Lk)
    q = torch.randn(nseq * Lq, d, generator=g)
    kv = torch.randn(nseq * Lk, 2 * d, generator=g)
    lengths = [max(1, (11 * i + 3) % (Lk - prefix)) for i in range(nseq)] if masked else None
    nk = None if lengths is None else [min(Lk, prefix + n) for n in lengths]
    ref = _attention_ref(q, kv[:, :d], kv[:, d:], nseq, Lq, Lk, heads, nk)
    for mode, name in ((2, "wgmma"), (0, "cuda-core")):
        y = eng.debug_attention(q, nseq, Lq, heads, lengths, mode=mode, kv=kv, Lk=Lk, kv_prefix=prefix).cpu().double()
        assert torch.isfinite(y).all(), name
        assert _rel(y, ref) < 5e-6, name


def test_product_path_runs_on_tcgen05(built_lib):
    """Kernel-choice introspection (mldb_kernel_stats): the text-to-motion path enqueues its GEMMs, FFN blocks
    and attention on the tensor-core kernels (wgmma on this architecture; the test keeps its first name) - no
    CUDA-core attention, no LayerNorm split off a GEMM."""
    from mld_b200 import synth
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(), 0)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
    eng.finalize()
    eng.set_mean_std(*synth.mean_std())
    eng.set_timesteps(2)
    ctx, noise = synth.text_context(8, 77, seed=5), synth.init_noise(8, seed=6)
    eng.kernel_stats(reset=True)
    eng.sample(ctx, noise, [196, 64, 120, 33, 196, 100, 7, 150], want=("joints",))
    st = eng.kernel_stats()
    assert st["attn_tc"] > 0 and st["ffn_tc"] > 0 and st["gemm_ln_tc"] > 0 and st["gemm_tc"] > 0
    assert st["attn_simt"] == 0 and st["attn_mma"] == 0 and st["ln_unfused"] == 0, st
    # CUDA-core GEMMs: only the time MLP (2 per set_timesteps) - nothing on the per-step path
    assert st["gemm_simt"] == 0, st
