"""GPU tests of the shapes the API accepts beyond the shipped configs (pytest -m gpu).

The rule under test: a shape the API accepts runs and matches a float64 reference (or the in-repo oracle);
a shape it cannot run is refused up front.  No kernel may fail at launch or leave stale output behind.

- The attention cores at the kernel level: the CUDA-core core (the last-resort fallback) at any key count and
  head size, and the documented limits of the mma.sync and wgmma cores.
- Long sequences through the model entry points (no-VAE denoiser, MldVae, ActorVae, feats2joints, a short
  sample through the captured graph) against ``oracle.mld_oracle``, with the attention core that ran read
  back from the kernel statistics.
- CLIP text towers of other shapes than ViT-L/14 against ``oracle.clip_text`` in float64, on both GEMM paths.
"""
import pytest
import torch

from mld_b200 import synth
from oracle import mld_oracle as O
from oracle.clip_text import ClipTextCfg, clip_text_forward

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ATTN_TOL = 5e-6      # one attention core vs float64 (the kernel suite's split-fp16 bound)
OP_TOL = 2e-4        # one model operator vs the fp32 oracle (as in test_gpu_parity.py)
# 1-2 layer text towers vs float64, per sequence, relative to max: the widest per-op bound on the way, the wgmma
# GEMM's 5e-6 per 1024 of K at K = 4096 (fc2 of hidden 1024).  Measured worst on an H100: 1.2e-5 (hidden 1024).
TOWER_TOL = 2e-5


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _rel_rows(a, b):
    return max(_rel(a[i], b[i]) for i in range(a.shape[0]))


@pytest.fixture(scope="module")
def eng(built_lib):
    from mld_b200.engine import Engine, make_config
    return Engine(make_config(num_layers=0, vae="none"), 0)


def _attention_ref(q, k, v, nseq, Lq, Lk, heads, nk=None, causal=False):
    """float64 softmax(q k^T / sqrt(hd)) v: q [nseq*Lq, d], k / v [nseq*Lk, d]; nk[s] valid keys of sequence s;
    causal: query i sees keys j <= i."""
    d = q.shape[1]
    hd = d // heads
    qh, kh, vh = (t.reshape(nseq, -1, heads, hd).permute(0, 2, 1, 3).double() for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) / hd ** 0.5
    mask = torch.zeros(nseq, Lq, Lk, dtype=torch.bool)
    if nk is not None:
        mask |= (torch.arange(Lk)[None, :] >= torch.as_tensor(nk)[:, None])[:, None, :]
    if causal:
        mask |= torch.ones(Lq, Lk, dtype=torch.bool).triu(1)[None]
    s = s.masked_fill(mask[:, None], float("-inf"))
    return (torch.softmax(s, -1) @ vh).permute(0, 2, 1, 3).reshape(nseq * Lq, d)


def _self_attention_case(nseq, L, heads, hd, masked, causal, seed):
    d = heads * hd
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(nseq * L, 3 * d, generator=g)
    lengths = [max(1, L - 37 * i - 5) for i in range(nseq)] if masked else None
    ref = _attention_ref(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], nseq, L, L, heads, lengths, causal)
    return qkv, lengths, ref


# ------------------------------------------------------------------ attention cores, kernel level
CUDA_CORE_CASES = [
    # hd, L: the CUDA-core core must run every key count, whatever its shared memory holds at once
    (64, 256), (64, 300), (64, 421), (64, 500), (64, 1000),
    (128, 215), (128, 216), (128, 300), (128, 500),
    (32, 100), (32, 700),
    (96, 77), (96, 300),
    (256, 107), (256, 108), (256, 300),
    (512, 52), (512, 77),
]


@pytest.mark.parametrize("variant", ["plain", "masked", "causal"])
@pytest.mark.parametrize("hd,L", CUDA_CORE_CASES)
def test_cuda_core_attention_any_length(eng, hd, L, variant):
    nseq, heads = 2, 2
    qkv, lengths, ref = _self_attention_case(nseq, L, heads, hd, variant == "masked", variant == "causal",
                                             seed=hd * 1009 + L)
    y = eng.debug_attention(qkv, nseq, L, heads, lengths, mode=0, causal=variant == "causal").cpu()
    assert torch.isfinite(y).all()
    assert _rel(y, ref) < ATTN_TOL


@pytest.mark.parametrize("Lk,hd", [(1000, 64), (500, 128)])
def test_cuda_core_cross_attention_long_memory(eng, Lk, hd):
    """Two query rows over a long masked key range with always-on prefix keys (the trimmed last layer of the
    VAE encoder)."""
    nseq, Lq, heads, prefix = 3, 2, 4, 2
    d = heads * hd
    g = torch.Generator().manual_seed(Lk + hd)
    q = torch.randn(nseq * Lq, d, generator=g)
    kv = torch.randn(nseq * Lk, 2 * d, generator=g)
    lengths = [Lk - prefix, Lk // 3, 1]
    nk = [min(Lk, prefix + n) for n in lengths]
    ref = _attention_ref(q, kv[:, :d], kv[:, d:], nseq, Lq, Lk, heads, nk)
    y = eng.debug_attention(q, nseq, Lq, heads, lengths, mode=0, kv=kv, Lk=Lk, kv_prefix=prefix).cpu()
    assert _rel(y, ref) < ATTN_TOL


def test_cuda_core_attention_refuses_what_it_cannot_hold(eng):
    """A head too wide for one query row per warp in shared memory is refused, not launched."""
    hd = 4096
    qkv = torch.randn(1, 3 * hd)
    with pytest.raises(RuntimeError, match="status 4"):
        eng.debug_attention(qkv, 1, 1, 1, mode=0)


TC_LIMITS = [
    # mode, hd, L, runs: 2 = wgmma (Lk <= 256, hd 64 / 128); 1 = mma.sync (shared-memory bound, Lk >= 8, no causal)
    (2, 64, 256, True), (2, 64, 257, False), (2, 128, 256, True), (2, 128, 257, False),
    (2, 96, 64, False), (2, 32, 64, False),
    (1, 64, 256, True), (1, 64, 257, False), (1, 128, 128, True), (1, 128, 129, False),
    (1, 64, 7, False), (1, 256, 64, False),
]


@pytest.mark.parametrize("mode,hd,L,runs", TC_LIMITS)
def test_tensor_core_attention_limits(eng, mode, hd, L, runs):
    """Inside its limits a tensor-core attention core matches float64; just past them it is refused with
    MLDB_ERR_UNSUPPORTED (the engine then falls back to the next core)."""
    nseq, heads = 2, 4
    qkv, lengths, ref = _self_attention_case(nseq, L, heads, hd, True, False, seed=mode * 7919 + hd + L)
    if not runs:
        with pytest.raises(RuntimeError, match="status 4"):
            eng.debug_attention(qkv, nseq, L, heads, lengths, mode=mode)
        return
    y = eng.debug_attention(qkv, nseq, L, heads, lengths, mode=mode).cpu()
    assert _rel(y, ref) < ATTN_TOL


# ------------------------------------------------------------------ long sequences, model level
def _loaded_engine(make, *state):
    eng = make()
    for sd, prefix in state:
        eng.load_state_dict(sd, prefix)
    eng.finalize()
    return eng


@pytest.fixture(scope="module")
def novae(built_lib):
    from mld_b200.engine import Engine, make_config
    nsd = synth.denoiser_state_dict(seed=3456, arch="trans_dec", d=512, diffusion_only=True)
    eng = _loaded_engine(lambda: Engine(make_config(arch="trans_dec", latent_dim=(1, 512), diffusion_only=True,
                                                   vae="none", scheduler="ddpm"), 0), (nsd, "denoiser."))
    eng.set_option("graph", "0")             # eager: the kernel statistics count every call
    return eng, nsd


@pytest.mark.parametrize("gemm", ["tc", "simt"])
@pytest.mark.parametrize("T", [216, 257, 300, 500])
def test_novae_denoiser_long_sequences(novae, T, gemm):
    """d = 512 (head_dim 128), T up to the 500-row PE table, ragged lengths.  Past 256 frames the self-attention
    leaves the wgmma core for the CUDA-core core; the 2-token cross-attention stays on wgmma."""
    eng, nsd = novae
    lengths = [T, T * 2 // 3] * 2
    gen = torch.Generator().manual_seed(T)
    x = torch.randn(2, T, 263, generator=gen).repeat(2, 1, 1)
    ctx = synth.text_context(2, 1, seed=T + 1)
    eng.set_option("gemm", gemm)
    try:
        eng.kernel_stats(reset=True)
        y = eng.denoise(x, 777, ctx, lengths)
        st = eng.kernel_stats()
    finally:
        eng.set_option("gemm", "tc")
    cfg = O.DenoiserCfg(arch="trans_dec", latent_dim=512, diffusion_only=True)
    yo = O.denoiser_forward(nsd, cfg, x, torch.tensor(777), ctx, lengths)
    assert _rel(y, yo) < OP_TOL
    assert float(y[1, lengths[1]:].abs().max()) == 0.0
    layers = cfg.num_layers
    if gemm == "simt":
        assert st["attn_simt"] == 2 * layers and st["attn_tc"] == 0 and st["attn_mma"] == 0, st
    elif T <= 256:
        assert st["attn_tc"] == 2 * layers and st["attn_simt"] == 0, st
    else:
        assert st["attn_simt"] == layers and st["attn_tc"] == layers and st["attn_mma"] == 0, st


@pytest.fixture(scope="module")
def mldvae(built_lib):
    from mld_b200.engine import Engine, make_config
    vsd = synth.mld_vae_state_dict(4321)
    eng = _loaded_engine(lambda: Engine(make_config(num_layers=0), 0), (vsd, "vae."))
    eng.set_mean_std(*synth.mean_std())
    eng.set_option("graph", "0")
    return eng, vsd


@pytest.mark.parametrize("T", [257, 421, 500])
def test_mld_vae_decode_long(mldvae, T):
    eng, vsd = mldvae
    lengths = [T, T // 2 + 1]
    z = synth.init_noise(2, seed=T).permute(1, 0, 2).contiguous()
    eng.kernel_stats(reset=True)
    feats = eng.vae_decode(z, lengths)
    st = eng.kernel_stats()
    assert _rel(feats, O.vae_decode(vsd, O.VaeCfg(), z, lengths)) < OP_TOL
    assert float(feats[1, lengths[1]:].abs().max()) == 0.0
    assert st["attn_simt"] == 9 and st["attn_tc"] == 0 and st["attn_mma"] == 0, st   # 9 self-attentions


@pytest.mark.parametrize("T", [257, 419, 498])
def test_mld_vae_encode_long(mldvae, T):
    eng, vsd = mldvae
    lengths = [T, T // 3]
    gen = torch.Generator().manual_seed(T)
    motion = torch.randn(2, T, 263, generator=gen)
    eng.kernel_stats(reset=True)
    mu, logvar = eng.vae_encode(motion, lengths)
    st = eng.kernel_stats()
    mo, lo = O.vae_encode(vsd, O.VaeCfg(), motion, lengths)
    assert _rel(mu, mo) < OP_TOL
    assert _rel(logvar.exp().pow(0.5), lo.exp().pow(0.5)) < OP_TOL
    # T + 2 keys: the 8 full-length layers fall back to CUDA cores; the trimmed last layer (2 query rows) may
    # still fit the mma.sync core
    assert st["attn_simt"] >= 8 and st["attn_simt"] + st["attn_mma"] == 9 and st["attn_tc"] == 0, st


def test_mld_vae_refuses_lengths_past_its_pe_table(mldvae):
    eng, _ = mldvae
    with pytest.raises(RuntimeError, match="status 1"):
        eng.vae_decode(synth.init_noise(1, seed=1).permute(1, 0, 2).contiguous(), [501])
    with pytest.raises(RuntimeError, match="status 1"):
        eng.vae_encode(torch.zeros(1, 499, 263), [499])


def test_actor_vae_decode_1000_frames(built_lib):
    """ActorVae's sine PE has 5000 rows: T = 1000 is accepted and must run."""
    from mld_b200.engine import Engine, make_config
    avsd = synth.actor_vae_state_dict(seed=777)
    eng = _loaded_engine(lambda: Engine(make_config(vae="actor", num_layers=0, vae_layers=6, vae_nfeats=150,
                                                   nfeats=150), 0), (avsd, "vae."))
    lengths = [1000, 333]
    z = synth.init_noise(2, seed=53).permute(1, 0, 2).contiguous()
    eng.kernel_stats(reset=True)
    feats = eng.vae_decode(z, lengths)
    st = eng.kernel_stats()
    fo = O.vae_decode(avsd, O.VaeCfg(kind="actor", nfeats=150, num_layers=6), z, lengths)
    assert _rel(feats, fo) < OP_TOL
    assert float(feats[1, 333:].abs().max()) == 0.0
    assert st["attn_simt"] == 6 and st["attn_tc"] == 0, st


@pytest.mark.parametrize("T", [1025, 4000])
def test_feats2joints_long(mldvae, T):
    eng, _ = mldvae
    mean, std = synth.mean_std()
    gen = torch.Generator().manual_seed(T)
    f = torch.randn(2, T, 263, generator=gen) * 0.3
    j = eng.feats2joints(f)
    jo = O.feats2joints(f, mean, std)
    assert j.shape == (2, T, 22, 3)
    err = max(_rel(j[b], jo[b]) for b in range(2))
    print(f"\n[envelope] feats2joints T={T}: {err:.2e} vs the oracle")
    assert err < OP_TOL


@pytest.mark.parametrize("T", [300, 450])
def test_long_sample_graph_equals_eager(built_lib, T):
    """A few DDIM steps + decode + joints at T frames through the captured graph equal the eager launches
    bit for bit, and the decoded motion matches the oracle's decode of the same latents (no stale rows)."""
    from mld_b200.engine import Engine, make_config
    dsd, vsd = synth.denoiser_state_dict(1234), synth.mld_vae_state_dict(4321)
    eng = _loaded_engine(lambda: Engine(make_config(), 0), (dsd, "denoiser."), (vsd, "vae."))
    eng.set_mean_std(*synth.mean_std())
    eng.set_timesteps(3)
    ctx, noise = synth.text_context(2, 77, seed=T), synth.init_noise(2, seed=T + 1)
    lengths = [T, T // 2]
    want = ("latents", "feats", "joints")
    eng.kernel_stats(reset=True)
    graphed = {k: v.clone() for k, v in eng.sample(ctx, noise, lengths, want=want).items()}
    assert eng.kernel_stats()["attn_simt"] > 0            # the decoder's self-attention fell back
    eng.set_option("graph", "0")
    eager = eng.sample(ctx, noise, lengths, want=want)
    for k in want:
        assert torch.equal(graphed[k], eager[k]), k
    fo = O.vae_decode(vsd, O.VaeCfg(), graphed["latents"].cpu(), lengths)
    assert _rel(graphed["feats"], fo) < OP_TOL


# ------------------------------------------------------------------ CLIP text towers
VOCAB, BOS, EOS = 1000, 998, 999
TOWERS = {
    # name: (config overrides, layers, sequence lengths)
    "clip_b32": (dict(hidden=512, heads=8, ff=2048, projection_dim=512, eos_token_id=2), 2, [77]),   # legacy eos rule
    "clip_l14": (dict(hidden=768, heads=12, ff=3072, projection_dim=768), 1, [77]),
    "clip_h14": (dict(hidden=1024, heads=16, ff=4096, projection_dim=1024), 1, [77]),
    "d128": (dict(hidden=128, heads=2, ff=512, projection_dim=128), 2, [77]),
    "d256_hd128": (dict(hidden=256, heads=2, ff=1024, projection_dim=256), 2, [77]),   # causal wgmma, head_dim 128
    "d384_hd96": (dict(hidden=384, heads=4, ff=1536, projection_dim=384), 2, [77]),    # causal CUDA-core core
    "d640": (dict(hidden=640, heads=10, ff=2560, projection_dim=640), 1, [77]),
    "d896": (dict(hidden=896, heads=14, ff=3584, projection_dim=896), 1, [77]),
    "ff1000": (dict(hidden=256, heads=4, ff=1000, projection_dim=256), 2, [77]),       # generic quick-GELU, CUDA-core fc2
    "proj100": (dict(hidden=256, heads=4, ff=1024, projection_dim=100), 2, [77]),
    "hd256": (dict(hidden=512, heads=2, ff=2048, projection_dim=512, max_positions=128), 1, [107, 128]),
    "hd512": (dict(hidden=1024, heads=2, ff=4096, projection_dim=1024), 1, [77]),
    "pos256": (dict(hidden=256, heads=4, ff=1024, projection_dim=256, max_positions=256), 2, [1, 255, 256]),
}


def _text_engine(over, layers):
    from mld_b200 import _lib
    from mld_b200.engine import Engine, make_config
    tc = _lib.default_text_config()
    tc.vocab_size, tc.eos_token_id, tc.layers = VOCAB, EOS, layers
    for k, v in over.items():
        setattr(tc, k, v)
    e = Engine(make_config(num_layers=0, vae="none"), 0)
    e.text_configure(tc)
    sd = synth.clip_text_state_dict(99, vocab_size=VOCAB, max_positions=tc.max_positions, hidden=tc.hidden,
                                    layers=layers, ff=tc.ff, projection_dim=tc.projection_dim)
    e.load_state_dict(sd, "text_encoder.")
    e.finalize()
    cfg = ClipTextCfg(vocab_size=VOCAB, max_positions=tc.max_positions, hidden=tc.hidden, heads=tc.heads,
                      layers=layers, ff=tc.ff, projection_dim=tc.projection_dim, eos_token_id=tc.eos_token_id)
    return e, sd, cfg


@pytest.mark.parametrize("name", list(TOWERS))
def test_text_tower_shapes_vs_float64(built_lib, name):
    from mld_b200 import _lib
    over, layers, Ls = TOWERS[name]
    e, sd, cfg = _text_engine(over, layers)
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    hd = cfg.hidden // cfg.heads
    worst = 0.0
    for L in Ls:
        ids = synth.clip_text_ids(4, L, seed=L, eos_lo=L // 2, eos_hi=L - 1, vocab_size=VOCAB, bos=BOS, eos=EOS)
        ref_h = clip_text_forward(sd64, ids.cuda(), "clip_hidden", cfg)
        ref_p = clip_text_forward(sd64, ids.cuda(), "clip", cfg)[:, 0]
        for gemm in ("tc", "simt"):
            e.set_option("gemm", gemm)
            e.kernel_stats(reset=True)
            hid = e.text_encode(ids, _lib.TEXT_HIDDEN)
            st = e.kernel_stats()
            pooled = e.text_encode(ids, _lib.TEXT_POOLED)
            assert hid.shape == (4, L, cfg.hidden) and pooled.shape == (4, cfg.projection_dim)
            err = max(_rel_rows(hid, ref_h), _rel_rows(pooled, ref_p))
            worst = max(worst, err)
            assert err < TOWER_TOL, (L, gemm, err)
            if gemm == "tc" and hd in (64, 128):
                assert st["attn_tc"] == layers and st["attn_simt"] == 0, st
            else:
                assert st["attn_simt"] == layers and st["attn_tc"] == 0, st
        e.set_option("gemm", "tc")
    print(f"\n[envelope] text tower {name}: {worst:.2e} vs float64")


@pytest.mark.parametrize("over", [dict(hidden=200, heads=4), dict(hidden=1152, heads=8), dict(hidden=768, heads=5),
                                  dict(max_positions=257)])
def test_text_configure_refuses_what_it_cannot_run(built_lib, over):
    from mld_b200 import _lib
    from mld_b200.engine import Engine, make_config
    tc = _lib.default_text_config()
    for k, v in over.items():
        setattr(tc, k, v)
    e = Engine(make_config(num_layers=0, vae="none"), 0)
    with pytest.raises(RuntimeError, match="status 4"):
        e.text_configure(tc)
