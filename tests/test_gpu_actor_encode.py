"""The ActorVae encoder on the GPU (pytest -m gpu): ``mldb_vae_encode`` for ``MLDB_VAE_ACTOR`` and
``B200ActorVae.encode`` against the reference's own ``ActorVae.encode`` (tests/golden/vae_actor_encode.npz) and the
oracle in float64.

Tolerance: 2e-4 relative to the max (OP_TOL), the single-operator bound of test_gpu_parity.py: fp32 re-association
plus the ~22-bit split-fp16 storage of the activations."""
import pytest
import torch

from conftest import golden
from mld_b200 import synth
from oracle import mld_oracle as O
from oracle.actor_encode import actor_encode
from oracle.make_golden_actor_encode import CASES, NFEATS, WEIGHT_SEED, case_motion
from test_gpu_isolation import _assert_isolated, _positions

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

OP_TOL = 2e-4
POISONS = (float("nan"), float("inf"), float("-inf"), 1e30)


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _cfg(layers):
    return O.VaeCfg(kind="actor", nfeats=NFEATS, num_layers=layers)


def _engine(sd, layers):
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(vae="actor", num_layers=0, vae_layers=layers, vae_nfeats=NFEATS, nfeats=NFEATS), 0)
    eng.load_state_dict(sd, "vae.")
    eng.finalize()
    return eng


@pytest.fixture(scope="module")
def actor(built_lib):
    sd = synth.actor_vae_state_dict(seed=WEIGHT_SEED)
    return _engine(sd, 6), sd


@pytest.fixture(scope="module")
def actor1(built_lib):
    sd = synth.actor_vae_state_dict(seed=778, num_layers=1)
    return _engine(sd, 1), sd


def _motion(B, T, seed):
    return torch.randn(B, T, NFEATS, generator=torch.Generator().manual_seed(seed))


def _oracle64(sd, layers, motion, lengths):
    sd64 = {k: v.double() for k, v in sd.items()}
    return actor_encode(sd64, _cfg(layers), motion.double(), lengths)


def _check(mu, logvar, ref_mu, ref_logvar, tol=OP_TOL):
    assert _rel(mu, ref_mu) < tol
    assert _rel(logvar.exp().pow(0.5), ref_logvar.exp().pow(0.5)) < tol


# ------------------------------------------------------------------ against the reference and float64
@pytest.mark.parametrize("tag", sorted(CASES))
def test_actor_encode_vs_reference_golden(actor, tag):
    """Case a: 62 keys; case b: 152 keys and a one-frame sequence."""
    eng, _ = actor
    g = golden("vae_actor_encode.npz")
    lengths = list(CASES[tag][2])
    mu, logvar = eng.vae_encode(case_motion(tag), lengths)
    assert mu.shape == logvar.shape == (1, len(lengths), 256)
    assert _rel(mu[0], g[f"{tag}_mu"]) < OP_TOL
    assert _rel(logvar[0].exp().pow(0.5), g[f"{tag}_std"]) < OP_TOL


@pytest.mark.parametrize("layers", [1, 6])
def test_actor_encode_vs_float64(actor, actor1, layers):
    eng, sd = actor if layers == 6 else actor1
    lengths = [60, 33, 1, 59]
    motion = _motion(4, 60, seed=70 + layers)
    _check(*eng.vae_encode(motion, lengths), *_oracle64(sd, layers, motion, lengths))


@pytest.mark.parametrize("T", [126, 254, 255])
def test_actor_encode_attention_boundaries(actor, T):
    """T + 2 = 128, 256 and 257 keys: the largest wgmma attention tiles, then the CUDA-core fallback."""
    eng, sd = actor
    lengths = [T, T // 2 + 1]
    motion = _motion(2, T, seed=T)
    eng.kernel_stats(reset=True)
    mu, logvar = eng.vae_encode(motion, lengths)
    st = eng.kernel_stats()
    _check(mu, logvar, *_oracle64(sd, 6, motion, lengths))
    if T + 2 <= 256:
        assert st["attn_tc"] == 6 and st["attn_simt"] == 0 and st["attn_mma"] == 0, st
    else:   # the 5 full-length layers fall back to CUDA cores; the trimmed last layer may fit the mma.sync core
        assert st["attn_simt"] >= 5 and st["attn_simt"] + st["attn_mma"] == 6 and st["attn_tc"] == 0, st


def test_actor_encode_long_sequences(actor):
    """The sine PE table has 5000 rows: T + 2 <= 5000 is accepted, T = 4999 is refused."""
    eng, sd = actor
    lengths = [1000, 377]
    motion = _motion(2, 1000, seed=1000)
    mu, logvar = eng.vae_encode(motion, lengths)
    _check(mu, logvar, *actor_encode(sd, _cfg(6), motion, lengths))
    mu, logvar = eng.vae_encode(_motion(1, 4998, seed=4998), [4998])
    assert torch.isfinite(mu).all() and torch.isfinite(logvar).all()
    with pytest.raises(RuntimeError, match="status 1"):
        eng.vae_encode(torch.zeros(1, 4999, NFEATS), [4999])


def test_actor_encode_kernel_stats_and_cuda_core_path(actor):
    """At T = 60 every operator runs on the tensor cores; gemm=simt runs the same math on CUDA cores."""
    eng, sd = actor
    lengths = [60, 40, 12]
    motion = _motion(3, 60, seed=60)
    ref = actor_encode(sd, _cfg(6), motion, lengths)
    eng.kernel_stats(reset=True)
    eng.vae_encode(motion, lengths)
    st = eng.kernel_stats(reset=True)
    assert st["attn_tc"] == 6, st
    assert st["gemm_simt"] == st["attn_simt"] == st["attn_mma"] == st["ln_unfused"] == 0, st
    for opt, val in (("gemm", "simt"), ("attn", "simt"), ("attn", "mma")):
        eng.set_option(opt, val)
        try:
            _check(*eng.vae_encode(motion, lengths), *ref)
        finally:
            eng.set_option("gemm", "tc")
            eng.set_option("attn", "tc")


# ------------------------------------------------------------------ isolation, determinism, batch invariance
def test_actor_encode_isolation(actor):
    """A poison in one sequence's valid frames reaches no other sequence; finite garbage in any sequence's padding
    frames changes no output bit (the reference's output does not depend on them either)."""
    eng, _ = actor
    B, T = 5, 60
    lengths = [60, 41, 1, 17, 60]
    feats = _motion(B, T, seed=5).cuda()
    clean = [t.clone() for t in eng.vae_encode(feats, lengths)]
    for p in _positions(B):
        for v in POISONS:
            f = feats.clone()
            f[p, :lengths[p]] = v
            _assert_isolated(clean, list(eng.vae_encode(f, lengths)), [1, 1], p, f"actor encode, poison {v}")
    g = torch.Generator().manual_seed(6)
    for garbage in (lambda n: 100.0 * torch.randn(n, NFEATS, generator=g), lambda n: torch.full((n, NFEATS), -1e3)):
        f = feats.clone()
        for b, n in enumerate(lengths):
            f[b, n:] = garbage(T - n).cuda()
        out = eng.vae_encode(f, lengths)
        assert all(torch.equal(c, o) for c, o in zip(clean, out))


def test_actor_encode_deterministic_and_batch_invariant(actor):
    eng, _ = actor
    B, T = 512, 60
    lengths = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(8)).tolist()
    lengths[0] = T
    feats = _motion(B, T, seed=9).cuda()
    idx = [0, 1, 255, 511]
    first = [t.clone() for t in eng.vae_encode(feats, lengths)]
    assert all(torch.equal(a, b) for a, b in zip(first, eng.vae_encode(feats, lengths)))
    # the default hidden-dimension split of the FFN sums leftover tiles piecewise, by batch size
    for i in idx:
        alone = eng.vae_encode(feats[i:i + 1], [lengths[i]])
        for a, b in zip(alone, first):
            assert _rel(a[:, 0], b[:, i]) < 1e-5
    eng.set_option("ffn_split", "0")
    try:
        big = [t.clone() for t in eng.vae_encode(feats, lengths)]
        for i in idx:
            alone = eng.vae_encode(feats[i:i + 1], [lengths[i]])
            assert all(torch.equal(a[:, 0], b[:, i]) for a, b in zip(alone, big)), i
    finally:
        eng.set_option("ffn_split", "1")


# ------------------------------------------------------------------ the key-spec rule
def test_actor_encoder_keys_all_or_none(actor):
    eng_full, sd = actor
    dec_only = {k: v for k, v in sd.items() if not k.startswith("encoder.")}
    eng = _engine(dec_only, 6)
    z = synth.init_noise(3, seed=51).permute(1, 0, 2).contiguous()
    assert torch.equal(eng.vae_decode(z, [60, 40, 12]), eng_full.vae_decode(z, [60, 40, 12]))
    with pytest.raises(RuntimeError, match=r"status 3\).*encoder"):
        eng.vae_encode(_motion(1, 8, seed=1), [8])
    from mld_b200.engine import Engine, make_config
    for drop in ("encoder.logvar_token", "encoder.seqTransEncoder.layers.5.norm2.bias"):
        part = Engine(make_config(vae="actor", num_layers=0, vae_layers=6, vae_nfeats=NFEATS, nfeats=NFEATS), 0)
        part.load_state_dict({k: v for k, v in sd.items() if k != drop}, "vae.")
        with pytest.raises(RuntimeError, match=f"status 3\\).*'vae.{drop}'"):
            part.finalize()


# ------------------------------------------------------------------ the drop-in module
def test_actor_dropin_encode_forward_and_a2m_round_trip(actor):
    from types import SimpleNamespace
    from mld_b200.modules import B200ActorVae
    eng, sd = actor
    vae = B200ActorVae(ablation=SimpleNamespace(), nfeats=NFEATS, latent_dim=[1, 256], num_layers=6)
    vae.load_state_dict(sd, strict=True)
    vae = vae.cuda()
    lengths = [60, 40, 12]
    x = case_motion("a").cuda()
    for s in (0, 123):
        torch.manual_seed(s)
        z, dist = vae.encode(x, lengths)
        torch.manual_seed(s)
        eps = torch.empty(3, 256, device="cuda").normal_()            # the draw Normal.rsample makes
        assert z.shape == (1, 3, 256) and dist.loc.shape == dist.scale.shape == (3, 256)
        assert _rel(z[0], dist.loc + eps * dist.scale) < 1e-6
    mu, logvar = eng.vae_encode(x, lengths)
    assert torch.equal(dist.loc, mu[0]) and torch.equal(dist.scale, logvar[0].exp().pow(0.5))
    z, _ = vae.encode(x)                                               # lengths=None: every length is T
    assert z.shape == (1, 3, 256)
    feats, z, dist = vae(x, lengths)
    assert feats.shape == (3, 60, NFEATS) and z.shape == (1, 3, 256)
    assert torch.equal(feats, vae.decode(z, lengths))
    # MLD.a2m_eval, stage vae (mld.py:721-729): decode the encoded motion
    rec = vae.decode(dist.loc[None], lengths)
    mu64, _ = _oracle64(sd, 6, x.cpu(), lengths)
    sd64 = {k: v.double() for k, v in sd.items()}
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)        # the oracle's decoder builds its queries in the default dtype
    try:
        rec64 = O.vae_decode(sd64, _cfg(6), mu64, lengths)
    finally:
        torch.set_default_dtype(prev)
    assert _rel(rec, rec64) < OP_TOL
