"""GPU: every model path with weights whose packs sit at split16 exponents 11-13 instead of 14 (pytest -m gpu).

``with_outliers`` (tests/weight_scales.py) sets a few elements of each packed weight to +-1.5, +-3 or +-6, so that
within a layer the out-projection and the two FFN weights, an in_proj's q rows and its k | v rows, and a GRU's
input and recurrent weights all pack at different exponents, while the model stays the synthetic one.  Each test
first checks those exponents, then runs the path against its oracle with the gate the path's own tests use: 2e-4 for
single operators (test_gpu_parity.py), 1e-3 on the joints of a sampling loop, 1e-4 per row for the CLIP tower
(test_gpu_text.py), the T2M gates of test_gpu_t2m.py."""
import pytest
import torch

from mld_b200 import _lib, synth
from oracle import mld_oracle as O
from oracle import t2m_eval as T2M
from oracle.actor_encode import actor_encode
from oracle.clip_text import ClipTextCfg, clip_text_forward
from weight_scales import OUTLIERS, packed_exponents, with_outliers

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

OP_TOL = 2e-4


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _rel_rows(a, b):
    a, b = a.double().cpu().flatten(1), b.double().cpu().flatten(1)
    return float(((a - b).abs().max(1).values / b.abs().max(1).values).max())


def _gate(name, err, tol=OP_TOL):
    print(f"[weight-scales models] {name}: {err:.2e} (gate {tol:.0e})")
    assert err < tol, (name, err)


def _joint_err(joints, ref_list, lengths):
    return max(_rel(joints[b, :n], ref_list[b]) for b, n in enumerate(lengths))


def _spread(sd):
    """The state dict's packs are all off 14, and use all three exponents."""
    ex = packed_exponents(sd)
    assert set(ex.values()) == set(OUTLIERS.values()), sorted(set(ex.values()))
    return ex


def _engine(cfg_kw, *sds):
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(**cfg_kw), 0)
    for sd, prefix in sds:
        eng.load_state_dict(sd, prefix)
    eng.finalize()
    return eng


@pytest.fixture(scope="module")
def text_model(built_lib):
    dsd = with_outliers(synth.denoiser_state_dict(1234), seed=1)
    vsd = with_outliers(synth.mld_vae_state_dict(4321), seed=2)
    eng = _engine({}, (dsd, "denoiser."), (vsd, "vae."))
    mean, std = synth.mean_std()
    eng.set_mean_std(mean, std)
    return dict(eng=eng, dsd=dsd, vsd=vsd, mean=mean, std=std)


# ------------------------------------------------------------------ text denoiser and MldVae
@pytest.mark.parametrize("S", [77, 1])
@pytest.mark.parametrize("B", [1, 8])
def test_text_denoiser(text_model, B, S):
    """Up to 2 m-tiles (one prompt, or eight with S = 1) the encoder layers run the fused tail, three scales in one
    launch; past that (eight prompts, S = 77) the out-projection + LayerNorm GEMM and the fused FFN."""
    eng, dsd = text_model["eng"], text_model["dsd"]
    ex = _spread(dsd)
    assert ex["encoder.middle_block.self_attn.out_proj.weight"] != ex["encoder.middle_block.linear1.weight"]
    lengths = synth.ragged_lengths(B, seed=S + B) * 2
    ctx = synth.text_context(B, S, seed=11 + B)
    x = synth.init_noise(B, seed=12 + S).repeat(2, 1, 1)
    for t in (981, 1):
        eng.kernel_stats(reset=True)
        y = eng.denoise(x, t, ctx, lengths)
        torch.cuda.synchronize()
        st = eng.kernel_stats()
        yo = O.denoiser_forward(dsd, O.DenoiserCfg(), x, torch.tensor(t), ctx, lengths)
        _gate(f"text denoiser B={B} S={S} t={t}", _rel(y, yo))
        assert st["ffn_tc"] > 0 and st["ln_unfused"] == 0, st
        fused = (2 * B * (S + 2) + 127) // 128 <= 2             # tokens: the latent, the time token, S text tokens
        assert (st["gemm_ln_tc"] == 0) == fused, st


def test_mld_vae_decode_and_encode(text_model):
    eng, vsd = text_model["eng"], text_model["vsd"]
    ex = _spread(vsd)
    ca = "decoder.middle_block.multihead_attn.in_proj_weight"
    assert ex[ca + "[q]"] != ex[ca + "[kv]"]
    lengths = [196, 120, 8]
    z = synth.init_noise(3, seed=41).permute(1, 0, 2).contiguous()
    feats = eng.vae_decode(z, lengths)
    _gate("MldVae decode", _rel(feats, O.vae_decode(vsd, O.VaeCfg(), z, lengths)))
    assert float(feats[1, 120:].abs().max()) == 0.0
    motion = torch.randn(3, 196, 263, generator=torch.Generator().manual_seed(42))
    mu, logvar = eng.vae_encode(motion, lengths)
    mo, lo = O.vae_encode(vsd, O.VaeCfg(), motion, lengths)
    _gate("MldVae encode mu", _rel(mu, mo))
    _gate("MldVae encode std", _rel(logvar.exp().pow(0.5), lo.exp().pow(0.5)))


@pytest.mark.parametrize("gemm", ["tc", "simt"])
def test_ragged_sampling_loop(text_model, gemm):
    """10 guided DDIM steps on ragged lengths, decode and joints, against the oracle; the time MLP runs on the
    CUDA-core GEMM either way, and gemm=simt sends every GEMM there."""
    eng = text_model["eng"]
    B, S, steps = 6, 5, 10
    lengths = synth.ragged_lengths(B, seed=3)
    ctx, noise = synth.text_context(B, S, seed=81), synth.init_noise(B, seed=82)
    eng.set_timesteps(steps)
    eng.set_option("gemm", gemm)
    try:
        out = eng.sample(ctx, noise, lengths, want=("joints",))
    finally:
        eng.set_option("gemm", "tc")
    jo, _, _ = O.mld_forward(text_model["dsd"], O.DenoiserCfg(), text_model["vsd"], O.VaeCfg(), O.DDIMScheduler(),
                             steps, ctx, noise, lengths, text_model["mean"], text_model["std"])
    err = _joint_err(out["joints"], jo, lengths)
    _gate(f"sampling loop joints gemm={gemm}", err, 1e-3)


# ------------------------------------------------------------------ no-VAE denoiser (decoder layers, d = 512)
def test_novae_denoiser(built_lib):
    nsd = with_outliers(synth.denoiser_state_dict(seed=3456, arch="trans_dec", d=512, diffusion_only=True), seed=3)
    ex = _spread(nsd)
    p = "decoder.layers.4.multihead_attn.in_proj_weight"
    assert len({ex[p + "[q]"], ex[p + "[kv]"], ex[p + "[v]"]}) == 3
    eng = _engine(dict(arch="trans_dec", latent_dim=(1, 512), diffusion_only=True, vae="none", scheduler="ddpm"),
                  (nsd, "denoiser."))
    lengths = [196, 132] * 2
    x = torch.randn(2, 196, 263, generator=torch.Generator().manual_seed(231)).repeat(2, 1, 1)
    ctx = synth.text_context(2, 1, seed=232)
    y = eng.denoise(x, 777, ctx, lengths)
    cfg = O.DenoiserCfg(arch="trans_dec", latent_dim=512, diffusion_only=True)
    _gate("no-VAE denoiser", _rel(y, O.denoiser_forward(nsd, cfg, x, torch.tensor(777), ctx, lengths)))
    assert float(y[1, 132:].abs().max()) == 0.0


# ------------------------------------------------------------------ action model and ActorVae
def test_action_denoiser(built_lib):
    asd = with_outliers(synth.denoiser_state_dict(seed=2345, condition="action", num_layers=15, nclasses=12,
                                                  nfeats=150), seed=4)
    _spread(asd)
    eng = _engine(dict(condition="action", num_layers=15, nclasses=12, nfeats=150, vae="none"), (asd, "denoiser."))
    actions = torch.randint(0, 12, (3, 1), generator=torch.Generator().manual_seed(21))
    cond = torch.cat([torch.zeros_like(actions), actions])
    x = synth.init_noise(3, seed=22).repeat(2, 1, 1)
    cfg = O.DenoiserCfg(condition="action", num_layers=15, nclasses=12, nfeats=150)
    for t in (501, 1):
        y = eng.denoise(x, t, cond, [60] * 6)
        _gate(f"action denoiser t={t}", _rel(y, O.denoiser_forward(asd, cfg, x, torch.tensor(t), cond, [60] * 6)))


def test_actor_vae_encode_and_decode(built_lib):
    avsd = with_outliers(synth.actor_vae_state_dict(seed=777), seed=5)
    ex = _spread(avsd)
    last = "encoder.seqTransEncoder.layers.5.self_attn.in_proj_weight"
    assert ex[last + "[q]"] != ex[last]
    eng = _engine(dict(vae="actor", num_layers=0, vae_layers=6, vae_nfeats=150, nfeats=150), (avsd, "vae."))
    cfg = O.VaeCfg(kind="actor", nfeats=150, num_layers=6)
    lengths = [60, 41, 1]
    motion = torch.randn(3, 60, 150, generator=torch.Generator().manual_seed(61))
    mu, logvar = eng.vae_encode(motion, lengths)
    sd64 = {k: v.double() for k, v in avsd.items()}
    mo, lo = actor_encode(sd64, cfg, motion.double(), lengths)
    _gate("ActorVae encode mu", _rel(mu, mo))
    _gate("ActorVae encode std", _rel(logvar.exp().pow(0.5), lo.exp().pow(0.5)))
    z = synth.init_noise(3, seed=51).permute(1, 0, 2).contiguous()
    feats = eng.vae_decode(z, [60, 40, 12])
    _gate("ActorVae decode", _rel(feats, O.vae_decode(avsd, cfg, z, [60, 40, 12])))
    assert float(feats[2, 12:].abs().max()) == 0.0


# ------------------------------------------------------------------ CLIP text tower
def test_clip_tower(built_lib):
    from oracle.make_golden_clip import WEIGHT_SEED
    sd = with_outliers(synth.clip_text_state_dict(WEIGHT_SEED), seed=6)
    _spread(sd)
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    eng.text_configure(_lib.default_text_config())
    eng.load_state_dict(sd, "text_encoder.")
    eng.finalize()
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    ids = synth.clip_text_ids(40, 77, seed=17)
    cfg = ClipTextCfg()
    hid = eng.text_encode(ids, _lib.TEXT_HIDDEN)
    pooled = eng.text_encode(ids, _lib.TEXT_POOLED)
    err_h = _rel_rows(hid, clip_text_forward(sd64, ids.cuda(), "clip_hidden", cfg))
    err_p = _rel_rows(pooled, clip_text_forward(sd64, ids.cuda(), "clip", cfg)[:, 0])
    _gate("CLIP hidden", err_h, 1e-4)
    _gate("CLIP pooled", err_p, 1e-4)


# ------------------------------------------------------------------ T2M evaluator
@pytest.fixture(scope="module")
def t2m(built_lib):
    from mld_b200.engine import Engine, make_config
    from oracle.make_golden_t2m import WEIGHT_SEED
    plain = synth.t2m_state_dicts(WEIGHT_SEED)
    sds = {k: with_outliers(plain[k], seed=7 + i) for i, k in enumerate(sorted(plain))}
    eng = Engine(make_config(num_layers=0, vae="none"), 0)
    eng.t2m_configure(_lib.default_t2m_config())
    for k, prefix in (("text_encoder", "t2m_textencoder."), ("movement_encoder", "t2m_moveencoder."),
                      ("motion_encoder", "t2m_motionencoder.")):
        eng.load_state_dict(sds[k], prefix)
    eng.finalize()
    return eng, sds, {k: {kk: vv.double().cuda() for kk, vv in v.items()} for k, v in sds.items()}


def test_t2m_movement(t2m):
    eng, sds, sd64 = t2m
    ex = packed_exponents(sds["movement_encoder"])
    assert 14 not in ex.values()
    x = torch.randn(5, 196, 259, generator=torch.Generator().manual_seed(5)).cuda()
    err = _rel_rows(eng.t2m_movement(x), T2M.movement(sd64["movement_encoder"], x.double()))
    _gate("T2M movement", err, 2e-5)


def _ragged(B, L, seed):
    ln = torch.randint(1, L + 1, (B,), generator=torch.Generator().manual_seed(seed))
    ln[0], ln[-1] = L, 1
    return ln


def test_t2m_motion(t2m):
    eng, sds, sd64 = t2m
    ex = _spread(sds["motion_encoder"])
    assert len({ex["gru.weight_hh"], ex["gru.weight_ih_l0"], ex["gru.weight_ih_l0_reverse"]}) == 3
    B, L = 37, 49
    x = (torch.randn(B, L, 512, generator=torch.Generator().manual_seed(B)) * 0.5).cuda()
    ln = _ragged(B, L, B)
    err = _rel_rows(eng.t2m_motion(x, ln), T2M.motion(sd64["motion_encoder"], x.double(), ln.tolist()))
    _gate("T2M motion", err, 5e-5)


def test_t2m_text(t2m):
    eng, sds, sd64 = t2m
    ex = _spread(sds["text_encoder"])
    assert len({ex["gru.weight_hh"], ex["gru.weight_ih_l0"], ex["gru.weight_ih_l0_reverse"]}) == 3
    B, L = 37, 22
    w, p = synth.t2m_text_inputs(B, L, seed=L)
    ln = _ragged(B, L, L + 1)
    err = _rel_rows(eng.t2m_text(w.cuda(), p.cuda(), ln), T2M.text(sd64["text_encoder"], w.double().cuda(),
                                                                    p.double().cuda(), ln.tolist()))
    _gate("T2M text", err, 2e-5)
