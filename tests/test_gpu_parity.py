"""GPU parity tests (pytest -m gpu): the CUDA path through the C ABI (``mld_b200.engine.Engine``
-> ``libmldb200.so``) against (a) the committed golden fixtures produced by the REFERENCE's own
modules and (b) the CPU oracle on the same seeded inputs.

Tolerances (fp32 path, stated per test): single operators 2e-4 relative-to-max (fp32
re-association + ~22-bit split-fp16 storage), the 50-step guided sampling loop 1e-3 relative on
the final joint positions per motion (north_star), integer scheduler indexing bit-exact.
"""
import numpy as np
import pytest
import torch

from conftest import golden
from mld_b200 import synth
from oracle import mld_oracle as O

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


def _rel(a, b):
    a, b = torch.as_tensor(a).float().cpu(), torch.as_tensor(b).float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _joint_err(joints, ref_list, lengths):
    worst = 0.0
    for b, n in enumerate(lengths):
        a, r = joints[b, :n].cpu(), ref_list[b]
        worst = max(worst, float((a - r).abs().max() / r.abs().max()))
    return worst


@pytest.fixture(scope="module")
def engines(built_lib):
    from mld_b200.engine import Engine, make_config
    assert torch.cuda.is_available()
    dsd, vsd = synth.denoiser_state_dict(1234), synth.mld_vae_state_dict(4321)
    mean, std = synth.mean_std()
    eng = Engine(make_config(), 0)
    eng.load_state_dict(dsd, "denoiser.")
    eng.load_state_dict(vsd, "vae.")
    eng.finalize()
    eng.set_mean_std(mean, std)
    eng.set_timesteps(50)
    return dict(text=eng, dsd=dsd, vsd=vsd, mean=mean, std=std)


# ------------------------------------------------------------------ single operators
@pytest.mark.parametrize("S", [77, 1])
def test_denoiser_forward_vs_reference_golden(engines, S):
    g = golden("denoiser_text.npz")
    ctx = synth.text_context(2, S, seed=11)
    x = synth.init_noise(2, seed=12).repeat(2, 1, 1)
    for t in (981, 1):
        y = engines["text"].denoise(x, t, ctx, [196, 100] * 2)
        assert y.shape == (4, 1, 256)
        assert _rel(y, g[f"S{S}_t{t}"]) < 2e-4


def test_vae_decode_vs_reference_golden(engines):
    g = golden("vae_mld.npz")
    lengths = [196, 120, 8]
    z = synth.init_noise(3, seed=41).permute(1, 0, 2).contiguous()
    feats = engines["text"].vae_decode(z, lengths)
    assert feats.shape == (3, 196, 263)
    assert _rel(feats, g["feats"]) < 2e-4
    # padded frames are exactly zero (mld_vae.py:245)
    assert float(feats[1, 120:].abs().max()) == 0.0 and float(feats[2, 8:].abs().max()) == 0.0


def test_vae_encode_vs_reference_golden(engines):
    g = golden("vae_mld.npz")
    gen = torch.Generator().manual_seed(42)
    motion = torch.randn(3, 196, 263, generator=gen)
    mu, logvar = engines["text"].vae_encode(motion, [196, 120, 8])
    assert mu.shape == (1, 3, 256)
    assert _rel(mu, g["mu"]) < 2e-4
    assert _rel(logvar.exp().pow(0.5), g["std"]) < 2e-4


def test_feats2joints_vs_reference_golden(engines):
    g = golden("feats2joints.npz")
    gen = torch.Generator().manual_seed(61)
    f = torch.randn(2, 196, 263, generator=gen) * 0.3
    j = engines["text"].feats2joints(f)
    assert j.shape == (2, 196, 22, 3)
    assert _rel(j, g["joints"]) < 1e-5


def test_scheduler_integer_indexing_bit_exact_and_step(engines):
    eng = engines["text"]
    ts = eng.set_timesteps(50)
    ref = O.DDIMScheduler()
    ref.set_timesteps(50)
    assert ts.dtype == torch.int64 and torch.equal(ts, ref.timesteps)          # int64 equality
    g = torch.Generator().manual_seed(3)
    x, e = torch.randn(5, 1, 256, generator=g), torch.randn(5, 1, 256, generator=g)
    for t in (981, 501, 1):
        out = eng.scheduler_step(e, t, x).cpu()
        assert torch.equal(out, ref.step(e, t, x))                             # same fp32 op order


def test_action_denoiser_vs_reference_golden(built_lib):
    from mld_b200.engine import Engine, make_config
    g = golden("denoiser_action.npz")
    asd = synth.denoiser_state_dict(seed=2345, condition="action", num_layers=15, nclasses=12, nfeats=150)
    eng = Engine(make_config(condition="action", num_layers=15, nclasses=12, nfeats=150, vae="none"), 0)
    eng.load_state_dict(asd, "denoiser.")
    eng.finalize()
    actions = torch.from_numpy(g["actions"])
    cond = torch.cat([torch.zeros_like(actions), actions])
    x = synth.init_noise(3, seed=22).repeat(2, 1, 1)
    assert _rel(eng.denoise(x, 501, cond, [60] * 6), g["y"]) < 2e-4


def test_actor_vae_decode_vs_reference_golden(built_lib):
    from mld_b200.engine import Engine, make_config
    g = golden("vae_actor.npz")
    avsd = synth.actor_vae_state_dict(seed=777)
    eng = Engine(make_config(vae="actor", num_layers=0, vae_layers=6, vae_nfeats=150, nfeats=150), 0)
    eng.load_state_dict(avsd, "vae.")
    eng.finalize()
    z = synth.init_noise(3, seed=51).permute(1, 0, 2).contiguous()
    feats = eng.vae_decode(z, [60, 40, 12])
    assert _rel(feats, g["feats"]) < 2e-4
    assert float(feats[2, 12:].abs().max()) == 0.0


# ------------------------------------------------------------------ the sampling loop
@pytest.mark.parametrize("S", [77, 1])
def test_sampling_loop_vs_reference_golden(engines, S):
    """BASELINE configs[1]-shaped: 50 guided DDIM steps -> decode -> joints, against the loop run
    with the reference's own modules (tests/golden/loop_S*.npz)."""
    g = golden(f"loop_S{S}.npz")
    lengths = [196, 88]
    ctx, noise = synth.text_context(2, S, seed=71), synth.init_noise(2, seed=72)
    out = engines["text"].sample(ctx, noise, lengths, want=("latents", "feats", "joints"))
    z_ref = torch.from_numpy(g["latents"][-1]).permute(1, 0, 2)
    assert _rel(out["latents"], z_ref) < 1e-3
    assert _rel(out["feats"], g["feats"]) < 1e-3
    jref = torch.from_numpy(g["joints"])
    err = _joint_err(out["joints"], [jref[0, :196], jref[1, :88]], lengths)
    assert err < 1e-3, f"joint positions differ by {err:.3e} relative (gate 1e-3)"
    # the un-fused reverse entry point returns the same latents
    z2 = engines["text"].diffusion_reverse(ctx, noise, lengths)
    assert torch.equal(z2, out["latents"])


def test_ragged_batch_vs_oracle(engines):
    B, S = 6, 5
    lengths = synth.ragged_lengths(B, seed=3)
    ctx, noise = synth.text_context(B, S, seed=81), synth.init_noise(B, seed=82)
    out = engines["text"].sample(ctx, noise, lengths, want=("joints",))
    jo, _, _ = O.mld_forward(engines["dsd"], O.DenoiserCfg(), engines["vsd"], O.VaeCfg(), O.DDIMScheduler(), 50,
                             ctx, noise, lengths, engines["mean"], engines["std"])
    assert _joint_err(out["joints"], jo, lengths) < 1e-3


def test_full_size_batch_invariance_and_oracle_subset(engines):
    """BASELINE configs[2] at full size (B=256, 77-token context, 50 DDIM steps).  Size-independent
    properties: (i) every motion is independent, so motion i of the 256-batch equals the same
    motion sampled in a batch of 4 - bit-exact with whole-tile FFN scheduling (no cross-row arithmetic
    anywhere), to fp32 re-association noise with the default hidden-dimension split of leftover tiles
    (which rows are summed piecewise depends on the batch size); (ii) the oracle on that 4-motion subset
    agrees within the 1e-3 joint gate; (iii) padded frames are zero."""
    eng = engines["text"]
    B, S = 256, 77
    lengths = [196] * B
    lengths[1], lengths[2] = 120, 64
    ctx, noise = synth.text_context(B, S, seed=1), synth.init_noise(B, seed=2)
    idx = [0, 1, 2, 255]
    sub_ctx = torch.cat([ctx[idx], ctx[[B + i for i in idx]]], 0)
    sub_len = [lengths[i] for i in idx]
    small = eng.sample(sub_ctx, noise[idx], sub_len, want=("latents", "feats", "joints"))
    small = {k: v.clone() for k, v in small.items()}
    big = eng.sample(ctx, noise, lengths, want=("latents", "feats", "joints"))
    assert float((big["latents"][:, idx] - small["latents"]).abs().max() / small["latents"].abs().max()) < 1e-4
    assert _joint_err(big["joints"][idx], [small["joints"][i, :n].cpu() for i, n in enumerate(sub_len)], sub_len) < 2e-4
    assert float(big["feats"][1, 120:].abs().max()) == 0.0
    eng.set_option("ffn_split", "0")
    try:
        small0 = {k: v.clone() for k, v in eng.sample(sub_ctx, noise[idx], sub_len, want=("latents", "joints")).items()}
        big0 = eng.sample(ctx, noise, lengths, want=("latents", "joints"))
        assert torch.equal(big0["latents"][:, idx], small0["latents"])
        assert torch.equal(big0["joints"][idx], small0["joints"])
    finally:
        eng.set_option("ffn_split", "1")
    jo, _, _ = O.mld_forward(engines["dsd"], O.DenoiserCfg(), engines["vsd"], O.VaeCfg(), O.DDIMScheduler(), 50,
                             sub_ctx, noise[idx], sub_len, engines["mean"], engines["std"])
    assert _joint_err(small["joints"], jo, sub_len) < 1e-3


def test_host_entry_point_matches_device_entry_point(engines):
    eng = engines["text"]
    B, S, T = 4, 77, 196
    lengths = [196, 64, 196, 100]
    ctx, noise = synth.text_context(B, S, seed=91), synth.init_noise(B, seed=92)
    dev = eng.sample(ctx, noise, lengths, want=("joints",))["joints"].cpu()
    joints = torch.empty((B, T, 22, 3), dtype=torch.float32).pin_memory()
    eng.sample_host(ctx.pin_memory(), noise.pin_memory(), torch.tensor(lengths, dtype=torch.int32).pin_memory(),
                    joints, T)
    torch.cuda.synchronize()
    assert torch.equal(joints, dev)


def test_dropin_modules_and_pipeline(engines):
    """The YAML-target drop-ins and the MLD-surface pipeline give the engine's numbers."""
    from types import SimpleNamespace
    from mld_b200.modules import B200MldDenoiser, B200MldVae
    from mld_b200.pipeline import B200MLD
    abl = SimpleNamespace(SKIP_CONNECT=True, VAE_TYPE="mld", DIFF_PE_TYPE="mld", PE_TYPE="mld", MLP_DIST=False)
    den = B200MldDenoiser(ablation=abl, nfeats=263, condition="text", latent_dim=[1, 256], ff_size=1024,
                          num_layers=9, num_heads=4, arch="trans_enc", text_encoded_dim=768)
    den.load_state_dict(engines["dsd"], strict=True)
    den = den.cuda()
    ctx = synth.text_context(2, 77, seed=11).cuda()
    x = synth.init_noise(2, seed=12).repeat(2, 1, 1).cuda()
    y = den(sample=x, timestep=torch.tensor(981).cuda(), encoder_hidden_states=ctx, lengths=[196, 100] * 2)[0]
    assert torch.equal(y, engines["text"].denoise(x, 981, ctx))
    vae = B200MldVae(ablation=abl, nfeats=263, latent_dim=[1, 256], arch="encoder_decoder").cuda()
    vae.load_state_dict({k: v.cuda() for k, v in engines["vsd"].items()}, strict=True)
    z = synth.init_noise(3, seed=41).permute(1, 0, 2).contiguous().cuda()
    assert torch.equal(vae.decode(z, [196, 120, 8]), engines["text"].vae_decode(z, [196, 120, 8]))
    model = B200MLD(engines["dsd"], engines["vsd"], mean=engines["mean"], std=engines["std"])
    lengths = [196, 88]
    batch = {"length": lengths, "text_emb": synth.text_context(2, 77, seed=71), "init_noise": synth.init_noise(2, seed=72)}
    joints = model(batch)
    assert [tuple(j.shape) for j in joints] == [(196, 22, 3), (88, 22, 3)]
    g = golden("loop_S77.npz")
    jref = torch.from_numpy(g["joints"])
    for a, r in zip(joints, [jref[0, :196], jref[1, :88]]):
        assert float((a - r).abs().max() / r.abs().max()) < 1e-3
    # the diffusers-style step loop through the drop-in scheduler (mld.py:323-346)
    sched = model.scheduler
    lat = batch["init_noise"].cuda() * sched.init_noise_sigma
    ctxg = batch["text_emb"].cuda()
    for t in sched.timesteps[:3]:
        eps = den(sample=torch.cat([lat] * 2), timestep=t, encoder_hidden_states=ctxg, lengths=lengths * 2)[0]
        u, c = eps.chunk(2)
        lat = sched.step(u + 7.5 * (c - u), t, lat, eta=0.0).prev_sample
    assert _rel(lat.cpu(), torch.from_numpy(g["latents"][2])) < 1e-3


# ------------------------------------------------------------------ no-VAE model (BASELINE configs[4] shape)
@pytest.fixture(scope="module")
def novae(built_lib):
    from mld_b200.engine import Engine, make_config
    nsd = synth.denoiser_state_dict(seed=3456, arch="trans_dec", d=512, diffusion_only=True)
    eng = Engine(make_config(arch="trans_dec", latent_dim=(1, 512), diffusion_only=True, vae="none",
                             scheduler="ddpm"), 0)
    eng.load_state_dict(nsd, "denoiser.")
    eng.finalize()
    return eng, nsd


def test_novae_denoiser_vs_reference_golden(novae):
    eng, _ = novae
    g = golden("denoiser_novae.npz")
    gen = torch.Generator().manual_seed(31)
    x = torch.randn(2, 24, 263, generator=gen).repeat(2, 1, 1)
    ctx = synth.text_context(2, 1, seed=32)
    y = eng.denoise(x, 999, ctx, [24, 16] * 2)
    assert y.shape == (4, 24, 263)
    assert _rel(y, g["y"]) < 2e-4
    assert float(y[1, 16:].abs().max()) == 0.0 and float(y[3, 16:].abs().max()) == 0.0


def test_novae_ddpm_loop_vs_oracle(novae):
    """Raw-motion diffusion with per-step injected noise (DDPM, fixed_small variance, CFG 7.5)."""
    eng, nsd = novae
    B, T, steps = 2, 24, 8
    lengths = [24, 16]
    ts = eng.set_timesteps(steps)
    ref = O.DDPMScheduler()
    ref.set_timesteps(steps)
    assert torch.equal(ts, ref.timesteps)
    gen = torch.Generator().manual_seed(41)
    x0 = torch.randn(B, T, 263, generator=gen)
    nz = torch.randn(steps, B, T, 263, generator=gen)
    ctx = synth.text_context(B, 1, seed=42)
    z = eng.diffusion_reverse(ctx, x0, lengths, step_noise=nz)
    cfg = O.DenoiserCfg(arch="trans_dec", latent_dim=512, diffusion_only=True)
    zo = O.diffusion_reverse(nsd, cfg, O.DDPMScheduler(), steps, ctx, x0, lengths, step_noise=nz)
    assert z.shape == (T, B, 263)
    assert _rel(z, zo) < 1e-3


# ------------------------------------------------------------------ action-to-motion (BASELINE configs[3] shape)
def test_action_to_motion_loop_vs_oracle(built_lib):
    """15-layer action-conditioned denoiser (EmbedAction, uncond half zeroed) + ActorVae decoder,
    50 guided DDIM steps, against the oracle."""
    from mld_b200.engine import Engine, make_config
    asd = synth.denoiser_state_dict(seed=2345, condition="action", num_layers=15, nclasses=12, nfeats=150)
    avsd = synth.actor_vae_state_dict(seed=777)
    eng = Engine(make_config(condition="action", num_layers=15, nclasses=12, nfeats=150, vae="actor",
                             vae_layers=6, vae_nfeats=150), 0)
    eng.load_state_dict(asd, "denoiser.")
    eng.load_state_dict(avsd, "vae.")
    eng.finalize()
    eng.set_timesteps(50)
    B, lengths = 5, [60, 60, 44, 60, 20]
    g = torch.Generator().manual_seed(91)
    actions = torch.randint(0, 12, (B, 1), generator=g)
    cond = torch.cat([torch.zeros_like(actions), actions])            # mld.py:716-717
    noise = synth.init_noise(B, seed=92)
    out = eng.sample(cond, noise, lengths, want=("latents", "feats"))
    acfg = O.DenoiserCfg(condition="action", num_layers=15, nclasses=12, nfeats=150)
    zo = O.diffusion_reverse(asd, acfg, O.DDIMScheduler(), 50, cond, noise, lengths)
    fo = O.vae_decode(avsd, O.VaeCfg(kind="actor", nfeats=150, num_layers=6), zo, lengths)
    assert out["feats"].shape == (B, 60, 150)
    assert _rel(out["latents"], zo) < 1e-3
    assert _rel(out["feats"], fo) < 1e-3
    assert float(out["feats"][4, 20:].abs().max()) == 0.0


# ------------------------------------------------------------------ latent_dim = [2, 256]
def test_two_latent_tokens_vs_reference_golden(built_lib):
    """n_lat = 2: denoiser forward (the trimmed last layer selects two rows per sequence), MldVae decode with
    TWO memory tokens (a real cross-attention softmax, not the one-token collapse) and encode (4 distribution
    tokens), against the reference's own modules."""
    from mld_b200.engine import Engine, make_config
    g = golden("nlat2.npz")
    dsd, vsd = synth.denoiser_state_dict(seed=5678), synth.mld_vae_state_dict(seed=8765, n_lat=2)
    eng = Engine(make_config(latent_dim=(2, 256)), 0)
    eng.load_state_dict(dsd, "denoiser.")
    eng.load_state_dict(vsd, "vae.")
    eng.finalize()
    ctx = synth.text_context(2, 77, seed=111)
    x = synth.init_noise(2, n_lat=2, seed=112).repeat(2, 1, 1)
    y = eng.denoise(x, 501, ctx, [196, 100] * 2)
    assert y.shape == (4, 2, 256)
    assert _rel(y, g["y"]) < 2e-4
    lengths = [196, 120, 8]
    z = synth.init_noise(3, n_lat=2, seed=141).permute(1, 0, 2).contiguous()
    eng.kernel_stats(reset=True)
    feats = eng.vae_decode(z, lengths)
    st = eng.kernel_stats()
    assert _rel(feats, g["feats"]) < 2e-4
    assert float(feats[2, 8:].abs().max()) == 0.0
    assert st["attn_simt"] == 0 and st["attn_tc"] == 2 * 9, st      # self- and cross-attention of 9 layers
    gen = torch.Generator().manual_seed(142)
    motion = torch.randn(3, 196, 263, generator=gen)
    mu, logvar = eng.vae_encode(motion, lengths)
    assert mu.shape == (2, 3, 256)
    assert _rel(mu, g["mu"]) < 2e-4
    assert _rel(logvar.exp().pow(0.5), g["std"]) < 2e-4


# ------------------------------------------------------------------ no-VAE model at its BASELINE shape
def test_novae_full_shape_vs_reference_golden_and_oracle(novae):
    """configs[4] shape: 196 frames x 263 features, d = 512 (head_dim 128), ragged lengths.  Single forward
    against the reference module's output, then 4 guided DDPM steps with injected noise against the oracle;
    the kernel statistics must show every attention (196 x 196 self-attention, 2-token cross-attention) on
    the wgmma kernel and every stack GEMM on the tensor cores."""
    eng, nsd = novae
    g = golden("denoiser_novae_T196.npz")
    lengths = [196, 132]
    gen = torch.Generator().manual_seed(231)
    x = torch.randn(2, 196, 263, generator=gen).repeat(2, 1, 1)
    ctx = synth.text_context(2, 1, seed=232)
    eng.kernel_stats(reset=True)
    y = eng.denoise(x, 777, ctx, lengths * 2)
    st = eng.kernel_stats()
    assert _rel(y, g["y"]) < 2e-4
    assert float(y[1, 132:].abs().max()) == 0.0
    assert st["attn_tc"] == 2 * 9 and st["attn_simt"] == 0 and st["attn_mma"] == 0, st
    assert st["gemm_tc"] >= 9 * 5, st                 # qkv, cross q / kv, FFN1 ... of 9 layers + both pose projections
    steps = 4
    eng.set_timesteps(steps)
    gen = torch.Generator().manual_seed(241)
    x0 = torch.randn(2, 196, 263, generator=gen)
    nz = torch.randn(steps, 2, 196, 263, generator=gen)
    z = eng.diffusion_reverse(ctx, x0, lengths, step_noise=nz)
    cfg = O.DenoiserCfg(arch="trans_dec", latent_dim=512, diffusion_only=True)
    zo = O.diffusion_reverse(nsd, cfg, O.DDPMScheduler(), steps, ctx, x0, lengths, step_noise=nz)
    assert z.shape == (196, 2, 263)
    assert _rel(z, zo) < 1e-3
    # replaying the captured step graph a second time gives the same motion (device-side step counter reset)
    assert torch.equal(eng.diffusion_reverse(ctx, x0, lengths, step_noise=nz), z)


# ------------------------------------------------------------------ DDPM on the latent model
def test_latent_ddpm_needs_and_uses_injected_noise(engines):
    """scheduler='ddpm' with the VAE model: diffusers' DDPMScheduler.step adds variance noise at t > 0; the
    caller injects it ([n_steps, B, n_lat, d]).  Without it the call fails instead of silently running the
    deterministic posterior mean."""
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(scheduler="ddpm", vae="none"), 0)
    eng.load_state_dict(engines["dsd"], "denoiser.")
    eng.finalize()
    steps, B = 6, 3
    eng.set_timesteps(steps)
    ctx, noise = synth.text_context(B, 5, seed=301), synth.init_noise(B, seed=302)
    with pytest.raises(RuntimeError, match="step_noise"):
        eng.diffusion_reverse(ctx, noise, [196] * B)
    gen = torch.Generator().manual_seed(303)
    nz = torch.randn(steps, B, 1, 256, generator=gen)
    z = eng.diffusion_reverse(ctx, noise, [196] * B, step_noise=nz)
    zo = O.diffusion_reverse(engines["dsd"], O.DenoiserCfg(), O.DDPMScheduler(), steps, ctx, noise, [196] * B,
                             step_noise=nz)
    assert _rel(z, zo) < 1e-3


def test_wrapper_rejects_bad_shapes(engines):
    """The C ABI borrows raw pointers; the torch-side wrapper refuses shapes that would read out of bounds."""
    eng = engines["text"]
    ctx, noise = synth.text_context(2, 77, seed=1), synth.init_noise(2, seed=2)
    with pytest.raises(ValueError):
        eng.sample(ctx[2:], noise, [196, 196])               # cond without the uncond half
    with pytest.raises(ValueError):
        eng.sample(ctx, noise[:, :, :128], [196, 196])       # wrong latent width
    with pytest.raises(ValueError):
        eng.sample(ctx, noise, [196])                        # len(lengths) != B
    with pytest.raises(ValueError):
        eng.diffusion_reverse(ctx[:, :, :512], noise, [196, 196])
