"""GPU (pytest -m gpu): stochastic sampling - DDIM with eta > 0, clip_sample and the three beta schedules -
on the library's kernels, against the scheduler restatement of tests/stochastic_ref.py driving the oracle.

Bars: one scheduler step is bit-exact with the fp32 restatement (same operation order); the 50-step loops meet
the parity tests' tolerances (1e-3 relative on latents and on the joints of each motion); everything that only
moves the same draws between entry points (host / device buffers, seeded / explicit noise) is bit-identical."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

import stochastic_ref as R
from mld_b200 import synth
from oracle import mld_oracle as O

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

FALLBACKS = ("attn_simt", "gemm_simt", "ln_unfused", "attn_mma")


def _rel(a, b):
    a, b = torch.as_tensor(a).float().cpu(), torch.as_tensor(b).float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _joint_err(joints, ref_list, lengths):
    return max(float((joints[b, :n].cpu() - ref_list[b]).abs().max() / ref_list[b].abs().max())
               for b, n in enumerate(lengths))


def _engine(dsd=None, vsd=None, steps=50, mean_std=None, **kw):
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(**kw), 0)
    if dsd is not None:
        eng.load_state_dict(dsd, "denoiser.")
    if vsd is not None:
        eng.load_state_dict(vsd, "vae.")
    eng.finalize()
    if mean_std is not None:
        eng.set_mean_std(*mean_std)
    eng.set_timesteps(steps)
    return eng


@pytest.fixture(scope="module")
def models(built_lib):
    dsd, vsd = synth.denoiser_state_dict(1234), synth.mld_vae_state_dict(4321)
    ms = synth.mean_std()
    e0 = _engine(dsd, vsd, mean_std=ms)
    e1 = _engine(dsd, vsd, mean_std=ms, eta=1.0)
    return dict(e0=e0, e1=e1, dsd=dsd, vsd=vsd, mean=ms[0], std=ms[1])


def _step_noise(steps, B, seed, tail=(1, 256)):
    return torch.randn(steps, B, *tail, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------ one scheduler step
@pytest.mark.parametrize("schedule", ["scaled_linear", "linear", "squaredcos_cap_v2"])
def test_scheduler_step_bit_exact(built_lib, schedule):
    g = torch.Generator().manual_seed(7)
    x, e, nz = torch.randn(6, 1, 256, generator=g) * 3, torch.randn(6, 1, 256, generator=g) * 3, torch.randn(6, 1, 256, generator=g)
    cases = [("ddim", eta, clip) for eta in (0.3, 1.0) for clip in (False, True)] + [("ddpm", 0.0, True)]
    for kind, eta, clip in cases:
        eng = _engine(num_layers=0, vae="none", scheduler=kind, eta=eta, beta_schedule=schedule, clip_sample=clip)
        if kind == "ddim":
            ref = R.DDIMScheduler(beta_schedule=schedule, clip_sample=clip)
            unclipped = R.DDIMScheduler(beta_schedule=schedule)
        else:
            ref = R.DDPMScheduler(beta_schedule=schedule, clip_sample=clip)
            unclipped = R.DDPMScheduler(beta_schedule=schedule)
        ref.set_timesteps(50)
        unclipped.set_timesteps(50)
        ts = eng.timesteps
        assert torch.equal(ts, ref.timesteps)
        for t in (int(ts[0]), int(ts[25]), int(ts[-1])):
            got = eng.scheduler_step(e, t, x, nz).cpu()
            if kind == "ddim":
                want, free = ref.step(e, t, x, eta=eta, noise=nz), unclipped.step(e, t, x, eta=eta, noise=nz)
            else:
                want, free = ref.step(e, t, x, noise=nz), unclipped.step(e, t, x, noise=nz)
            assert torch.equal(got, want), (kind, eta, clip, t)
            if clip:
                assert not torch.equal(want, free), "inputs too small: clipping did not trigger"
        with pytest.raises(RuntimeError, match="noise"):            # the first step adds noise in every case
            eng.scheduler_step(e, int(ts[0]), x)


# ------------------------------------------------------------------ the reverse loop
@pytest.mark.parametrize("S", [1, 77])
def test_diffusion_reverse_eta1_vs_oracle(models, S):
    B, lengths = 4, [196, 120, 64, 196]
    ctx, noise = synth.text_context(B, S, seed=501), synth.init_noise(B, seed=502)
    nz = _step_noise(50, B, 503)
    z = models["e1"].diffusion_reverse(ctx, noise, lengths, step_noise=nz)
    zo = O.diffusion_reverse(models["dsd"], O.DenoiserCfg(), R.DDIMScheduler(step_noise=nz), 50, ctx, noise,
                             lengths, eta=1.0)
    assert _rel(z, zo) < 1e-3
    # the noise matters: the deterministic loop lands elsewhere
    assert _rel(models["e0"].diffusion_reverse(ctx, noise, lengths), zo) > 1e-2


def test_sample_eta1_matches_pieces_oracle_host_and_kernels(models):
    e0, e1 = models["e0"], models["e1"]
    B, S, T = 5, 77, 196                      # a shape no earlier test captured: the stats see every kernel
    lengths = [196, 64, 196, 100, 150]
    ctx, noise = synth.text_context(B, S, seed=511), synth.init_noise(B, seed=512)
    nz = _step_noise(50, B, 513)
    e0.kernel_stats(reset=True)
    e0.sample(ctx, noise, lengths, want=("joints",))
    st0 = e0.kernel_stats()
    e1.kernel_stats(reset=True)
    out = {k: v.clone() for k, v in e1.sample(ctx, noise, lengths, want=("latents", "feats", "joints"),
                                               step_noise=nz).items()}
    st1 = e1.kernel_stats()
    assert st1 == st0, (st0, st1)                                  # same kernels as the eta = 0 path
    assert all(st1[k] == 0 for k in FALLBACKS), st1
    # == diffusion_reverse -> vae_decode -> feats2joints, bit for bit
    z = e1.diffusion_reverse(ctx, noise, lengths, step_noise=nz)
    feats = e1.vae_decode(z, lengths)
    assert torch.equal(out["latents"], z) and torch.equal(out["feats"], feats)
    assert torch.equal(out["joints"], e1.feats2joints(feats))
    # repeated calls replay the same graph on the same draws
    again = e1.sample(ctx, noise, lengths, want=("joints",), step_noise=nz)["joints"]
    assert torch.equal(again, out["joints"])
    # host entry point
    joints = torch.empty((B, T, 22, 3), dtype=torch.float32).pin_memory()
    e1.sample_host(ctx.pin_memory(), noise.pin_memory(), torch.tensor(lengths, dtype=torch.int32).pin_memory(),
                   joints, T, step_noise=nz.pin_memory())
    torch.cuda.synchronize()
    assert torch.equal(joints, out["joints"].cpu())
    # the oracle on the same draws
    jo, _, _ = O.mld_forward(models["dsd"], O.DenoiserCfg(), models["vsd"], O.VaeCfg(), R.DDIMScheduler(step_noise=nz),
                             50, ctx, noise, lengths, models["mean"], models["std"], eta=1.0)
    err = _joint_err(out["joints"], jo, lengths)
    assert err < 1e-3, f"joint positions differ by {err:.3e} relative (gate 1e-3)"


def test_stochastic_needs_step_noise_and_deterministic_ignores_it(models):
    e0, e1 = models["e0"], models["e1"]
    B, lengths = 2, [196, 88]
    ctx, noise = synth.text_context(B, 77, seed=521), synth.init_noise(B, seed=522)
    nz = _step_noise(50, B, 523)
    with pytest.raises(RuntimeError, match="step_noise"):
        e1.sample(ctx, noise, lengths)
    with pytest.raises(RuntimeError, match="step_noise"):
        e1.diffusion_reverse(ctx, noise, lengths)
    with pytest.raises(ValueError, match="step_noise"):
        e1.sample(ctx, noise, lengths, step_noise=nz[:10])
    a = e0.sample(ctx, noise, lengths, want=("latents", "joints"))
    a = {k: v.clone() for k, v in a.items()}
    b = e0.sample(ctx, noise, lengths, want=("latents", "joints"), step_noise=nz)
    assert torch.equal(a["latents"], b["latents"]) and torch.equal(a["joints"], b["joints"])
    assert torch.equal(e0.diffusion_reverse(ctx, noise, lengths),
                       e0.diffusion_reverse(ctx, noise, lengths, step_noise=nz))


def test_clip_and_schedule_on_the_fused_path(models):
    """DDPM with clip_sample (the commented block of the shipped scheduler.yaml) and a DDIM eta = 0.5 run on
    the cosine schedule with clipping, 10 steps, through mldb_sample against the oracle."""
    B, lengths = 3, [196, 100, 40]
    ctx, noise = synth.text_context(B, 5, seed=531), synth.init_noise(B, seed=532)
    steps = 10
    for kw, ref, eta in (
            (dict(scheduler="ddpm", clip_sample=True), R.DDPMScheduler(clip_sample=True), 0.0),
            (dict(eta=0.5, beta_schedule="squaredcos_cap_v2", clip_sample=True), None, 0.5)):
        nz = _step_noise(steps, B, 533)
        if ref is None:
            ref = R.DDIMScheduler(beta_schedule="squaredcos_cap_v2", clip_sample=True, step_noise=nz)
        eng = _engine(models["dsd"], models["vsd"], steps=steps, mean_std=(models["mean"], models["std"]), **kw)
        out = eng.sample(ctx, noise, lengths, want=("latents", "joints"), step_noise=nz)
        zo = O.diffusion_reverse(models["dsd"], O.DenoiserCfg(), ref, steps, ctx, noise, lengths, eta=eta,
                                 step_noise=nz)
        assert _rel(out["latents"], zo) < 1e-3, kw
        jo = O.feats2joints(O.vae_decode(models["vsd"], O.VaeCfg(), zo, lengths), models["mean"], models["std"])
        assert _joint_err(out["joints"], [jo[b, :n] for b, n in enumerate(lengths)], lengths) < 1e-3, kw


# ------------------------------------------------------------------ no-VAE model, DDIM eta > 0
def test_novae_ddim_eta_vs_oracle(built_lib):
    """modules_novae/scheduler.yaml's DDIM block (steps_offset 1, set_alpha_to_one false) with eta = 0.8."""
    nsd = synth.denoiser_state_dict(seed=3456, arch="trans_dec", d=512, diffusion_only=True)
    steps, B, T = 4, 2, 24
    eng = _engine(nsd, steps=steps, arch="trans_dec", latent_dim=(1, 512), diffusion_only=True, vae="none",
                  scheduler="ddim", eta=0.8)
    lengths = [24, 16]
    gen = torch.Generator().manual_seed(541)
    x0 = torch.randn(B, T, 263, generator=gen)
    nz = torch.randn(steps, B, T, 263, generator=gen)
    ctx = synth.text_context(B, 1, seed=542)
    with pytest.raises(RuntimeError, match="step_noise"):
        eng.diffusion_reverse(ctx, x0, lengths)
    z = eng.diffusion_reverse(ctx, x0, lengths, step_noise=nz)
    cfg = O.DenoiserCfg(arch="trans_dec", latent_dim=512, diffusion_only=True)
    zo = O.diffusion_reverse(nsd, cfg, R.DDIMScheduler(step_noise=nz), steps, ctx, x0, lengths, eta=0.8)
    assert z.shape == (T, B, 263)
    assert _rel(z, zo) < 1e-3
    assert torch.equal(eng.diffusion_reverse(ctx, x0, lengths, step_noise=nz), z)


# ------------------------------------------------------------------ seeded draws in the reference's order
def _documented_draws(seed, B, steps, device):
    torch.manual_seed(seed)
    z0 = torch.randn((B, 1, 256), device=device, dtype=torch.float)
    return z0, torch.stack([torch.randn((B, 1, 256), device=device, dtype=torch.float) for _ in range(steps)])


def test_pipeline_seeded_draws_equal_explicit_noise(models):
    from types import SimpleNamespace
    from mld_b200.modules import B200MldDenoiser
    from mld_b200.pipeline import B200MLD
    model = B200MLD(models["dsd"], models["vsd"], mean=models["mean"], std=models["std"], eta=1.0)
    B, lengths, seed = 2, [196, 88], 1234
    ctx = synth.text_context(B, 77, seed=551)
    torch.manual_seed(seed)
    seeded = model({"length": lengths, "text_emb": ctx})
    z0, sn = _documented_draws(seed, B, 50, model.device)
    explicit = model({"length": lengths, "text_emb": ctx, "init_noise": z0, "step_noise": sn})
    assert all(torch.equal(a, b) for a, b in zip(seeded, explicit))
    # the reference's own loop (mld.py:303-346) through the drop-in denoiser and scheduler
    abl = SimpleNamespace(SKIP_CONNECT=True, VAE_TYPE="mld", DIFF_PE_TYPE="mld", PE_TYPE="mld", MLP_DIST=False)
    den = B200MldDenoiser(ablation=abl, nfeats=263, condition="text", latent_dim=[1, 256], ff_size=1024,
                          num_layers=9, num_heads=4, arch="trans_enc", text_encoded_dim=768)
    den.load_state_dict(models["dsd"], strict=True)
    den = den.cuda()
    sched, ctxg = model.scheduler, ctx.cuda()

    def loop(explicit_noise):
        lat = (z0.clone() if explicit_noise else torch.randn((B, 1, 256), device="cuda", dtype=torch.float))
        lat = lat * sched.init_noise_sigma
        for i, t in enumerate(sched.timesteps):
            eps = den(sample=torch.cat([lat] * 2), timestep=t, encoder_hidden_states=ctxg, lengths=lengths * 2)[0]
            u, c = eps.chunk(2)
            kw = dict(variance_noise=sn[i]) if explicit_noise else {}
            lat = sched.step(u + 7.5 * (c - u), t, lat, eta=1.0, **kw).prev_sample
        return lat

    torch.manual_seed(seed)
    a = loop(False)
    b = loop(True)
    assert torch.equal(a, b)
    # and it samples what the fused path samples on those draws
    z = model.engine.diffusion_reverse(ctx, z0, lengths, step_noise=sn)
    assert _rel(a.permute(1, 0, 2), z) < 1e-3
    zeros = torch.zeros(B, 1, 256, device="cuda")
    with pytest.raises(ValueError, match="eta"):                  # the coefficients follow the configured eta
        sched.step(zeros, sched.timesteps[0], zeros, eta=0.0)


def test_pipeline_ddpm_leaves_the_last_slice_undrawn(models):
    from mld_b200.pipeline import B200MLD
    model = B200MLD(models["dsd"], models["vsd"], mean=models["mean"], std=models["std"], scheduler="ddpm",
                    num_inference_timesteps=10)
    torch.manual_seed(7)
    sn = model._draw_step_noise(3)
    assert sn.shape == (10, 3, 1, 256) and int(model.scheduler.timesteps[-1]) == 0
    assert float(sn[-1].abs().max()) == 0.0 and float(sn[:-1].abs().min()) > 0.0
    torch.manual_seed(7)
    want = torch.stack([torch.randn((3, 1, 256), device=model.device) for _ in range(9)])
    assert torch.equal(sn[:-1], want)


# ------------------------------------------------------------------ two GPUs
B2, S2, STEPS2 = 4, 77, 4
LENGTHS2 = [196, 64, 120, 33]


def _eta_engine(device):
    from mld_b200.engine import Engine, make_config
    eng = Engine(make_config(eta=1.0), device)
    eng.load_state_dict(synth.denoiser_state_dict(1234), "denoiser.")
    eng.load_state_dict(synth.mld_vae_state_dict(4321), "vae.")
    eng.finalize()
    eng.set_mean_std(*synth.mean_std())
    eng.set_timesteps(STEPS2)
    return eng


def _worker(rank, world, port, out_path):
    import torch.distributed as dist
    from mld_b200.distributed import sample_sharded_engine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    eng = _eta_engine(rank)
    eng.comm_init()
    ctx, noise = synth.text_context(B2, S2, seed=561), synth.init_noise(B2, seed=562)
    j = sample_sharded_engine(eng, ctx, noise, LENGTHS2, step_noise=_step_noise(STEPS2, B2, 563))
    torch.cuda.synchronize()
    torch.save(j.cpu(), f"{out_path}.{rank}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_sharded_eta1_equals_single_gpu(tmp_path, built_lib):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    out_path = str(tmp_path / "gathered.pt")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out_path)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
        assert p.exitcode == 0
    eng = _eta_engine(0)
    c, z = synth.text_context(B2, S2, seed=561), synth.init_noise(B2, seed=562)
    want = eng.sample(c, z, LENGTHS2, want=("joints",), step_noise=_step_noise(STEPS2, B2, 563))["joints"].cpu()
    for r in range(2):
        assert torch.equal(torch.load(f"{out_path}.{r}"), want), f"rank {r}"
