"""Generate tests/golden/*.npz by running the REFERENCE's own modules (TEST INFRASTRUCTURE).

Run in the build container only (``/root/reference`` does not exist ):

    python -m oracle.make_golden

For each case the seeded synthetic state dict from ``mld_b200.synth`` is loaded into the
reference ``nn.Module`` with ``strict=True`` (pinning the state-dict key contract), the
module is run on seeded inputs in fp32/eval/no_grad, and the outputs are stored.  Inputs and
weights are NOT stored - tests rebuild them from the same seeds.  ``MLD`` itself cannot be
imported (needs pytorch_lightning/torchmetrics), nor diffusers, so the sampling loop case
drives the reference denoiser/VAE modules with the loop body of ``mld.py:323-346`` restated
here and the oracle's DDIM restatement.
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

REF = os.environ.get("MLD_REFERENCE", "/root/reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden")


def _ref_modules():
    sys.path.insert(0, REF)
    from mld.models.architectures.mld_denoiser import MldDenoiser
    from mld.models.architectures.mld_vae import MldVae
    from mld.models.architectures.actor_vae import ActorVae
    from mld.data.humanml.scripts.motion_process import recover_from_ric
    return MldDenoiser, MldVae, ActorVae, recover_from_ric


def abl(vae_type="mld"):
    return SimpleNamespace(SKIP_CONNECT=True, VAE_TYPE=vae_type, DIFF_PE_TYPE="mld",
                           PE_TYPE="mld", MLP_DIST=False)


def build_text_denoiser(MldDenoiser, sd):
    m = MldDenoiser(ablation=abl(), nfeats=263, condition="text", latent_dim=[1, 256],
                    ff_size=1024, num_layers=9, num_heads=4, dropout=0.1,
                    normalize_before=False, activation="gelu", flip_sin_to_cos=True,
                    return_intermediate_dec=False, position_embedding="learned",
                    arch="trans_enc", freq_shift=0, guidance_scale=7.5, guidance_uncondp=0.1,
                    text_encoded_dim=768, nclasses=10)
    m.load_state_dict(sd, strict=True)
    return m.eval()


def golden_nlat2():
    """latent_dim = [2, 256] (two latent tokens): denoiser forward, MldVae decode (2 memory tokens: the
    cross-attention is a real softmax, not the 1-token collapse) and encode (4 distribution tokens)."""
    from mld_b200 import synth
    from oracle import mld_oracle as O
    MldDenoiser, MldVae, _, _ = _ref_modules()
    torch.set_grad_enabled(False)
    dsd = synth.denoiser_state_dict(seed=5678)
    den = MldDenoiser(ablation=abl(), nfeats=263, condition="text", latent_dim=[2, 256], ff_size=1024,
                      num_layers=9, num_heads=4, arch="trans_enc", text_encoded_dim=768)
    den.load_state_dict(dsd, strict=True)
    den.eval()
    ctx = synth.text_context(2, 77, seed=111)
    x = synth.init_noise(2, n_lat=2, seed=112).repeat(2, 1, 1)
    y = den(sample=x, timestep=torch.tensor(501), encoder_hidden_states=ctx, lengths=[196, 100] * 2)[0]
    yo = O.denoiser_forward(dsd, O.DenoiserCfg(n_lat=2), x, torch.tensor(501), ctx, [196, 100] * 2)
    print(f"n_lat=2 denoiser: oracle-vs-ref max abs {float((y - yo).abs().max()):.3e}")
    vsd = synth.mld_vae_state_dict(seed=8765, n_lat=2)
    vae = MldVae(ablation=abl(), nfeats=263, latent_dim=[2, 256], ff_size=1024, num_layers=9, num_heads=4,
                 dropout=0.1, arch="encoder_decoder", normalize_before=False, activation="gelu",
                 position_embedding="learned")
    vae.load_state_dict(vsd, strict=True)
    vae.eval()
    lengths = [196, 120, 8]
    z = synth.init_noise(3, n_lat=2, seed=141).permute(1, 0, 2).contiguous()      # [2, B, 256]
    feats = vae.decode(z, lengths)
    fo = O.vae_decode(vsd, O.VaeCfg(n_lat=2), z, lengths)
    print(f"n_lat=2 vae decode: oracle-vs-ref max abs {float((feats - fo).abs().max()):.3e}")
    g = torch.Generator().manual_seed(142)
    motion = torch.randn(3, 196, 263, generator=g)
    _, dist = vae.encode(motion, lengths)
    mo, lvo = O.vae_encode(vsd, O.VaeCfg(n_lat=2), motion, lengths)
    print(f"n_lat=2 vae encode: oracle-vs-ref mu {float((dist.loc - mo).abs().max()):.3e}")
    np.savez(os.path.join(OUT, "nlat2.npz"), y=y.numpy(), feats=feats.numpy(), mu=dist.loc.numpy(),
             std=dist.scale.numpy())


def golden_novae196():
    """The no-VAE denoiser at its BASELINE shape: 196 frames x 263 features, d = 512 (head 128), ragged lengths."""
    from mld_b200 import synth
    from oracle import mld_oracle as O
    MldDenoiser, _, _, _ = _ref_modules()
    torch.set_grad_enabled(False)
    nsd = synth.denoiser_state_dict(seed=3456, arch="trans_dec", d=512, diffusion_only=True)
    nden = MldDenoiser(ablation=abl("no"), nfeats=263, condition="text", latent_dim=[1, 512], ff_size=1024,
                       num_layers=9, num_heads=4, arch="trans_dec", text_encoded_dim=768)
    nden.load_state_dict(nsd, strict=True)
    nden.eval()
    lengths = [196, 132]
    g = torch.Generator().manual_seed(231)
    x = torch.randn(2, 196, 263, generator=g).repeat(2, 1, 1)
    ctx = synth.text_context(2, 1, seed=232)
    y = nden(sample=x, timestep=torch.tensor(777), encoder_hidden_states=ctx, lengths=lengths * 2)[0]
    ncfg = O.DenoiserCfg(arch="trans_dec", latent_dim=512, diffusion_only=True)
    yo = O.denoiser_forward(nsd, ncfg, x, torch.tensor(777), ctx, lengths * 2)
    print(f"denoiser no-VAE T=196: oracle-vs-ref max abs {float((y - yo).abs().max()):.3e}")
    np.savez(os.path.join(OUT, "denoiser_novae_T196.npz"), y=y.numpy())


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "nlat2":
        return golden_nlat2()
    if len(sys.argv) > 1 and sys.argv[1] == "novae196":
        return golden_novae196()
    from mld_b200 import synth
    from oracle import mld_oracle as O
    MldDenoiser, MldVae, ActorVae, recover_from_ric = _ref_modules()
    os.makedirs(OUT, exist_ok=True)
    torch.set_grad_enabled(False)
    torch.set_num_threads(8)

    # ---- 1. text denoiser single forward, S in {77, 1}
    dsd = synth.denoiser_state_dict(seed=1234)
    den = build_text_denoiser(MldDenoiser, dsd)
    out = {}
    for S in (77, 1):
        ctx = synth.text_context(2, S, seed=11)
        x = synth.init_noise(2, seed=12).repeat(2, 1, 1)
        for t in (981, 1):
            y = den(sample=x, timestep=torch.tensor(t), encoder_hidden_states=ctx,
                    lengths=[196, 100] * 2)[0]
            out[f"S{S}_t{t}"] = y.numpy()
            yo = O.denoiser_forward(dsd, O.DenoiserCfg(), x, torch.tensor(t), ctx, [196, 100] * 2)
            print(f"denoiser text S={S} t={t}: oracle-vs-ref max abs {float((y - yo).abs().max()):.3e}")
    np.savez(os.path.join(OUT, "denoiser_text.npz"), **out)

    # ---- 2. action denoiser (15 layers, 12 classes)
    asd = synth.denoiser_state_dict(seed=2345, condition="action", num_layers=15, nclasses=12,
                                    nfeats=150)
    aden = MldDenoiser(ablation=abl(), nfeats=150, condition="action", latent_dim=[1, 256],
                       ff_size=1024, num_layers=15, num_heads=4, arch="trans_enc",
                       guidance_scale=7.5, text_encoded_dim=768, nclasses=12)
    aden.load_state_dict(asd, strict=True)
    aden.eval()
    g = torch.Generator().manual_seed(21)
    actions = torch.randint(0, 12, (3, 1), generator=g)
    cond = torch.cat([torch.zeros_like(actions), actions])            # mld.py:716-717
    x = synth.init_noise(3, seed=22).repeat(2, 1, 1)
    y = aden(sample=x, timestep=torch.tensor(501), encoder_hidden_states=cond, lengths=[60] * 6)[0]
    acfg = O.DenoiserCfg(condition="action", num_layers=15, nclasses=12, nfeats=150)
    yo = O.denoiser_forward(asd, acfg, x, torch.tensor(501), cond, [60] * 6)
    print(f"denoiser action: oracle-vs-ref max abs {float((y - yo).abs().max()):.3e}")
    np.savez(os.path.join(OUT, "denoiser_action.npz"), y=y.numpy(), actions=actions.numpy())

    # ---- 3. no-VAE trans_dec denoiser (d=512)
    nsd = synth.denoiser_state_dict(seed=3456, arch="trans_dec", d=512, diffusion_only=True)
    nden = MldDenoiser(ablation=abl("no"), nfeats=263, condition="text", latent_dim=[1, 512],
                       ff_size=1024, num_layers=9, num_heads=4, arch="trans_dec",
                       text_encoded_dim=768)
    nden.load_state_dict(nsd, strict=True)
    nden.eval()
    lengths = [24, 16]
    g = torch.Generator().manual_seed(31)
    x = torch.randn(2, 24, 263, generator=g).repeat(2, 1, 1)
    ctx = synth.text_context(2, 1, seed=32)
    y = nden(sample=x, timestep=torch.tensor(999), encoder_hidden_states=ctx, lengths=lengths * 2)[0]
    ncfg = O.DenoiserCfg(arch="trans_dec", latent_dim=512, diffusion_only=True)
    yo = O.denoiser_forward(nsd, ncfg, x, torch.tensor(999), ctx, lengths * 2)
    print(f"denoiser no-VAE: oracle-vs-ref max abs {float((y - yo).abs().max()):.3e}")
    np.savez(os.path.join(OUT, "denoiser_novae.npz"), y=y.numpy())

    # ---- 4. MldVae decode / encode
    vsd = synth.mld_vae_state_dict(seed=4321)
    vae = MldVae(ablation=abl(), nfeats=263, latent_dim=[1, 256], ff_size=1024, num_layers=9,
                 num_heads=4, dropout=0.1, arch="encoder_decoder", normalize_before=False,
                 activation="gelu", position_embedding="learned")
    vae.load_state_dict(vsd, strict=True)
    vae.eval()
    lengths = [196, 120, 8]
    z = synth.init_noise(3, seed=41).permute(1, 0, 2).contiguous()     # [1,B,256]
    feats = vae.decode(z, lengths)
    fo = O.vae_decode(vsd, O.VaeCfg(), z, lengths)
    print(f"vae decode: oracle-vs-ref max abs {float((feats - fo).abs().max()):.3e}")
    g = torch.Generator().manual_seed(42)
    motion = torch.randn(3, 196, 263, generator=g)
    _, dist = vae.encode(motion, lengths)
    mu, std = dist.loc, dist.scale
    mo, lvo = O.vae_encode(vsd, O.VaeCfg(), motion, lengths)
    print(f"vae encode: oracle-vs-ref mu {float((mu - mo).abs().max()):.3e} "
          f"std {float((std - lvo.exp().pow(0.5)).abs().max()):.3e}")
    np.savez(os.path.join(OUT, "vae_mld.npz"), feats=feats.numpy(), mu=mu.numpy(), std=std.numpy())

    # ---- 5. ActorVae decode
    avsd = synth.actor_vae_state_dict(seed=777)
    avae = ActorVae(ablation=abl(), nfeats=150, latent_dim=[1, 256], ff_size=1024, num_layers=6,
                    num_heads=4, dropout=0.1, activation="gelu")
    avae.load_state_dict(avsd, strict=True)
    avae.eval()
    lengths = [60, 40, 12]
    z = synth.init_noise(3, seed=51).permute(1, 0, 2).contiguous()
    feats = avae.decode(z, lengths)
    vcfg = O.VaeCfg(kind="actor", nfeats=150, num_layers=6)
    fo = O.vae_decode(avsd, vcfg, z, lengths)
    print(f"actor decode: oracle-vs-ref max abs {float((feats - fo).abs().max()):.3e}")
    np.savez(os.path.join(OUT, "vae_actor.npz"), feats=feats.numpy())

    # ---- 6. feats2joints (recover_from_ric) on de-normalised random feats
    g = torch.Generator().manual_seed(61)
    f = torch.randn(2, 196, 263, generator=g) * 0.3
    mean, std = synth.mean_std()
    joints = recover_from_ric(f * std + mean, 22)                      # HumanML3D.py:41-45
    jo = O.feats2joints(f, mean, std)
    print(f"feats2joints: oracle-vs-ref max abs {float((joints - jo).abs().max()):.3e}")
    np.savez(os.path.join(OUT, "feats2joints.npz"), joints=joints.numpy())

    # ---- 7. full sampling loop, B=2, S=77 and S=1: reference modules + restated loop
    vsd = synth.mld_vae_state_dict(seed=4321)
    for S in (77, 1):
        B, lengths = 2, [196, 88]
        ctx = synth.text_context(B, S, seed=71)
        noise = synth.init_noise(B, seed=72)
        sched = O.DDIMScheduler()
        sched.set_timesteps(50)
        latents = noise * sched.init_noise_sigma
        lat_trace = []
        for t in sched.timesteps:                                      # mld.py:323-346
            x_in = torch.cat([latents] * 2)
            eps = den(sample=x_in, timestep=t, encoder_hidden_states=ctx, lengths=lengths * 2)[0]
            u, c = eps.chunk(2)
            eps = u + 7.5 * (c - u)
            latents = sched.step(eps, t, latents, eta=0.0)
            lat_trace.append(latents.numpy().copy())
        z = latents.permute(1, 0, 2)
        feats = vae.decode(z, lengths)
        joints = recover_from_ric(feats * std + mean, 22)
        zo = O.diffusion_reverse(dsd, O.DenoiserCfg(), O.DDIMScheduler(), 50, ctx, noise, lengths)
        print(f"loop S={S}: oracle-vs-ref latents max abs {float((z - zo).abs().max()):.3e} "
              f"(|z|max {float(z.abs().max()):.3f})")
        np.savez(os.path.join(OUT, f"loop_S{S}.npz"), latents=np.stack(lat_trace),
                 feats=feats.numpy(), joints=joints.numpy())
    golden_nlat2()
    golden_novae196()
    print("golden written to", OUT)


if __name__ == "__main__":
    main()
