"""``B200MLD``: the inference surface of ``mld.models.modeltype.mld.MLD`` (no Lightning).

Methods mirror the reference one to one:
  forward(batch)                      mld.py:216-265
  _diffusion_reverse(emb, lengths)    mld.py:290-360   (one CUDA graph per batch shape)
  gen_from_latent(batch)              mld.py:267-275
  recon_from_motion(batch)            mld.py:277-288
and a scheduler object with the diffusers surface the reference touches
(``init_noise_sigma``, ``set_timesteps``, ``timesteps``, ``step(...).prev_sample``,
``config.num_train_timesteps``; mld.py:310-320,345).

The text encoder is a separate callable ``text_encoder(List[str]) -> Tensor[2B, S, 768]``: the native
``mld_b200.text.B200TextEncoder`` (CLIP on this library's kernels) or the reference's ``MldTextEncoder``.
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace
from typing import Callable, Dict, List, Optional, Sequence

import torch

from . import _lib
from .engine import Engine, make_config


def remove_padding(tensors, lengths):
    """mld/utils/temos_utils.py:24-28."""
    return [t[:n] for t, n in zip(tensors, lengths)]


class B200Scheduler:
    """diffusers ``DDIMScheduler`` / ``DDPMScheduler`` surface backed by the engine's kernels."""

    def __init__(self, engine: Engine):
        self._e = engine
        self.init_noise_sigma = 1.0
        self.config = SimpleNamespace(num_train_timesteps=engine.cfg.num_train_timesteps)
        self.timesteps: Optional[torch.Tensor] = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.timesteps = self._e.set_timesteps(num_inference_steps)
        return self

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output, timestep, sample, eta: float = 0.0, noise=None, generator=None,
             variance_noise=None, **kw):
        """``DDIMScheduler.step`` / ``DDPMScheduler.step``.  The step adds noise when the scheduler is DDIM with
        ``eta > 0`` or DDPM at ``t > 0``.  That N(0,1) tensor is ``variance_noise`` (``noise`` is the same
        argument under its earlier name); when it is not given it is drawn here as current diffusers' ``randn_tensor``
        does: ``torch.randn(model_output.shape, generator=generator, device=model_output.device,
        dtype=model_output.dtype)``.  Older diffusers releases drew it on the CPU and moved it to the device, so
        their seeded runs give other numbers.  The DDIM coefficients are built in the library from the
        configured ``eta`` (``make_config(eta=...)``); ``eta`` here must equal it."""
        cfg = self._e.cfg
        ddim = cfg.sched_kind == _lib.SCHED_DDIM
        if ddim and C.c_float(eta).value != cfg.eta:
            raise ValueError(f"eta={eta} differs from the configured eta={cfg.eta}; build the model with that eta")
        if variance_noise is not None:
            noise = variance_noise
        if generator is not None and noise is not None:
            raise ValueError("pass either generator or variance_noise, not both")
        t = int(timestep.reshape(-1)[0]) if torch.is_tensor(timestep) else int(timestep)
        if noise is None and (eta > 0 if ddim else t > 0):
            noise = torch.randn(model_output.shape, generator=generator, device=model_output.device,
                                dtype=model_output.dtype)
        return SimpleNamespace(prev_sample=self._e.scheduler_step(model_output, t, sample, noise))


class B200MLD:
    """Text/action-to-motion sampler with the reference ``MLD`` call surface.

    ``cfg_kwargs`` are :func:`make_config`'s, the scheduler's among them: ``scheduler``, ``eta``,
    ``beta_schedule``, ``clip_sample``, ...  When the scheduler adds noise at its steps (DDIM with ``eta > 0``,
    DDPM), :meth:`forward` draws with torch's default generator in the reference's order: the initial latents,
    then one ``[B, n_lat, d]`` draw per step (DDPM: none for the last step, ``t == 0``, whose slice stays zero).
    ``batch["init_noise"]`` and ``batch["step_noise"]`` ([n_steps, B, n_lat, d]) replace those draws."""

    def __init__(self, denoiser_sd: Dict[str, torch.Tensor], vae_sd: Dict[str, torch.Tensor], *,
                 mean: torch.Tensor, std: torch.Tensor, text_encoder: Optional[Callable] = None,
                 device: int = 0, num_inference_timesteps: int = 50, condition: str = "text",
                 stage: str = "diffusion", **cfg_kwargs):
        self.cfg = make_config(condition=condition, **cfg_kwargs)
        self.engine = Engine(self.cfg, device)
        self.engine.load_state_dict(denoiser_sd, "denoiser.")
        self.engine.load_state_dict(vae_sd, "vae.")
        self.engine.finalize()
        self.engine.set_mean_std(mean, std)
        self.scheduler = B200Scheduler(self.engine)
        self.scheduler.set_timesteps(num_inference_timesteps)
        self.text_encoder = text_encoder
        self.condition = condition
        self.stage = stage
        self.guidance_scale = float(self.cfg.guidance_scale)
        self.do_classifier_free_guidance = self.guidance_scale > 1.0          # mld.py:115
        self.latent_dim = [self.cfg.n_lat, self.cfg.latent_dim]
        self.device = self.engine.device

    # -- mld.py:216-265 ------------------------------------------------------------------
    def forward(self, batch) -> List[torch.Tensor]:
        lengths = batch["length"]
        if self.stage in ("diffusion", "vae_diffusion"):
            text_emb = self._encode_condition(batch)
            noise = batch.get("init_noise")
            if noise is None:                                                  # mld.py:303-307
                B = len(lengths)
                noise = torch.randn((B, self.latent_dim[0], self.latent_dim[-1]), device=self.device,
                                    dtype=torch.float)
            step_noise = batch.get("step_noise")
            if step_noise is None:
                step_noise = self._draw_step_noise(noise.shape[0])
            out = self.engine.sample(text_emb, noise, lengths, want=("joints",), step_noise=step_noise)
            joints = out["joints"]
        elif self.stage == "vae":
            z, _ = self._encode_motion(batch["motion"], lengths)
            feats = self.engine.vae_decode(z, lengths)
            joints = self.engine.feats2joints(feats)
        else:
            raise ValueError(self.stage)
        return remove_padding(joints.cpu(), lengths)                          # mld.py:264-265

    __call__ = forward

    def _encode_condition(self, batch) -> torch.Tensor:
        if "text_emb" in batch:                       # pre-computed CLIP output [2B, S, 768]
            return batch["text_emb"]
        if self.condition == "action":
            actions = batch["action"]
            if self.do_classifier_free_guidance:                               # mld.py:716-717
                actions = torch.cat([torch.zeros_like(actions), actions], 0)
            return actions
        texts = list(batch["text"])
        if self.do_classifier_free_guidance:                                   # mld.py:224-230
            texts = [""] * len(texts) + texts
        if self.text_encoder is None:
            raise RuntimeError("no text_encoder was given; pass batch['text_emb'] instead")
        return self.text_encoder(texts)

    # -- mld.py:290-360 ------------------------------------------------------------------
    def _diffusion_reverse(self, encoder_hidden_states: torch.Tensor, lengths=None,
                           init_noise: Optional[torch.Tensor] = None,
                           step_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        bsz = encoder_hidden_states.shape[0]
        if self.do_classifier_free_guidance:
            bsz = bsz // 2
        if init_noise is None:
            init_noise = torch.randn((bsz, self.latent_dim[0], self.latent_dim[-1]), device=self.device,
                                     dtype=torch.float)
        if step_noise is None:
            step_noise = self._draw_step_noise(bsz)
        return self.engine.diffusion_reverse(encoder_hidden_states, init_noise * self.scheduler.init_noise_sigma,
                                             lengths, step_noise=step_noise)

    def _draw_step_noise(self, B: int) -> Optional[torch.Tensor]:
        """The N(0,1) draws of the reference loop's ``scheduler.step`` calls (mld.py:345), in its order, as
        ``[n_steps, B, n_lat, d]``: DDIM with eta > 0 draws at every step, DDPM at every step with t > 0
        (the slice of a step that draws nothing is zero).  None when no step draws (DDIM, eta == 0)."""
        if not self.engine.stochastic:
            return None
        shape = (B, self.latent_dim[0], self.latent_dim[-1])
        ddpm = self.cfg.sched_kind == _lib.SCHED_DDPM
        ts = self.scheduler.timesteps.tolist()
        out = torch.zeros((len(ts), *shape), device=self.device, dtype=torch.float)
        for i, t in enumerate(ts):
            if not (ddpm and t == 0):
                out[i] = torch.randn(shape, device=self.device, dtype=torch.float)
        return out

    def _encode_motion(self, motion: torch.Tensor, lengths: Sequence[int]):
        mu, logvar = self.engine.vae_encode(motion, lengths)
        std = logvar.exp().pow(0.5)
        dist = torch.distributions.Normal(mu, std)
        return dist.rsample(), dist

    # -- mld.py:267-288 ------------------------------------------------------------------
    def gen_from_latent(self, batch):
        feats = self.engine.vae_decode(batch["latent"], batch["length"])
        return remove_padding(self.engine.feats2joints(feats).cpu(), batch["length"])

    def recon_from_motion(self, batch):
        feats_ref, length = batch["motion"], batch["length"]
        z, _ = self._encode_motion(feats_ref, length)
        feats = self.engine.vae_decode(z, length)
        joints = self.engine.feats2joints(feats).cpu()
        joints_ref = self.engine.feats2joints(feats_ref).cpu()
        return remove_padding(joints, length), remove_padding(joints_ref, length)

    def feats2joints(self, feats: torch.Tensor) -> torch.Tensor:
        return self.engine.feats2joints(feats)
