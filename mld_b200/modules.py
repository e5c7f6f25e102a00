"""Drop-in replacements for the reference's networks, selectable through the YAML ``target:``
factory (``instantiate_from_config``, mld/config.py:106-121):

    denoiser.target:   mld_b200.modules.B200MldDenoiser     (was mld...mld_denoiser.MldDenoiser)
    motion_vae.target: mld_b200.modules.B200MldVae          (was mld...mld_vae.MldVae)
                       mld_b200.modules.B200ActorVae        (was mld...actor_vae.ActorVae)

Same ctor kwargs, same ``state_dict`` keys/shapes (so ``load_state_dict(strict=True)`` of a
reference checkpoint works, demo.py:150), same call signatures and return conventions; the
math runs in ``libmldb200.so``.  Inference only (parameters do not require grad).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
from torch import nn

from . import synth
from .engine import Engine, make_config


def _register_tree(root: nn.Module, tensors: Dict[str, torch.Tensor]):
    """Create nested sub-modules so that ``root.state_dict()`` has exactly these keys."""
    for key, value in tensors.items():
        parts = key.split(".")
        m = root
        for p in parts[:-1]:
            if p not in m._modules:
                m.add_module(p, nn.Module())
            m = m._modules[p]
        m.register_parameter(parts[-1], nn.Parameter(value.clone(), requires_grad=False))


class _EngineModule(nn.Module):
    """Common machinery: lazily builds an ``Engine`` from the module's own parameters."""
    _prefix = ""

    def __init__(self):
        super().__init__()
        self._engine: Optional[Engine] = None
        self._engine_epoch = -1
        self._weights_epoch = 0

    def _make_config(self):
        raise NotImplementedError

    def _load_from_state_dict(self, *args, **kwargs):   # weights changed -> rebuild engine
        self._weights_epoch += 1
        return super()._load_from_state_dict(*args, **kwargs)

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        self._weights_epoch += 1
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def engine(self) -> Engine:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError(f"{type(self).__name__} runs on a H100 only: move it with .cuda() "
                               "(no CPU/PyTorch fallback exists)")
        if self._engine is None or self._engine_epoch != self._weights_epoch or self._engine.device != dev:
            eng = Engine(self._make_config(), dev)
            eng.load_state_dict(self.state_dict(), self._prefix)
            eng.finalize()
            self._engine, self._engine_epoch = eng, self._weights_epoch
        return self._engine


class B200MldDenoiser(_EngineModule):
    """``MldDenoiser`` (mld/models/architectures/mld_denoiser.py:16-228)."""
    _prefix = "denoiser."

    def __init__(self, ablation, nfeats: int = 263, condition: str = "text", latent_dim: list = [1, 256],
                 ff_size: int = 1024, num_layers: int = 6, num_heads: int = 4, dropout: float = 0.1,
                 normalize_before: bool = False, activation: str = "gelu", flip_sin_to_cos: bool = True,
                 return_intermediate_dec: bool = False, position_embedding: str = "learned",
                 arch: str = "trans_enc", freq_shift: int = 0, guidance_scale: float = 7.5,
                 guidance_uncondp: float = 0.1, text_encoded_dim: int = 768, nclasses: int = 10,
                 **kwargs) -> None:
        super().__init__()
        if condition not in ("text", "action"):
            raise TypeError(f"condition type {condition} not supported")       # mld_denoiser.py:79
        if arch not in ("trans_enc", "trans_dec"):
            raise ValueError(f"Not supported architechure{arch}!")             # mld_denoiser.py:131
        if getattr(ablation, "DIFF_PE_TYPE", "mld") != "mld" or position_embedding != "learned":
            raise ValueError("Not Support PE type")                            # mld_denoiser.py:89
        if normalize_before or activation != "gelu" or not getattr(ablation, "SKIP_CONNECT", True):
            raise NotImplementedError("B200MldDenoiser implements the shipped configuration: post-norm, "
                                      "gelu, skip-connected encoder")
        self.latent_dim = latent_dim[-1]
        self.condition, self.arch = condition, arch
        self.diffusion_only = getattr(ablation, "VAE_TYPE", "mld") == "no"
        self._kw = dict(condition=condition, arch=arch, latent_dim=tuple(latent_dim), ff_size=ff_size,
                        num_layers=num_layers, num_heads=num_heads, text_encoded_dim=text_encoded_dim,
                        nclasses=nclasses, nfeats=nfeats, diffusion_only=self.diffusion_only,
                        flip_sin_to_cos=flip_sin_to_cos, freq_shift=float(freq_shift),
                        guidance_scale=guidance_scale)
        sd = synth.denoiser_state_dict(seed=0, condition=condition, arch=arch, d=self.latent_dim, ff=ff_size,
                                       num_layers=num_layers, text_dim=text_encoded_dim, nclasses=nclasses,
                                       nfeats=nfeats, diffusion_only=self.diffusion_only)
        _register_tree(self, sd)

    def _make_config(self):
        return make_config(vae="none", **self._kw)

    def forward(self, sample, timestep, encoder_hidden_states, lengths=None, **kwargs):
        # returns a 1-tuple like the reference (mld_denoiser.py:228)
        t = int(timestep.reshape(-1)[0]) if torch.is_tensor(timestep) else int(timestep)
        return (self.engine().denoise(sample, t, encoder_hidden_states, lengths),)


class B200MldVae(_EngineModule):
    """``MldVae`` (mld/models/architectures/mld_vae.py:33-248), arch ``encoder_decoder``."""
    _prefix = "vae."

    def __init__(self, ablation, nfeats: int, latent_dim: list = [1, 256], ff_size: int = 1024,
                 num_layers: int = 9, num_heads: int = 4, dropout: float = 0.1, arch: str = "all_encoder",
                 normalize_before: bool = False, activation: str = "gelu",
                 position_embedding: str = "learned", **kwargs) -> None:
        super().__init__()
        if arch != "encoder_decoder":
            raise ValueError("Not support architecture!") if arch != "all_encoder" else NotImplementedError(
                "B200MldVae implements arch='encoder_decoder' (configs/modules/motion_vae.yaml:5)")
        if getattr(ablation, "PE_TYPE", "mld") != "mld" or getattr(ablation, "MLP_DIST", False):
            raise NotImplementedError("B200MldVae implements PE_TYPE 'mld', MLP_DIST False")
        self.latent_size, self.latent_dim = latent_dim[0], latent_dim[-1]
        self._kw = dict(latent_dim=tuple(latent_dim), vae_ff=ff_size, vae_layers=num_layers,
                        vae_heads=num_heads, vae_nfeats=nfeats, nfeats=nfeats)
        _register_tree(self, synth.mld_vae_state_dict(seed=0, nfeats=nfeats, d=self.latent_dim, ff=ff_size,
                                                      num_layers=num_layers, n_lat=self.latent_size))

    def _make_config(self):
        return make_config(vae="mld", num_layers=0, **self._kw)

    def encode(self, features: torch.Tensor, lengths: Optional[List[int]] = None):
        if lengths is None:
            lengths = [len(f) for f in features]
        mu, logvar = self.engine().vae_encode(features, lengths)
        std = logvar.exp().pow(0.5)                                   # mld_vae.py:181-183
        dist = torch.distributions.Normal(mu, std)
        return dist.rsample(), dist

    def decode(self, z: torch.Tensor, lengths: List[int]):
        return self.engine().vae_decode(z, lengths)

    def forward(self, features, lengths=None):
        print("Should Not enter here")                                # mld_vae.py:118
        z, dist = self.encode(features, lengths)
        return self.decode(z, lengths), z, dist


class B200ActorVae(_EngineModule):
    """``ActorVae`` decode path (mld/models/architectures/actor_vae.py:11-235)."""
    _prefix = "vae."

    def __init__(self, ablation, nfeats: int, latent_dim: list = [1, 256], ff_size: int = 1024,
                 num_layers: int = 9, num_heads: int = 4, dropout: float = 0.1, is_vae: bool = True,
                 activation: str = "gelu", position_embedding: str = "learned", **kwargs) -> None:
        super().__init__()
        self.latent_size, self.latent_dim = latent_dim[0], latent_dim[-1]
        self._kw = dict(latent_dim=tuple(latent_dim), vae_ff=ff_size, vae_layers=num_layers,
                        vae_heads=num_heads, vae_nfeats=nfeats, nfeats=nfeats)
        _register_tree(self, synth.actor_vae_state_dict(seed=0, nfeats=nfeats, d=self.latent_dim, ff=ff_size,
                                                        num_layers=num_layers))

    def _make_config(self):
        return make_config(vae="actor", num_layers=0, **self._kw)

    def decode(self, z: torch.Tensor, lengths: List[int]):
        return self.engine().vae_decode(z, lengths)

    def encode(self, features, lengths=None):
        raise NotImplementedError("ActorVae.encode is not on the sampling path (SURVEY.md section 8)")
