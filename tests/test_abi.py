"""CPU: the C-ABI library loads and exports every symbol include/mldb.h declares; the host
logic that needs no GPU behaves (errors are loud, there is no fallback)."""
import ctypes as C
import os
import re

import pytest
import torch

from conftest import ROOT
from mld_b200 import _lib


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "mldb.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mldb_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported(built_lib):
    names = _declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(built_lib, n), f"{n} declared in include/mldb.h but not exported"
        assert n in _lib._SIGNATURES, f"{n} has no ctypes signature in mld_b200/_lib.py"
    assert built_lib.mldb_abi_version() == _lib.MLDB_ABI_VERSION


def test_config_struct_layout_matches_header(built_lib):
    cfg = _lib.default_config()
    # defaults == shipped yaml (configs/modules/denoiser.yaml, motion_vae.yaml, scheduler.yaml)
    assert (cfg.latent_dim, cfg.n_lat, cfg.num_heads, cfg.ff_size, cfg.num_layers) == (256, 1, 4, 1024, 9)
    assert (cfg.text_dim, cfg.vae_layers, cfg.vae_nfeats, cfg.njoints) == (768, 9, 263, 22)
    assert abs(cfg.guidance_scale - 7.5) < 1e-6 and cfg.beta_start == 0.00085 and cfg.beta_end == 0.012
    assert (cfg.num_train_timesteps, cfg.steps_offset, cfg.set_alpha_to_one) == (1000, 1, 0)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_no_cpu_fallback(built_lib):
    cfg = _lib.default_config()
    h = C.c_void_p()
    rc = built_lib.mldb_create(C.byref(cfg), 0, C.byref(h))
    assert rc != 0 and h.value is None
    assert built_lib.mldb_last_error()          # a message is recorded
    from mld_b200.engine import Engine
    with pytest.raises(RuntimeError):
        Engine(cfg, 0)


@pytest.mark.parametrize("field, value, code, cause", [
    ("abi_version", -1, 1, b"abi_version"),
    ("latent_dim", 250, 1, b"latent_dim must be a multiple"),
    ("latent_dim", 2048, 4, b"latent_dim > 1024"),
])
def test_create_failure_records_its_own_message(built_lib, field, value, code, cause):
    """A refused mldb_create names its own cause: the message of an earlier failure is never left behind."""
    stale = _lib.default_config()
    stale.eta = 1.25
    assert built_lib.mldb_create(C.byref(stale), 0, C.byref(C.c_void_p())) == 1
    assert b"eta" in built_lib.mldb_last_error()
    cfg = _lib.default_config()
    setattr(cfg, field, value)
    h = C.c_void_p()
    assert built_lib.mldb_create(C.byref(cfg), 0, C.byref(h)) == code and h.value is None
    msg = built_lib.mldb_last_error()
    assert cause in msg and b"eta" not in msg, msg


def test_modules_keep_reference_state_dict_keys():
    """The drop-in modules expose exactly the reference's state-dict keys and shapes."""
    from types import SimpleNamespace
    from mld_b200 import synth
    from mld_b200.modules import B200ActorVae, B200MldDenoiser, B200MldVae
    abl = SimpleNamespace(SKIP_CONNECT=True, VAE_TYPE="mld", DIFF_PE_TYPE="mld", PE_TYPE="mld", MLP_DIST=False)
    den = B200MldDenoiser(ablation=abl, nfeats=263, condition="text", latent_dim=[1, 256], ff_size=1024,
                          num_layers=9, num_heads=4, arch="trans_enc", text_encoded_dim=768)
    ref = synth.denoiser_state_dict(1234)
    assert {k: tuple(v.shape) for k, v in den.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.items()}
    den.load_state_dict(ref, strict=True)
    vae = B200MldVae(ablation=abl, nfeats=263, latent_dim=[1, 256], arch="encoder_decoder")
    vae.load_state_dict(synth.mld_vae_state_dict(4321), strict=True)
    act = B200ActorVae(ablation=abl, nfeats=150, latent_dim=[1, 256], num_layers=6)
    act.load_state_dict(synth.actor_vae_state_dict(777), strict=True)
    with pytest.raises(RuntimeError):        # CPU tensors: loud failure, no fallback
        den(torch.zeros(2, 1, 256), torch.tensor(1), torch.zeros(2, 1, 768))
