"""The ActorVae encoder's oracle (CPU): against the reference's own ``ActorVae.encode`` through
tests/golden/vae_actor_encode.npz, and the float64 restatement against the fp32 one."""
import pytest
import torch

from conftest import golden
from mld_b200 import synth
from oracle import mld_oracle as O
from oracle.actor_encode import actor_encode
from oracle.make_golden_actor_encode import CASES, NFEATS, NUM_LAYERS, WEIGHT_SEED, case_motion

torch.set_grad_enabled(False)
CFG = O.VaeCfg(kind="actor", nfeats=NFEATS, num_layers=NUM_LAYERS)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("tag", sorted(CASES))
def test_actor_encode_oracle_matches_reference(tag):
    g = golden("vae_actor_encode.npz")
    sd = synth.actor_vae_state_dict(seed=WEIGHT_SEED)
    mu, logvar = actor_encode(sd, CFG, case_motion(tag), CASES[tag][2])
    assert mu.shape == logvar.shape == (1, len(CASES[tag][2]), 256)
    assert _rel(mu[0], g[f"{tag}_mu"]) < 1e-5
    assert _rel(logvar[0].exp().pow(0.5), g[f"{tag}_std"]) < 1e-5


def test_actor_encode_oracle_float64_matches_float32():
    sd = synth.actor_vae_state_dict(seed=WEIGHT_SEED)
    sd64 = {k: v.double() for k, v in sd.items()}
    motion, lengths = case_motion("a"), CASES["a"][2]
    mu, logvar = actor_encode(sd, CFG, motion, lengths)
    mu64, logvar64 = actor_encode(sd64, CFG, motion, lengths)
    assert mu64.dtype == torch.float64 and mu.dtype == torch.float32
    assert _rel(mu, mu64) < 1e-5 and _rel(logvar, logvar64) < 1e-5


def test_actor_dropin_keeps_reference_state_dict_keys():
    """B200ActorVae registers the encoder keys it now uses, with the reference's names and shapes."""
    from types import SimpleNamespace
    from mld_b200.modules import B200ActorVae
    m = B200ActorVae(ablation=SimpleNamespace(), nfeats=NFEATS, latent_dim=[1, 256], num_layers=NUM_LAYERS)
    ref = synth.actor_vae_state_dict(seed=WEIGHT_SEED)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.items()}
    assert any(k.startswith("encoder.seqTransEncoder.") for k in ref)


def test_actor_encode_is_vae_false_raises():
    from types import SimpleNamespace
    from mld_b200.modules import B200ActorVae
    m = B200ActorVae(ablation=SimpleNamespace(), nfeats=NFEATS, latent_dim=[1, 256], num_layers=1, is_vae=False)
    with pytest.raises(NotImplementedError, match="is_vae"):
        m.encode(torch.zeros(1, 4, NFEATS))
