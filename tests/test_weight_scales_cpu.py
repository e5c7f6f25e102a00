"""The weight-exponent helpers of tests/weight_scales.py (no GPU): ``weight_at`` gives the exponent it claims, and
``with_outliers`` moves every pack of every synthetic state dict off s = 14 with the spread the GPU tests rely on,
changing values only."""
import pytest
import torch

from mld_b200 import synth
from split16_ref import weight_scale_log2
from weight_scales import OUTLIERS, engine_exponent, is_packed, packed_exponents, weight_at, with_outliers

SDS = {
    "denoiser_text": lambda: synth.denoiser_state_dict(1234),
    "denoiser_action": lambda: synth.denoiser_state_dict(2345, condition="action", num_layers=15, nfeats=150),
    "denoiser_novae": lambda: synth.denoiser_state_dict(3456, arch="trans_dec", d=512, diffusion_only=True),
    "mld_vae": lambda: synth.mld_vae_state_dict(4321),
    "actor_vae": lambda: synth.actor_vae_state_dict(777),
    "clip": lambda: synth.clip_text_state_dict(4242, layers=2),
    "t2m_text": lambda: synth.t2m_state_dicts()["text_encoder"],
    "t2m_movement": lambda: synth.t2m_state_dicts()["movement_encoder"],
    "t2m_motion": lambda: synth.t2m_state_dicts()["motion_encoder"],
}


@pytest.fixture(scope="module", params=sorted(SDS))
def pair(request):
    sd = SDS[request.param]()
    return request.param, sd, with_outliers(sd, seed=7)


@pytest.mark.parametrize("s", range(-14, 15))
def test_weight_at_gives_its_exponent(s):
    W = weight_at(37, 96, s, torch.Generator().manual_seed(s + 100))
    assert W.dtype == torch.float32 and W.shape == (37, 96)
    assert engine_exponent(W) == weight_scale_log2(W) == s
    assert float(W.abs().max()) == 1.5 * 2.0 ** (13 - s)


def test_engine_exponent_edges():
    assert engine_exponent(torch.zeros(4, 8)) == 0
    assert engine_exponent(torch.full((2, 2), 1e-38)) == 14          # 16384 / max overflows fp32: clamped, not UB
    assert engine_exponent(torch.full((2, 2), 1e12)) == -14
    W = torch.full((4, 8), 3.0)
    for bad in (float("inf"), float("-inf"), float("nan")):
        W[1, 3] = bad
        assert engine_exponent(W) == 12, bad                           # the finite elements set the scale
    assert engine_exponent(torch.full((2, 2), float("inf"))) == 0
    for mag, s in OUTLIERS.items():
        assert weight_scale_log2(torch.tensor([[mag]])) == s


def test_synthetic_weights_all_sit_at_the_clamp(pair):
    """What makes this helper necessary: every pack of the unmodified synthetic weights is at s = 14."""
    _, sd, _ = pair
    assert set(packed_exponents(sd).values()) == {14}


def test_outliers_change_values_only(pair):
    _, sd, mod = pair
    assert list(mod) == list(sd)
    for k in sd:
        assert mod[k].shape == sd[k].shape and mod[k].dtype == sd[k].dtype, k
        changed = int((mod[k] != sd[k]).sum())
        if not is_packed(k, sd[k]):
            assert changed == 0, f"table {k} was modified"
        else:
            assert 2 <= changed <= 6 and set(mod[k][mod[k] != sd[k]].abs().tolist()) <= set(OUTLIERS), k
    assert with_outliers(sd, seed=7).keys() == mod.keys()
    assert all(torch.equal(a, b) for a, b in zip(with_outliers(sd, seed=7).values(), mod.values())), "seeded"


def test_outliers_move_every_pack_off_14(pair):
    name, _, mod = pair
    ex = packed_exponents(mod)
    assert ex and all(s in OUTLIERS.values() for s in ex.values()), (name, {k: s for k, s in ex.items() if s == 14})


def test_outliers_spread_within_layers(pair):
    """The exponents a kernel could mix up in one launch, or an engine could take from the wrong pack, differ."""
    name, _, mod = pair
    ex = packed_exponents(mod)
    trios = 0
    for k in ex:
        for l1, l2 in (("linear1.weight", "linear2.weight"), ("mlp.fc1.weight", "mlp.fc2.weight")):
            if k.endswith(l1):
                p = k[:-len(l1)]
                trio = {ex[p + "self_attn.out_proj.weight"], ex[k], ex[p + l2]}
                assert len(trio) == 3, (name, p)
                trios += 1
    subs = 0
    for k in ex:
        if k.endswith("self_attn.in_proj_weight[q]"):
            base = k[:-len("[q]")]
            assert ex[k] != ex[base] and ex[k] != ex[base + "[kv]"], (name, k)
            subs += 1
        if k.endswith("multihead_attn.in_proj_weight[q]"):
            base = k[:-len("[q]")]
            assert len({ex[k], ex[base + "[kv]"], ex[base + "[v]"]}) == 3, (name, k)
            subs += 1
        if k.endswith("gru.weight_hh"):
            p = k[:-len("weight_hh")]
            assert len({ex[k], ex[p + "weight_ih_l0"], ex[p + "weight_ih_l0_reverse"]}) == 3, (name, k)
            subs += 1
    if name == "clip":
        for i in range(2):
            p = f"text_model.text_model.encoder.layers.{i}.self_attn."
            assert len({engine_exponent(mod[p + n + "_proj.weight"]) for n in "qkv"}) == 3
    expect = {"denoiser_text": (9, 1), "denoiser_action": (15, 1), "denoiser_novae": (9, 9), "mld_vae": (18, 10),
              "actor_vae": (12, 7), "clip": (2, 0), "t2m_text": (0, 1), "t2m_movement": (0, 0), "t2m_motion": (0, 1)}
    assert (trios, subs) == expect[name]


def test_outliers_keep_the_model(pair):
    """Only a handful of elements move, so outputs stay in the range the synthetic model gives."""
    _, sd, mod = pair
    for k in sd:
        if is_packed(k, sd[k]):
            assert float(sd[k].abs().max()) < min(OUTLIERS), k
            assert float(mod[k].abs().max()) in OUTLIERS, k
