"""CPU tests of the HumanAct12 action classifier port: the float64 restatement against the fixture made with the
reference's own modules (and float64 against fp32), the drop-ins' state-dict contract, their initial-state draw, the
default config, and the argument checks that run before anything touches a GPU."""
import pytest
import torch

from conftest import golden
from mld_b200 import synth
from oracle import a2m_gru as O
from oracle.make_golden_a2m import EXPLICIT_LENS, RNG_SEED, SEEDED_LENS, WEIGHT_SEED, golden_inputs, key_list

torch.set_grad_enabled(False)


def _rel_rows(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float(((a - b).abs().max(1).values / b.abs().max(1).values).max())


@pytest.fixture(scope="module")
def sd():
    return synth.a2m_state_dict(WEIGHT_SEED)


def test_restatement_matches_reference_golden(sd):
    g = golden("a2m_gru.npz")
    x1, h0, x2 = golden_inputs()
    sd64 = {k: v.double() for k, v in sd.items()}
    logits, feats = O.classify(sd64, x1.double(), EXPLICIT_LENS, h0.double())
    assert _rel_rows(logits, g["logits_explicit"]) < 1e-5
    assert _rel_rows(feats, g["features_explicit"]) < 1e-5
    L, H = synth.A2M_DIMS["hidden_layer"], synth.A2M_DIMS["hidden_size"]
    torch.manual_seed(RNG_SEED)
    ha, hb = torch.randn(L, len(SEEDED_LENS), H), torch.randn(L, len(SEEDED_LENS), H)
    assert _rel_rows(O.classify(sd64, x2.double(), SEEDED_LENS, ha.double())[0], g["logits_seeded"]) < 1e-5
    assert _rel_rows(O.classify(sd64, x2.double(), SEEDED_LENS, hb.double())[1], g["features_seeded"]) < 1e-5


def test_float64_matches_fp32(sd):
    x1, h0, _ = golden_inputs()
    l64, f64 = O.classify({k: v.double() for k, v in sd.items()}, x1.double(), EXPLICIT_LENS, h0.double())
    l32, f32 = O.classify(sd, x1, EXPLICIT_LENS, h0)
    assert _rel_rows(l32, l64) < 1e-5 and _rel_rows(f32, f64) < 1e-5


def test_torch_yardstick_matches_restatement(sd):
    x1, h0, _ = golden_inputs()
    net = O.TorchDiscriminator(sd, **synth.A2M_DIMS)
    logits, feats = net.both(x1, torch.tensor(EXPLICIT_LENS), h0)
    l64, f64 = O.classify({k: v.double() for k, v in sd.items()}, x1.double(), EXPLICIT_LENS, h0.double())
    assert _rel_rows(logits, l64) < 1e-5 and _rel_rows(feats, f64) < 1e-5


def test_synth_keys_match_fixture(sd):
    assert list(key_list(sd)) == list(golden("a2m_gru.npz")["keys"])


def _dropins(**dims):
    from mld_b200.evaluator import B200MotionDiscriminator, B200MotionDiscriminatorForFID
    d = {**synth.A2M_DIMS, **dims}
    return B200MotionDiscriminator(**d), B200MotionDiscriminatorForFID(**d)


@pytest.mark.parametrize("dims", [{}, {"hidden_size": 64, "hidden_layer": 3, "output_size": 5}])
def test_dropins_keep_reference_state_dict_keys(dims):
    d = {**synth.A2M_DIMS, **dims}
    ref = O.TorchDiscriminator(synth.a2m_state_dict(1, **dims), **d).state_dict()     # nn.GRU's own key names
    for m in _dropins(**dims):
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.items()}
        m.load_state_dict(ref, strict=True)                                           # reference -> drop-in
        O.TorchDiscriminator(m.state_dict(), **d)                                      # drop-in -> reference (strict)
        with pytest.raises(RuntimeError):
            m.load_state_dict({**ref, "extra.weight": torch.zeros(1)}, strict=True)
        assert (m.input_size, m.hidden_size, m.hidden_layer, m.use_noise) == (d["input_size"], d["hidden_size"],
                                                                            d["hidden_layer"], None)
    assert list(key_list(_dropins()[0].state_dict())) == list(golden("a2m_gru.npz")["keys"])


def test_init_hidden_draws_as_the_reference():
    cls, fid = _dropins()
    torch.manual_seed(5)
    a = cls.initHidden(7, 2)
    b = fid.initHidden(7, 2)
    after = torch.get_rng_state()
    torch.manual_seed(5)
    ra, rb = torch.randn(2, 7, 128, requires_grad=False), torch.randn(2, 7, 128, requires_grad=False)
    assert torch.equal(a, ra) and torch.equal(b, rb) and a.shape == (2, 7, 128)
    assert torch.equal(after, torch.get_rng_state())


def test_default_config_is_the_shipped_one(built_lib):
    from mld_b200 import _lib
    c = _lib.default_a2m_config()
    assert c.abi_version == _lib.MLDB_A2M_ABI_VERSION == 1
    assert {k: getattr(c, k) for k in synth.A2M_DIMS} == synth.A2M_DIMS
    assert _lib.MLDB_ABI_VERSION == 4 and len(_lib.KSTAT_NAMES) == 12


def test_dropins_refuse_bad_lengths_before_any_launch():
    cls, fid = _dropins()
    x = torch.zeros(3, 24, 3, 10)
    for m in (cls, fid):
        for bad in ([10, 0, 5], [11, 3, 3], [1, 2], None, torch.tensor([1.0, 2.0, 3.0])):
            with pytest.raises(ValueError):
                m(x, lengths=bad)
