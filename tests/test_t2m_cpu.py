"""CPU tests of the T2M evaluator port: the float64 restatement against the fixture made with the reference's own
modules, the synthetic weights' key/shape contract, the default config, and the drop-in modules' argument checks
(which run before anything touches a GPU)."""
import pytest
import torch

from conftest import golden
from mld_b200 import synth
from oracle import t2m_eval as O
from oracle.make_golden_t2m import MOTION_LENS, MOVE_HEAD, TEXT_LENS, WEIGHT_SEED, golden_inputs, key_list

torch.set_grad_enabled(False)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


@pytest.fixture(scope="module")
def sd64():
    return {k: {kk: vv.double() for kk, vv in v.items()} for k, v in synth.t2m_state_dicts(WEIGHT_SEED).items()}


def test_restatement_matches_reference_golden(sd64):
    g = golden("t2m_eval.npz")
    word, pos, motions = golden_inputs()
    text = O.text(sd64["text_encoder"], word.double(), pos.double(), TEXT_LENS)
    assert _rel(text, g["text_emb"]) < 1e-5
    mov = O.movement(sd64["movement_encoder"], motions[..., :-4].double())
    assert mov.shape == (len(MOTION_LENS), 49, 512)
    assert _rel(mov[:, :MOVE_HEAD], g["movement_head"]) < 1e-5
    emb = O.motion(sd64["motion_encoder"], mov, [n // 4 for n in MOTION_LENS])
    assert _rel(emb, g["motion_emb"]) < 1e-5


def test_synth_keys_match_fixture():
    g = golden("t2m_eval.npz")
    assert list(key_list(synth.t2m_state_dicts(0))) == list(g["keys"])


def test_padding_frames_are_not_zero_after_renorm():
    """renorm4t2m maps the zero padding rows of normalised motions to (mean - mean_eval) / std_eval."""
    _, _, motions = golden_inputs()
    n = MOTION_LENS[-1]
    assert motions[-1, n:].abs().min() > 0


def test_default_config_is_the_shipped_yaml(built_lib):
    from mld_b200 import _lib
    c = _lib.default_t2m_config()
    assert c.abi_version == _lib.MLDB_T2M_ABI_VERSION == 1
    assert c.parts == _lib.T2M_TEXT | _lib.T2M_MOVEMENT | _lib.T2M_MOTION
    got = {k: getattr(c, k) for k in synth.T2M_DIMS}
    assert got == synth.T2M_DIMS
    assert _lib.KSTAT_NAMES.index("gru_tc") == 11 and len(_lib.KSTAT_NAMES) == 12


def _modules():
    from mld_b200.evaluator import B200MotionEncoderBiGRUCo, B200MovementConvEncoder, B200TextEncoderBiGRUCo
    te = B200TextEncoderBiGRUCo(word_size=300, pos_size=15, hidden_size=512, output_size=512)
    mv = B200MovementConvEncoder(input_size=259, hidden_size=512, output_size=512)
    mo = B200MotionEncoderBiGRUCo(input_size=512, hidden_size=1024, output_size=512)
    return te, mv, mo


def test_modules_keep_reference_state_dict_keys():
    sds = synth.t2m_state_dicts(WEIGHT_SEED)
    for m, k in zip(_modules(), ("text_encoder", "movement_encoder", "motion_encoder")):
        assert {n: tuple(v.shape) for n, v in m.state_dict().items()} == {n: tuple(v.shape) for n, v in sds[k].items()}
        m.load_state_dict(sds[k], strict=True)
        with pytest.raises(RuntimeError):
            m.load_state_dict({**sds[k], "extra.weight": torch.zeros(1)}, strict=True)


def test_modules_refuse_what_pack_padded_sequence_refuses():
    te, _, mo = _modules()
    x = torch.zeros(3, 10, 512)
    w, p = synth.t2m_text_inputs(3, 5)
    for bad in ([10, 0, 0], [4, 10, 2], torch.tensor([3, 5, 4])):
        with pytest.raises(RuntimeError, match="greater than 0|decreasing"):
            mo(x, bad)
    with pytest.raises(RuntimeError, match="greater than 0|decreasing"):
        te(w, p, torch.tensor([5, 0, 0]))
    with pytest.raises(RuntimeError, match="exceeds"):
        te(w, p, torch.tensor([6, 5, 1]))
    with pytest.raises(ValueError):
        te(w, p, torch.tensor([5, 1]))
    # valid lengths on CPU tensors: a loud failure, no fallback
    with pytest.raises(RuntimeError, match="H100"):
        mo(x, torch.tensor([10, 4, 1]))
