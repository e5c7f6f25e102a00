"""CPU: the CLIP text tower's plain-torch restatement against transformers (tests/golden/clip_text.npz), the
synthetic state dict's key contract, and B200TextEncoder's host-side logic (argument checks, the two exact
savings) - none of which needs a GPU."""
import pytest
import torch

from conftest import golden
from mld_b200 import synth
from mld_b200.text import B200TextEncoder, ClipTextConfig, eos_positions, plan_ids
from oracle.clip_text import ClipTextCfg, clip_text_forward
from oracle.make_golden_clip import WEIGHT_SEED, golden_ids

torch.set_grad_enabled(False)
SMALL = dict(vocab_size=1000, max_positions=77, hidden=128, heads=2, layers=2, ff=256, projection_dim=64)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max())


@pytest.fixture(scope="module")
def full_sd():
    return synth.clip_text_state_dict(WEIGHT_SEED)


def test_oracle_matches_transformers_golden(full_sd):
    g, ids = golden("clip_text.npz"), golden_ids()
    hid = clip_text_forward(full_sd, ids, "clip_hidden", ClipTextCfg())[:, torch.from_numpy(g["hidden_pos"])]
    for s in range(ids.shape[0]):
        assert _rel(hid[s], g["hidden"][s]) < 1e-5
    pooled = clip_text_forward(full_sd, ids, "clip", ClipTextCfg())
    assert pooled.shape == (ids.shape[0], 1, 768)
    assert _rel(pooled[:, 0], g["pooled"]) < 1e-5
    legacy = clip_text_forward(full_sd, ids, "clip", ClipTextCfg(eos_token_id=2))
    assert _rel(legacy[:, 0], g["pooled_legacy"]) < 1e-5


def test_eos_rules():
    ids = torch.tensor([[49406, 320, 49407, 49407], [49406, 320, 321, 322], [5, 49407, 9, 49407]])
    assert eos_positions(ids, 49407).tolist() == [2, 0, 1]          # first eos; 0 when absent
    assert eos_positions(ids, 2).tolist() == [2, 0, 1]              # legacy: argmax, first maximum


def test_synth_keys_are_the_text_tower_of_mld_text_encoder():
    transformers = pytest.importorskip("transformers")
    shape = dict(vocab_size=1000, max_positions=77, hidden=64, layers=2, ff=128, projection_dim=32)
    sd = synth.clip_text_state_dict(3, **shape)
    tcfg = transformers.CLIPTextConfig(vocab_size=1000, hidden_size=64, intermediate_size=128, projection_dim=32,
                                       num_hidden_layers=2, num_attention_heads=2, max_position_embeddings=77)
    # MldTextEncoder.text_model is AutoModel.from_pretrained(clip path): a CLIPModel (text + vision towers)
    vcfg = transformers.CLIPVisionConfig(hidden_size=32, intermediate_size=64, num_hidden_layers=1,
                                         num_attention_heads=2, image_size=32, patch_size=16)
    full = transformers.CLIPModel(transformers.CLIPConfig(text_config=tcfg.to_dict(), vision_config=vcfg.to_dict(),
                                                          projection_dim=32))
    tower = {"text_model." + k: tuple(v.shape) for k, v in full.state_dict().items()
             if k.startswith(("text_model.", "text_projection.")) and not k.endswith("position_ids")}
    assert {k: tuple(v.shape) for k, v in sd.items()} == tower
    m = transformers.CLIPTextModelWithProjection(tcfg)
    m.load_state_dict({k[len("text_model."):]: v for k, v in sd.items()}, strict=True)


def test_text_encoder_rejects_before_touching_a_device():
    sd = synth.clip_text_state_dict(1, **SMALL)
    with pytest.raises(NotImplementedError):
        B200TextEncoder("./deps/clip-vit-large-patch14", finetune=True)
    with pytest.raises(ValueError):
        B200TextEncoder("./deps/distilbert-base-uncased")
    enc = B200TextEncoder.from_state_dict(sd, config=ClipTextConfig(**SMALL))
    assert set(enc.state_dict()) == set(sd)
    for bad in (torch.tensor([[1, 1000]]), torch.tensor([[-1, 3]]), torch.ones(1, 78, dtype=torch.long),
                torch.ones(2, 3)):
        with pytest.raises((ValueError, TypeError)):
            enc.encode_ids(bad)
    with pytest.raises(RuntimeError):          # no tokenizer was given
        enc([""])
    # the position_ids buffer of older checkpoints is dropped when it is arange, refused otherwise
    B200TextEncoder.from_state_dict({**sd, "text_model.text_model.embeddings.position_ids": torch.arange(77)[None]},
                                    config=ClipTextConfig(**SMALL))
    with pytest.raises(ValueError):
        B200TextEncoder.from_state_dict({**sd, "text_model.text_model.embeddings.position_ids": torch.zeros(1, 77)},
                                        config=ClipTextConfig(**SMALL))


@pytest.mark.parametrize("eos", [999, 2])
def test_dedupe_and_eos_truncation_are_exact(eos):
    """The host-side savings: distinct rows once, and in pooled mode the columns after the last eos dropped."""
    cfg = ClipTextCfg(**{**SMALL, "eos_token_id": eos})
    sd = synth.clip_text_state_dict(2, **SMALL)
    ids = synth.clip_text_ids(6, 77, seed=9, eos_lo=3, eos_hi=20, vocab_size=999, bos=998, eos=999)
    ids = torch.cat([torch.tensor([[998] + [999] * 76] * 3), ids])          # three identical "" rows first
    if eos == 2:
        ids[ids == 999] = 2
        ids[ids == 998] = 0
        ids[:, 1:] = torch.where(ids[:, 1:] == 2, ids[:, 1:], ids[:, 1:] % 2)   # words below the eos id
    rows, inv = plan_ids(ids, True, eos)
    assert rows.shape[0] == ids.shape[0] - 2
    assert rows.shape[1] == int(eos_positions(ids, eos).max()) + 1 < 77
    full = clip_text_forward(sd, ids, "clip", cfg)
    assert _rel(clip_text_forward(sd, rows, "clip", cfg)[inv], full) < 1e-12
    rows_h, inv_h = plan_ids(ids, False, eos)
    assert rows_h.shape == (ids.shape[0] - 2, 77)
    assert torch.equal(rows_h[inv_h], ids)
