"""Drop-in replacements for the T2M evaluator's three networks (``MLD._get_t2m_evaluator``,
mld/models/modeltype/mld.py:145-190), whose embeddings feed R-precision, matching score, FID, diversity and
MultiModality:

    t2m_textencoder:   mld_b200.evaluator.B200TextEncoderBiGRUCo   (was t2m_textenc.TextEncoderBiGRUCo)
    t2m_moveencoder:   mld_b200.evaluator.B200MovementConvEncoder  (was t2m_motionenc.MovementConvEncoder)
    t2m_motionencoder: mld_b200.evaluator.B200MotionEncoderBiGRUCo (was t2m_motionenc.MotionEncoderBiGRUCo)

Same ctor kwargs, same ``state_dict`` keys and shapes (``hidden`` included, so finest.tar's dicts load with
``strict=True``), same forward signatures and return shapes; the math runs in ``libmldb200.so``.  Inference only.
Like ``pack_padded_sequence``, the GRU encoders refuse lengths that are zero or not in decreasing order.
"""
from __future__ import annotations

import torch

from . import _lib, synth
from .engine import make_config
from .modules import _EngineModule, _register_tree


def _lengths(lengths, B: int, L: int) -> torch.Tensor:
    """pack_padded_sequence(..., enforce_sorted=True)'s checks on the host copy of the lengths."""
    ln = torch.as_tensor(lengths).reshape(-1).cpu()
    if ln.numel() != B:
        raise ValueError(f"expected {B} lengths, got {ln.numel()}")
    if B and int(ln.min()) <= 0:
        raise RuntimeError("Length of all samples has to be greater than 0")
    if B > 1 and bool((ln[1:] > ln[:-1]).any()):
        raise RuntimeError("`lengths` array must be sorted in decreasing order when `enforce_sorted` is True")
    if B and int(ln.max()) > L:
        raise RuntimeError(f"a length exceeds the padded sequence length {L}")
    return ln


class _T2mModule(_EngineModule):
    _part = 0

    def __init__(self, **dims):
        super().__init__()
        cfg = _lib.default_t2m_config()
        cfg.parts = self._part
        for k, v in dims.items():
            setattr(cfg, k, int(v))
        self._t2m_cfg = cfg
        _register_tree(self, synth.t2m_state_dicts(seed=0, **dims)[self._key])

    def _make_config(self):
        return make_config(num_layers=0, vae="none")            # a handle that holds only this evaluator part

    def _configure_engine(self, eng):
        eng.t2m_configure(self._t2m_cfg)


class B200TextEncoderBiGRUCo(_T2mModule):
    """``TextEncoderBiGRUCo`` (mld/models/architectures/t2m_textenc.py:6-48)."""
    _prefix, _part, _key = "t2m_textencoder.", _lib.T2M_TEXT, "text_encoder"

    def __init__(self, word_size: int, pos_size: int, hidden_size: int, output_size: int):
        super().__init__(dim_word=word_size, dim_pos_ohot=pos_size, dim_text_hidden=hidden_size,
                         dim_coemb_hidden=output_size)
        self.hidden_size = hidden_size

    def forward(self, word_embs: torch.Tensor, pos_onehot: torch.Tensor, cap_lens) -> torch.Tensor:
        _lengths(cap_lens, word_embs.shape[0], word_embs.shape[1])
        return self.engine().t2m_text(word_embs, pos_onehot, cap_lens)


class B200MovementConvEncoder(_T2mModule):
    """``MovementConvEncoder`` (mld/models/architectures/t2m_motionenc.py:6-25)."""
    _prefix, _part, _key = "t2m_moveencoder.", _lib.T2M_MOVEMENT, "movement_encoder"

    def __init__(self, input_size: int, hidden_size: int, output_size: int):
        super().__init__(dim_pose=input_size, dim_move_hidden=hidden_size, dim_move_latent=output_size)

    def forward(self, inputs: torch.Tensor) -> torch.Tensor:
        return self.engine().t2m_movement(inputs)


class B200MotionEncoderBiGRUCo(_T2mModule):
    """``MotionEncoderBiGRUCo`` (mld/models/architectures/t2m_motionenc.py:28-64)."""
    _prefix, _part, _key = "t2m_motionencoder.", _lib.T2M_MOTION, "motion_encoder"

    def __init__(self, input_size: int, hidden_size: int, output_size: int):
        super().__init__(dim_move_latent=input_size, dim_motion_hidden=hidden_size, dim_motion_latent=output_size)
        self.hidden_size = hidden_size

    def forward(self, inputs: torch.Tensor, m_lens) -> torch.Tensor:
        _lengths(m_lens, inputs.shape[0], inputs.shape[1])
        return self.engine().t2m_motion(inputs, m_lens)
