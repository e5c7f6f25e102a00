"""Drop-in replacements for the T2M evaluator's three networks (``MLD._get_t2m_evaluator``,
mld/models/modeltype/mld.py:145-190), whose embeddings feed R-precision, matching score, FID, diversity and
MultiModality:

    t2m_textencoder:   mld_b200.evaluator.B200TextEncoderBiGRUCo   (was t2m_textenc.TextEncoderBiGRUCo)
    t2m_moveencoder:   mld_b200.evaluator.B200MovementConvEncoder  (was t2m_motionenc.MovementConvEncoder)
    t2m_motionencoder: mld_b200.evaluator.B200MotionEncoderBiGRUCo (was t2m_motionenc.MotionEncoderBiGRUCo)

Same ctor kwargs, same ``state_dict`` keys and shapes (``hidden`` included, so finest.tar's dicts load with
``strict=True``), same forward signatures and return shapes; the math runs in ``libmldb200.so``.  Inference only.
Like ``pack_padded_sequence``, the GRU encoders refuse lengths that are zero or not in decreasing order.

And for the HumanAct12 action classifier of ``HUMANACTMetrics`` (mld/models/metrics/gru.py:32-36), whose logits feed
the action model's accuracy and whose features feed its FID, diversity and multimodality:

    gru_classifier:         mld_b200.evaluator.B200MotionDiscriminator        (was humanact12_gru.MotionDiscriminator)
    gru_classifier_for_fid: mld_b200.evaluator.B200MotionDiscriminatorForFID  (was ...MotionDiscriminatorForFID)

And for the UESTC action classifier of ``UESTCMetrics`` (mld/models/metrics/stgcn.py:32), whose yhat feeds the action
model's accuracy and whose pooled features feed its FID, diversity and multimodality:

    stgcn_classifier:       mld_b200.evaluator.B200STGCN                      (was uestc_stgcn.STGCN)
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


class _EvaluatorModule(_EngineModule):
    """An evaluation network: its engine's handle holds only this network."""

    def _make_config(self):
        return make_config(num_layers=0, vae="none")


class _T2mModule(_EvaluatorModule):
    _part = 0

    def __init__(self, **dims):
        super().__init__()
        cfg = _lib.default_t2m_config()
        cfg.parts = self._part
        for k, v in dims.items():
            setattr(cfg, k, int(v))
        self._t2m_cfg = cfg
        _register_tree(self, synth.t2m_state_dicts(seed=0, **dims)[self._key])

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


class B200MotionDiscriminator(_EvaluatorModule):
    """``MotionDiscriminator`` (mld/models/architectures/humanact12_gru.py:6-55): nn.GRU(input_size, hidden_size,
    hidden_layer), the output at ``lengths - 1``, Linear(hidden_size, 30), tanh, Linear(30, output_size).

    ``hidden_unit=None`` draws the initial state exactly as the reference does (``torch.randn(layer, bs, H)`` on the
    CPU default generator, then ``.to(device)``), so a seeded caller draws the same states in the same order.
    Every length must lie in [1, T]: the reference wraps a zero length around to the last frame (``gru_o[-1]``),
    which is not reproduced; such lengths raise before anything runs.  ``use_noise`` is kept and unused, as there."""
    _prefix = "gru_classifier."

    def __init__(self, input_size: int, hidden_size: int, hidden_layer: int, output_size: int = 12, use_noise=None):
        super().__init__()
        self.input_size = input_size
        self.hidden_size = hidden_size
        self.hidden_layer = hidden_layer
        self.use_noise = use_noise
        cfg = _lib.default_a2m_config()
        cfg.input_size, cfg.hidden_size, cfg.hidden_layer, cfg.output_size = input_size, hidden_size, hidden_layer, output_size
        self._a2m_cfg = cfg
        _register_tree(self, synth.a2m_state_dict(seed=0, input_size=input_size, hidden_size=hidden_size,
                                                   hidden_layer=hidden_layer, output_size=output_size))

    def _configure_engine(self, eng):
        eng.a2m_configure(self._a2m_cfg)

    def initHidden(self, num_samples: int, layer: int) -> torch.Tensor:
        return torch.randn(layer, num_samples, self.hidden_size, requires_grad=False)

    def _classify(self, motion_sequence: torch.Tensor, lengths, hidden_unit):
        bs, njoints, nfeats, num_frames = motion_sequence.shape
        if lengths is None:
            raise ValueError("lengths is required (the reference indexes the GRU output with lengths - 1)")
        ln = torch.as_tensor(lengths).reshape(-1)
        if ln.numel() != bs:
            raise ValueError(f"expected {bs} lengths, got {ln.numel()}")
        if ln.dtype.is_floating_point or ln.dtype == torch.bool:
            raise ValueError("lengths must be integers")
        if int(ln.min()) < 1 or int(ln.max()) > num_frames:
            raise ValueError(f"lengths must lie in [1, {num_frames}] (a zero length is not wrapped to the last frame)")
        x = motion_sequence.reshape(bs, njoints * nfeats, num_frames)
        if hidden_unit is None:
            hidden_unit = self.initHidden(bs, self.hidden_layer).to(motion_sequence.device)
        return self.engine().a2m_classify(x, ln, hidden_unit)

    def forward(self, motion_sequence: torch.Tensor, lengths=None, hidden_unit=None) -> torch.Tensor:
        return self._classify(motion_sequence, lengths, hidden_unit)[0]


class B200MotionDiscriminatorForFID(B200MotionDiscriminator):
    """``MotionDiscriminatorForFID`` (humanact12_gru.py:58-85): the 30-d ``tanh(linear1)`` features."""

    def forward(self, motion_sequence: torch.Tensor, lengths=None, hidden_unit=None) -> torch.Tensor:
        return self._classify(motion_sequence, lengths, hidden_unit)[1]


class B200STGCN(_EvaluatorModule):
    """``STGCN`` (mld/models/architectures/uestc_stgcn.py:8-130), the UESTC action classifier of ``UESTCMetrics``
    (mld/models/metrics/stgcn.py:32-40): data_bn, ten st_gcn blocks over the SMPL graph, a global average pool and a
    1 x 1 convolution head.  Same constructor kwargs; ``A`` is built from ``kintree_path`` with the same spatial
    partition, so a fresh module equals the reference before loading.  Same 172 state-dict keys, shapes and dtypes
    (``A``, the running statistics and ``num_batches_tracked`` are buffers), so ``uestc_rot6d_stgcn.tar`` loads with
    ``strict=True``.  ``forward`` returns ``{"output", "features", "yhat"}`` with the reference's squeeze.  Only the
    ``smpl`` layout, the ``spatial`` strategy and edge importance weighting are implemented; anything else raises
    ``ValueError`` at construction, as does a motion of another joint or channel count, or with no frame."""
    _prefix = "stgcn_classifier."
    _BUFFERS = ("A", "running_mean", "running_var", "num_batches_tracked")

    def __init__(self, in_channels, num_class, kintree_path, graph_args, edge_importance_weighting, **kwargs):
        super().__init__()
        ga = dict(graph_args)
        if ga.get("layout", "openpose") != "smpl" or ga.get("strategy", "uniform") != "spatial":
            raise ValueError(f"only graph_args layout='smpl', strategy='spatial' is implemented, got {ga}")
        if ga.get("max_hop", 1) != 1 or ga.get("dilation", 1) != 1:
            raise ValueError(f"only max_hop = dilation = 1 is implemented, got {ga}")
        if not edge_importance_weighting:
            raise ValueError("only edge_importance_weighting=True is implemented")
        from .graph import smpl_adjacency
        A = smpl_adjacency(kintree_path)                 # ValueError unless the table describes SMPL's 24 joints
        self.num_class = num_class
        self.in_channels = in_channels
        cfg = _lib.default_stgcn_config()
        cfg.in_channels, cfg.num_class = in_channels, num_class
        self._stgcn_cfg = cfg
        sd = synth.stgcn_state_dict(seed=0, in_channels=in_channels, num_class=num_class)
        sd["A"] = A
        bn_init = {"running_mean": 0.0, "running_var": 1.0, "num_batches_tracked": 0}
        for k in sd:                                     # as the reference initialises them: unit edge importances,
            if k.startswith("edge_importance."):         # identity BatchNorms
                sd[k] = torch.ones(3, 24, 24)
            elif k.rsplit(".", 1)[-1] in bn_init:
                sd[k] = torch.full_like(sd[k], bn_init[k.rsplit(".", 1)[-1]])
                if "num_batches_tracked" not in k:
                    w = k.rsplit(".", 1)[0]
                    sd[w + ".weight"], sd[w + ".bias"] = torch.ones_like(sd[k]), torch.zeros_like(sd[k])
        _register_tree(self, sd, buffers=self._BUFFERS)

    def _configure_engine(self, eng):
        eng.stgcn_configure(self._stgcn_cfg)

    def forward(self, motion: torch.Tensor):
        if motion.dim() != 4 or motion.shape[1] != 24 or motion.shape[2] != self.in_channels or motion.shape[3] < 1 \
                or motion.shape[0] < 1:
            raise ValueError(f"motion must be [B >= 1, 24, {self.in_channels}, T >= 1], got {tuple(motion.shape)}")
        yhat, features = self.engine().stgcn_classify(motion.contiguous())
        return {"output": motion, "features": features.squeeze(), "yhat": yhat}
