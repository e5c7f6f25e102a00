"""Thin torch-side wrapper over the C ABI: one ``Engine`` == one ``mldb_handle`` on one GPU.

PyTorch is plumbing only here: it owns the device tensors and the current CUDA stream; every
FLOP of the sampling path runs inside ``libmldb200.so``.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from ._lib import MldbConfig, check


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _f32c(t: torch.Tensor, device) -> torch.Tensor:
    return t.to(device=device, dtype=torch.float32).contiguous()


class Engine:
    """Owns an ``mldb_handle``.  ``cfg`` is an :class:`MldbConfig` (see ``make_config``)."""

    def __init__(self, cfg: MldbConfig, device: int | torch.device = 0):
        self._h = None
        self.lib = _lib.lib()
        if not torch.cuda.is_available():
            raise RuntimeError("mld_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        dev = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        self.device = dev
        self.cfg = cfg
        h = C.c_void_p()
        check(self.lib.mldb_create(C.byref(cfg), dev.index or 0, C.byref(h)), "mldb_create")
        self._h = h
        self.timesteps: Optional[torch.Tensor] = None

    def __del__(self):
        try:
            if self._h is not None:
                self.lib.mldb_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], prefix: str = ""):
        """Feed every tensor of a reference state dict (keys get ``prefix``, e.g. 'denoiser.')."""
        for k, v in sd.items():
            t = v.detach().to(dtype=torch.float32).contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            check(self.lib.mldb_load_tensor(self._h, (prefix + k).encode(), _ptr(t), shape, t.dim(),
                                            _lib.DTYPE_F32), f"mldb_load_tensor({prefix + k})")

    def finalize(self):
        check(self.lib.mldb_finalize_weights(self._h, None), "mldb_finalize_weights")

    def set_mean_std(self, mean: torch.Tensor, std: torch.Tensor):
        m = mean.detach().float().contiguous().cpu()
        s = std.detach().float().contiguous().cpu()
        check(self.lib.mldb_set_mean_std(self._h, _ptr(m), _ptr(s), m.numel()), "mldb_set_mean_std")

    def set_option(self, name: str, value: str):
        check(self.lib.mldb_set_option(self._h, name.encode(), value.encode()), "mldb_set_option")

    def profile_op(self, op: str, B: int, S_ctx: int, iters: int = 20) -> float:
        """Average ms of one operator of denoiser layer 0 in isolation (bench.py roofline leg)."""
        ms = C.c_float()
        check(self.lib.mldb_profile_op(self._h, op.encode(), B, S_ctx, iters, C.byref(ms)), "mldb_profile_op")
        return float(ms.value)

    def profile_steps(self, cond: torch.Tensor, init_noise: torch.Tensor):
        """Device time (ms) of every scheduler step of the reverse loop, launched eagerly (mldb_profile_steps)."""
        c, z0 = self._cond(cond), _f32c(init_noise, self.device)
        B = z0.shape[0]
        self._check_latent(z0, B, "init_noise")
        self._check_cond(c, 2 * B if self.cfg_on else B)
        S = c.shape[1] if c.dim() == 3 else 1
        n = 0 if self.timesteps is None else len(self.timesteps)
        ms = (C.c_float * n)()
        check(self.lib.mldb_profile_steps(self._h, _ptr(c), _ptr(z0), B, S, ms), "mldb_profile_steps")
        return [float(v) for v in ms]

    def debug_gemm(self, A, W, bias=None, gamma=None, beta=None, R=None, K1=0, act=0, use_tc=True, split_out=False,
                   in_place=False):
        """Kernel unit-test hook (mldb_debug_gemm): A [M,K] (device), W [N,K] / bias / gamma / beta (host).
        ``R`` without ``gamma``: the residual-add epilogue A W^T + b + R; ``in_place`` runs it with out == R."""
        A = _f32c(A, self.device)
        Wc = W.detach().float().contiguous().cpu()
        host = [None if t is None else t.detach().float().contiguous().cpu() for t in (bias, gamma, beta)]
        Rd = None if R is None else _f32c(R, self.device)
        M, K = A.shape
        N = Wc.shape[0]
        out = torch.empty((M, N), dtype=torch.float32, device=self.device)
        if in_place:
            if Rd is None or gamma is not None:
                raise ValueError("in_place needs R and no gamma (the residual-add epilogue)")
            out = Rd = Rd.clone()
        check(self.lib.mldb_debug_gemm(self._h, _ptr(A), _ptr(Wc), _ptr(host[0]), _ptr(host[1]), _ptr(host[2]),
                                       _ptr(Rd), M, N, K, K1, act, int(use_tc), int(split_out), _ptr(out), self._stream()),
              "mldb_debug_gemm")
        return out

    def debug_ffn(self, X, W1, b1, W2, b2, gamma, beta, mode=2):
        """Kernel unit-test hook (mldb_debug_ffn): LayerNorm(X + W2 gelu(W1 X + b1) + b2); mode 0 CUDA-core,
        1 wgmma GEMMs (two launches), 2 fused wgmma FFN kernel.  X [M,d] (device), the rest host."""
        X = _f32c(X, self.device)
        host = [t.detach().float().contiguous().cpu() for t in (W1, b1, W2, b2, gamma, beta)]
        M, d = X.shape
        ff = host[0].shape[0]
        out = torch.empty((M, d), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_debug_ffn(self._h, _ptr(X), *[_ptr(t) for t in host], M, d, ff, int(mode), _ptr(out),
                                      self._stream()), "mldb_debug_ffn")
        return out

    def debug_tail(self, att, X, Wo, bo, g1, be1, W1, b1, W2, b2, g2, be2, mode=2, pad=None):
        """Kernel unit-test hook (mldb_debug_tail): x1 = LayerNorm1(att Wo^T + bo + X), then
        LayerNorm2(x1 + W2 gelu(W1 x1 + b1) + b2); mode 0 CUDA-core, 1 the two wgmma kernels (out-projection + LN
        GEMM, fused FFN), 2 one fused launch.  att, X [M,d] (device), the rest host; biases may be None.
        pad: optional [P, d] rows placed in the output buffer past row M before the op; the result is then
        [M + P, d], its last P rows read back from that buffer after the op."""
        att, X = _f32c(att, self.device), _f32c(X, self.device)
        host = [None if t is None else t.detach().float().contiguous().cpu()
                for t in (Wo, bo, g1, be1, W1, b1, W2, b2, g2, be2)]
        M, d = X.shape
        ff = host[4].shape[0]
        out = torch.empty((M, d), dtype=torch.float32, device=self.device)
        if pad is not None:
            out = torch.cat([out, _f32c(pad, self.device)]).contiguous()
        check(self.lib.mldb_debug_tail(self._h, _ptr(att), _ptr(X), *[_ptr(t) for t in host], M, d, ff, int(mode),
                                       out.shape[0], _ptr(out), self._stream()), "mldb_debug_tail")
        return out

    def debug_attention(self, q, nseq, Lq, heads, lengths=None, mode=2, kv=None, Lk=None, kv_prefix=0,
                        causal=False):
        """Kernel unit-test hook (mldb_debug_attention).  ``kv is None``: ``q`` is a packed qkv
        [nseq*Lq, 3*heads*hd] tensor (self-attention, the layout the stacks use); else ``q`` [nseq*Lq, d] and
        ``kv`` [nseq*Lk, 2*d] (cross-attention).  mode 0 CUDA-core, 1 mma.sync, 2 wgmma (product).
        ``causal``: query i attends to keys j <= i (mldb_debug_attention_causal; self-attention only).
        Returns [nseq*Lq, heads*hd]."""
        q = _f32c(q, self.device)
        kvd = None if kv is None else _f32c(kv, self.device)
        d = q.shape[1] // 3 if kv is None else q.shape[1]
        Lk = Lq if Lk is None else Lk
        if q.shape[0] != nseq * Lq or (kvd is not None and tuple(kvd.shape) != (nseq * Lk, 2 * d)):
            raise ValueError("debug_attention: shape mismatch")
        ln = None if lengths is None else torch.as_tensor(lengths, dtype=torch.int32, device=self.device).contiguous()
        out = torch.empty((nseq * Lq, d), dtype=torch.float32, device=self.device)
        fn = self.lib.mldb_debug_attention_causal if causal else self.lib.mldb_debug_attention
        check(fn(self._h, _ptr(q), _ptr(kvd), _ptr(ln), int(kv_prefix), nseq, Lq, Lk, heads, d // heads, int(mode),
                 _ptr(out), self._stream()), "mldb_debug_attention")
        return out

    # ------------------------------------------------------------------ CLIP text tower
    def text_configure(self, tcfg):
        """Add the text tower's keys (``text_encoder.`` prefix) to the strict key spec; before :meth:`finalize`."""
        check(self.lib.mldb_text_configure(self._h, C.byref(tcfg)), "mldb_text_configure")
        self.text_cfg = tcfg

    def text_encode(self, ids: torch.Tensor, mode: int = _lib.TEXT_POOLED) -> torch.Tensor:
        """int64 token ids [n, L] -> last_hidden_state [n, L, hidden] (TEXT_HIDDEN) or get_text_features [n, proj]
        (TEXT_POOLED), on the current stream.  Ids outside the vocabulary are rejected here, before the launch."""
        tc = self._configured("text_cfg", "text_configure() was not called before finalize()")
        if ids.dim() != 2 or ids.shape[0] < 1 or not 1 <= ids.shape[1] <= tc.max_positions:
            raise ValueError(f"ids must be [n, L] with 1 <= L <= {tc.max_positions}, got {tuple(ids.shape)}")
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= tc.vocab_size):
            raise ValueError(f"token ids must lie in [0, {tc.vocab_size})")
        d_ids = ids.to(device=self.device, dtype=torch.int64).contiguous()
        n, L = d_ids.shape
        shape = (n, L, tc.hidden) if mode == _lib.TEXT_HIDDEN else (n, tc.projection_dim)
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        check(self.lib.mldb_text_encode(self._h, _ptr(d_ids), n, L, int(mode), _ptr(out), self._stream()),
              "mldb_text_encode")
        return out

    # ------------------------------------------------------------------ BERT text tower
    def bert_configure(self, bcfg):
        """Add the BERT tower's keys (``text_encoder.`` prefix) to the strict key spec; before :meth:`finalize`."""
        check(self.lib.mldb_bert_configure(self._h, C.byref(bcfg)), "mldb_bert_configure")
        self.bert_cfg = bcfg

    def bert_encode(self, ids: torch.Tensor, lengths) -> torch.Tensor:
        """int64 token ids [n, L] + real tokens per row (each in [1, L], the right-padded attention mask) ->
        last_hidden_state [n, L, hidden], every position, on the current stream.  Bad ids are rejected here."""
        bc = self._configured("bert_cfg", "bert_configure() was not called before finalize()")
        if ids.dim() != 2 or ids.shape[0] < 1 or not 1 <= ids.shape[1] <= bc.max_positions:
            raise ValueError(f"ids must be [n, L] with 1 <= L <= {bc.max_positions}, got {tuple(ids.shape)}")
        if int(ids.min()) < 0 or int(ids.max()) >= bc.vocab_size:
            raise ValueError(f"token ids must lie in [0, {bc.vocab_size})")
        d_ids = ids.to(device=self.device, dtype=torch.int64).contiguous()
        n, L = d_ids.shape
        ln = self._seq_lengths(lengths, n, L)
        out = torch.empty((n, L, bc.hidden), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_bert_encode(self._h, _ptr(d_ids), _ptr(ln), n, L, _ptr(out), self._stream()),
              "mldb_bert_encode")
        return out

    # ------------------------------------------------------------------ T2M evaluator
    def t2m_configure(self, tcfg):
        """Add the evaluator parts' keys (``t2m_textencoder.`` / ``t2m_moveencoder.`` / ``t2m_motionencoder.``) to the
        strict key spec; before :meth:`finalize`."""
        check(self.lib.mldb_t2m_configure(self._h, C.byref(tcfg)), "mldb_t2m_configure")
        self.t2m_cfg = tcfg

    def _t2m(self, part: int, name: str):
        msg = f"the T2M {name} encoder was not configured (t2m_configure) before finalize()"
        tc = self._configured("t2m_cfg", msg)
        if not tc.parts & part:
            raise RuntimeError(msg)
        return tc

    def _configured(self, attr: str, msg: str):
        """The config that ``*_configure`` stored as ``attr``; RuntimeError(msg) if it was not called."""
        cfg = getattr(self, attr, None)
        if cfg is None:
            raise RuntimeError(msg)
        return cfg

    def _seq_lengths(self, lengths, B: int, L: int) -> torch.Tensor:
        """B integer sequence lengths, each in [1, L], as a contiguous int32 tensor on the device."""
        ln = torch.as_tensor(lengths).reshape(-1)
        if ln.numel() != B:
            raise ValueError(f"lengths must hold {B} values, got {ln.numel()}")
        if ln.dtype.is_floating_point or ln.dtype == torch.bool:
            raise ValueError("lengths must be integers")
        if B and (int(ln.min()) < 1 or int(ln.max()) > L):
            raise ValueError(f"lengths must lie in [1, {L}]")
        return ln.to(device=self.device, dtype=torch.int32).contiguous()

    def t2m_movement(self, x: torch.Tensor) -> torch.Tensor:
        """MovementConvEncoder: [B, T, dim_pose] (T >= 4; the last dimension may be a strided slice such as
        ``feats[..., :-4]``) -> [B, T // 2 // 2, dim_move_latent]."""
        tc = self._t2m(_lib.T2M_MOVEMENT, "movement")
        if x.dim() != 3 or x.shape[2] != tc.dim_pose or x.shape[0] < 1 or x.shape[1] < 4:
            raise ValueError(f"x must be [B >= 1, T >= 4, {tc.dim_pose}], got {tuple(x.shape)}")
        x = x.to(device=self.device, dtype=torch.float32)
        if x.stride(2) != 1 or x.stride(0) != x.shape[1] * x.stride(1):
            x = x.contiguous()
        B, T = x.shape[:2]
        out = torch.empty((B, T // 2 // 2, tc.dim_move_latent), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_t2m_movement(self._h, _ptr(x), x.stride(1), B, T, _ptr(out), self._stream()),
              "mldb_t2m_movement")
        return out

    def t2m_motion(self, x: torch.Tensor, lengths) -> torch.Tensor:
        """MotionEncoderBiGRUCo: [B, L, dim_move_latent] + lengths (any order, each in [1, L]) -> [B, dim_motion_latent]."""
        tc = self._t2m(_lib.T2M_MOTION, "motion")
        if x.dim() != 3 or x.shape[2] != tc.dim_move_latent or x.shape[0] < 1 or x.shape[1] < 1:
            raise ValueError(f"x must be [B >= 1, L >= 1, {tc.dim_move_latent}], got {tuple(x.shape)}")
        xd = _f32c(x, self.device)
        B, L = xd.shape[:2]
        ln = self._seq_lengths(lengths, B, L)
        out = torch.empty((B, tc.dim_motion_latent), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_t2m_motion(self._h, _ptr(xd), _ptr(ln), B, L, _ptr(out), self._stream()), "mldb_t2m_motion")
        return out

    def t2m_text(self, word_embs: torch.Tensor, pos_ohot: torch.Tensor, lengths) -> torch.Tensor:
        """TextEncoderBiGRUCo: word_embs [B, L, dim_word], pos_ohot [B, L, dim_pos_ohot] + lengths (any order, each
        in [1, L]) -> [B, dim_coemb_hidden]."""
        tc = self._t2m(_lib.T2M_TEXT, "text")
        if word_embs.dim() != 3 or word_embs.shape[2] != tc.dim_word or word_embs.shape[0] < 1 or word_embs.shape[1] < 1:
            raise ValueError(f"word_embs must be [B >= 1, L >= 1, {tc.dim_word}], got {tuple(word_embs.shape)}")
        if tuple(pos_ohot.shape) != (*word_embs.shape[:2], tc.dim_pos_ohot):
            raise ValueError(f"pos_ohot must be [{word_embs.shape[0]}, {word_embs.shape[1]}, {tc.dim_pos_ohot}], "
                             f"got {tuple(pos_ohot.shape)}")
        w, p = _f32c(word_embs, self.device), _f32c(pos_ohot, self.device)
        B, L = w.shape[:2]
        ln = self._seq_lengths(lengths, B, L)
        out = torch.empty((B, tc.dim_coemb_hidden), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_t2m_text(self._h, _ptr(w), _ptr(p), _ptr(ln), B, L, _ptr(out), self._stream()),
              "mldb_t2m_text")
        return out

    # ------------------------------------------------------------------ HumanAct12 action classifier
    def a2m_configure(self, acfg):
        """Add the classifier's keys (``gru_classifier.`` prefix) to the strict key spec; before :meth:`finalize`."""
        check(self.lib.mldb_a2m_configure(self._h, C.byref(acfg)), "mldb_a2m_configure")
        self.a2m_cfg = acfg

    def a2m_classify(self, x: torch.Tensor, lengths, h0: torch.Tensor):
        """MotionDiscriminator with an explicit initial state: x [B, input_size, T] (or [B, njoints, nfeats, T]),
        lengths (each in [1, T]), h0 [hidden_layer, B, hidden_size] -> (logits [B, output_size], features [B, 30])."""
        ac = self._configured("a2m_cfg", "the action classifier was not configured (a2m_configure) before finalize()")
        if x.dim() == 4:
            x = x.reshape(x.shape[0], x.shape[1] * x.shape[2], x.shape[3])
        if x.dim() != 3 or x.shape[1] != ac.input_size or x.shape[0] < 1 or x.shape[2] < 1:
            raise ValueError(f"x must be [B >= 1, {ac.input_size}, T >= 1], got {tuple(x.shape)}")
        xd = _f32c(x, self.device)
        B, T = xd.shape[0], xd.shape[2]
        if tuple(h0.shape) != (ac.hidden_layer, B, ac.hidden_size):
            raise ValueError(f"h0 must be [{ac.hidden_layer}, {B}, {ac.hidden_size}], got {tuple(h0.shape)}")
        ln = self._seq_lengths(lengths, B, T)
        hd = _f32c(h0, self.device)
        logits = torch.empty((B, ac.output_size), dtype=torch.float32, device=self.device)
        feats = torch.empty((B, 30), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_a2m_classify(self._h, _ptr(xd), _ptr(ln), _ptr(hd), B, T, _ptr(logits), _ptr(feats),
                                         self._stream()), "mldb_a2m_classify")
        return logits, feats

    # ------------------------------------------------------------------ UESTC action classifier
    def stgcn_configure(self, scfg):
        """Add the classifier's keys (``stgcn_classifier.`` prefix) to the strict key spec; before :meth:`finalize`."""
        check(self.lib.mldb_stgcn_configure(self._h, C.byref(scfg)), "mldb_stgcn_configure")
        self.stgcn_cfg = scfg

    def stgcn_classify(self, motion: torch.Tensor):
        """STGCN: motion [B, 24, in_channels, T] -> (yhat [B, num_class], features [B, 256])."""
        sc = self._configured("stgcn_cfg", "the UESTC classifier was not configured (stgcn_configure) before finalize()")
        if motion.dim() != 4 or motion.shape[0] < 1 or motion.shape[1] != 24 or motion.shape[2] != sc.in_channels \
                or motion.shape[3] < 1:
            raise ValueError(f"motion must be [B >= 1, 24, {sc.in_channels}, T >= 1], got {tuple(motion.shape)}")
        xd = _f32c(motion, self.device)
        B, T = xd.shape[0], xd.shape[3]
        yhat = torch.empty((B, sc.num_class), dtype=torch.float32, device=self.device)
        feats = torch.empty((B, 256), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_stgcn_classify(self._h, _ptr(xd), B, T, _ptr(yhat), _ptr(feats), self._stream()),
              "mldb_stgcn_classify")
        return yhat, feats

    # ------------------------------------------------------------------ SMPL layer
    def smpl_configure(self, scfg):
        """Add the SMPL model's keys (``smpl.`` prefix) to the strict key spec; before :meth:`finalize`."""
        check(self.lib.mldb_smpl_configure(self._h, C.byref(scfg)), "mldb_smpl_configure")
        self.smpl_cfg = scfg

    def smpl_forward(self, feats: torch.Tensor, mask: Optional[torch.Tensor], jointstype: int,
                     vertstrans: bool) -> torch.Tensor:
        """Rotation2xyz on rot6d features [B, T, 150] (MLD's layout before its view / permute) with an optional
        bool mask [B, T] -> [B, 24, 3, T] (SMPL_JOINTS) or [B, V, 3, T] (SMPL_VERTICES), float32."""
        sc = self._configured("smpl_cfg", "the SMPL layer was not configured (smpl_configure) before finalize()")
        if feats.dim() != 3 or feats.shape[0] < 1 or feats.shape[1] < 1 or feats.shape[2] != 150:
            raise ValueError(f"feats must be [B >= 1, T >= 1, 150], got {tuple(feats.shape)}")
        if jointstype not in (_lib.SMPL_JOINTS, _lib.SMPL_VERTICES):
            raise ValueError(f"jointstype must be SMPL_JOINTS or SMPL_VERTICES, got {jointstype}")
        f = _f32c(feats, self.device)
        B, T = f.shape[:2]
        md = None
        if mask is not None:
            if tuple(mask.shape) != (B, T):
                raise ValueError(f"mask must be [{B}, {T}], got {tuple(mask.shape)}")
            md = mask.to(device=self.device, dtype=torch.uint8).contiguous()
        n = 24 if jointstype == _lib.SMPL_JOINTS else sc.num_vertices
        out = torch.empty((B, n, 3, T), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_smpl_forward(self._h, _ptr(f), _ptr(md), B, T, int(jointstype), int(bool(vertstrans)),
                                         _ptr(out), self._stream()), "mldb_smpl_forward")
        return out

    # ------------------------------------------------------------------ APE / AVE metric
    def ape_ave(self, jts_text: torch.Tensor, jts_ref: torch.Tensor, lengths: torch.Tensor, jointstype: int,
                force_in_meter: bool) -> torch.Tensor:
        """ComputeMetrics.update's increments of joints [B, T, J, 3] (contiguous float32 on this device) with device
        int32 lengths [B], each in [2, T] -> float32 [4 J + 2] in ComputeMetrics.metrics order (mldb_ape_ave)."""
        if jts_text.dim() != 4 or jts_text.shape[-1] != 3 or jts_text.shape != jts_ref.shape:
            raise ValueError(f"joints must be two [B, T, J, 3] tensors, got {tuple(jts_text.shape)} and "
                             f"{tuple(jts_ref.shape)}")
        for t in (jts_text, jts_ref):
            if t.dtype != torch.float32 or t.device != self.device or not t.is_contiguous():
                raise ValueError("joints must be contiguous float32 tensors on the engine's device")
        B, T, J = jts_text.shape[:3]
        if lengths.dtype != torch.int32 or lengths.device != self.device or tuple(lengths.shape) != (B,):
            raise ValueError(f"lengths must be int32 [{B}] on the engine's device")
        out = torch.empty(4 * J + 2, dtype=torch.float32, device=self.device)
        check(self.lib.mldb_ape_ave(self._h, _ptr(jts_text), _ptr(jts_ref), _ptr(lengths.contiguous()), B, T, J,
                                    int(jointstype), int(bool(force_in_meter)), _ptr(out), self._stream()),
              "mldb_ape_ave")
        return out

    def kernel_stats(self, reset: bool = False) -> Dict[str, int]:
        """Which kernel each operator was enqueued on since the last reset (mldb_kernel_stats)."""
        arr = (C.c_int64 * len(_lib.KSTAT_NAMES))()
        check(self.lib.mldb_kernel_stats(self._h, arr, len(_lib.KSTAT_NAMES)), "mldb_kernel_stats")
        if reset:
            check(self.lib.mldb_reset_kernel_stats(self._h), "mldb_reset_kernel_stats")
        return {k: int(v) for k, v in zip(_lib.KSTAT_NAMES, arr)}

    @property
    def launch_count(self) -> int:
        return int(self.lib.mldb_launch_count(self._h))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # ------------------------------------------------------------------ scheduler
    def set_timesteps(self, n: int) -> torch.Tensor:
        ts = torch.empty(n, dtype=torch.int64)
        check(self.lib.mldb_scheduler_set_timesteps(self._h, n, _ptr(ts)), "mldb_scheduler_set_timesteps")
        self.timesteps = ts
        return ts

    def scheduler_step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor,
                       noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        mo, sa = _f32c(model_output, self.device), _f32c(sample, self.device)
        nz = None if noise is None else _f32c(noise, self.device)
        out = torch.empty_like(sa)
        check(self.lib.mldb_scheduler_step(self._h, _ptr(mo), int(timestep), _ptr(sa), _ptr(nz),
                                           sa.numel(), _ptr(out), self._stream()), "mldb_scheduler_step")
        return out

    # ------------------------------------------------------------------ argument checks
    # The C ABI takes raw pointers: a wrong shape would be a silent out-of-bounds access on the device.
    @property
    def cfg_on(self) -> bool:
        return self.cfg.guidance_scale > 1.0

    def _check_cond(self, c: torch.Tensor, Bx: int):
        if self.cfg.cond_kind == _lib.COND_TEXT:
            if c.dim() != 3 or c.shape[0] != Bx or c.shape[2] != self.cfg.text_dim or c.shape[1] < 1:
                raise ValueError(f"condition must be [{Bx}, S, {self.cfg.text_dim}] (uncond half first when guidance "
                                 f"is on), got {tuple(c.shape)}")
        elif c.numel() != Bx:
            raise ValueError(f"action condition must hold {Bx} class ids ([{Bx}, 1]), got {tuple(c.shape)}")

    def _check_latent(self, x: torch.Tensor, rows: int, what: str):
        cfg = self.cfg
        want = (rows, x.shape[1], cfg.nfeats) if cfg.diffusion_only else (rows, cfg.n_lat, cfg.latent_dim)
        if x.dim() != 3 or tuple(x.shape) != want:
            raise ValueError(f"{what} must be {list(want)}, got {tuple(x.shape)}")

    def _check_lengths(self, ln: Optional[torch.Tensor], B: int, T: Optional[int] = None):
        if ln is None:
            return
        if ln.numel() != B:
            raise ValueError(f"lengths must have {B} entries, got {ln.numel()}")
        if T is not None and not isinstance(T, bool):
            host = ln if ln.device.type == "cpu" else None
            if host is not None and (int(host.max()) > T or int(host.min()) < 1):
                raise ValueError(f"lengths must lie in [1, {T}]")

    @property
    def stochastic(self) -> bool:
        """True when the scheduler adds noise at its steps (DDPM, or DDIM with eta > 0): the sampling calls
        then need ``step_noise`` [n_steps, B, ...] of N(0,1) draws."""
        return self.cfg.sched_kind == _lib.SCHED_DDPM or self.cfg.eta > 0.0

    def _step_noise(self, step_noise: Optional[torch.Tensor], latent_shape, device=None) -> Optional[torch.Tensor]:
        """``step_noise`` as a contiguous fp32 tensor on ``device`` (default: the engine's), shape-checked
        against [n_steps, *latent_shape]."""
        if step_noise is None:
            return None
        sn = step_noise.to(device=self.device if device is None else device, dtype=torch.float32).contiguous()
        n_steps = 0 if self.timesteps is None else len(self.timesteps)
        if tuple(sn.shape) != (n_steps, *latent_shape):
            raise ValueError(f"step_noise must be [{n_steps}, {', '.join(map(str, latent_shape))}], got {tuple(sn.shape)}")
        return sn

    # ------------------------------------------------------------------ denoiser
    def _cond(self, cond: torch.Tensor) -> torch.Tensor:
        if self.cfg.cond_kind == _lib.COND_TEXT:
            return _f32c(cond, self.device)
        return cond.to(device=self.device, dtype=torch.int64).contiguous()

    def _lengths(self, lengths) -> Optional[torch.Tensor]:
        if lengths is None:
            return None
        if isinstance(lengths, torch.Tensor):
            return lengths.to(device=self.device, dtype=torch.int32).contiguous()
        return torch.tensor(list(lengths), dtype=torch.int32, device=self.device)

    def denoise(self, sample: torch.Tensor, timestep: int, cond: torch.Tensor,
                lengths=None) -> torch.Tensor:
        x, c = _f32c(sample, self.device), self._cond(cond)
        ln = self._lengths(lengths)
        Bx = x.shape[0]
        self._check_latent(x, Bx, "sample")
        self._check_cond(c, Bx)
        self._check_lengths(ln, Bx)
        S = c.shape[1] if c.dim() == 3 else 1
        T = x.shape[1] if self.cfg.diffusion_only else 0
        out = torch.empty_like(x)
        check(self.lib.mldb_denoise(self._h, _ptr(x), int(timestep), _ptr(c), _ptr(ln), Bx, S, T,
                                    _ptr(out), self._stream()), "mldb_denoise")
        return out

    def diffusion_reverse(self, cond: torch.Tensor, init_noise: torch.Tensor, lengths=None,
                          step_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        c, z0 = self._cond(cond), _f32c(init_noise, self.device)
        ln = self._lengths(lengths)
        B = z0.shape[0]
        self._check_latent(z0, B, "init_noise")
        self._check_cond(c, 2 * B if self.cfg_on else B)
        self._check_lengths(ln, B)
        S = c.shape[1] if c.dim() == 3 else 1
        T = z0.shape[1] if self.cfg.diffusion_only else 0
        out = torch.empty((z0.shape[1], B, z0.shape[2]), dtype=torch.float32, device=self.device)
        sn = self._step_noise(step_noise, z0.shape)
        check(self.lib.mldb_diffusion_reverse(self._h, _ptr(c), _ptr(z0), _ptr(sn), _ptr(ln), B, S, T,
                                              _ptr(out), self._stream()), "mldb_diffusion_reverse")
        return out

    # ------------------------------------------------------------------ VAE / joints
    def vae_decode(self, z: torch.Tensor, lengths) -> torch.Tensor:
        zz = _f32c(z, self.device)
        ln = self._lengths(lengths)
        if zz.dim() != 3 or zz.shape[0] != self.cfg.n_lat or zz.shape[2] != self.cfg.latent_dim:
            raise ValueError(f"z must be [{self.cfg.n_lat}, B, {self.cfg.latent_dim}], got {tuple(zz.shape)}")
        B = zz.shape[1]
        self._check_lengths(ln, B)
        T = int(max(lengths)) if not isinstance(lengths, torch.Tensor) else int(lengths.max())
        out = torch.empty((B, T, self.cfg.vae_nfeats), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_vae_decode(self._h, _ptr(zz), _ptr(ln), B, T, _ptr(out), self._stream()),
              "mldb_vae_decode")
        return out

    def vae_encode(self, feats: torch.Tensor, lengths):
        """feats [B, T, vae_nfeats] -> (mu, logvar), each [n_lat, B, d] (MldVae) or [1, B, d] (ActorVae)."""
        f = _f32c(feats, self.device)
        ln = self._lengths(lengths)
        if f.dim() != 3 or f.shape[2] != self.cfg.vae_nfeats:
            raise ValueError(f"feats must be [B, T, {self.cfg.vae_nfeats}], got {tuple(f.shape)}")
        B, T = f.shape[0], f.shape[1]
        self._check_lengths(ln, B)
        n_tok = 1 if self.cfg.vae_kind == _lib.VAE_ACTOR else self.cfg.n_lat
        shape = (n_tok, B, self.cfg.latent_dim)
        mu = torch.empty(shape, dtype=torch.float32, device=self.device)
        logvar = torch.empty(shape, dtype=torch.float32, device=self.device)
        check(self.lib.mldb_vae_encode(self._h, _ptr(f), _ptr(ln), B, T, _ptr(mu), _ptr(logvar),
                                       self._stream()), "mldb_vae_encode")
        return mu, logvar

    def feats2joints(self, feats: torch.Tensor) -> torch.Tensor:
        f = _f32c(feats, self.device)
        F = self.cfg.vae_nfeats if self.cfg.vae_kind != _lib.VAE_NONE else self.cfg.nfeats
        if f.dim() != 3 or f.shape[2] != F:
            raise ValueError(f"feats must be [B, T, {F}], got {tuple(f.shape)}")
        B, T = f.shape[0], f.shape[1]
        out = torch.empty((B, T, self.cfg.njoints, 3), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_feats2joints(self._h, _ptr(f), B, T, _ptr(out), self._stream()),
              "mldb_feats2joints")
        return out

    # ------------------------------------------------------------------ fused sample
    def sample(self, cond: torch.Tensor, init_noise: torch.Tensor, lengths, want=("joints",), *,
               step_noise: Optional[torch.Tensor] = None):
        """reverse diffusion -> decode -> feats2joints on device tensors.  Returns a dict with the
        requested subset of {"latents" [n_lat,B,d], "feats" [B,T,F], "joints" [B,T,J,3]}.
        ``step_noise`` [n_steps, B, n_lat, d]: the N(0,1) draws of the scheduler steps, required when
        :attr:`stochastic` (as for :meth:`diffusion_reverse`)."""
        c, z0 = self._cond(cond), _f32c(init_noise, self.device)
        sn = self._step_noise(step_noise, z0.shape)
        ln = self._lengths(lengths)
        B = z0.shape[0]
        self._check_latent(z0, B, "init_noise")
        self._check_cond(c, 2 * B if self.cfg_on else B)
        self._check_lengths(ln, B)
        S = c.shape[1] if c.dim() == 3 else 1
        T = int(max(lengths)) if not isinstance(lengths, torch.Tensor) else int(lengths.max())
        if T < 1 or int(min(lengths)) < 1:
            raise ValueError("lengths must be >= 1")
        cfg = self.cfg
        out = {}
        lat = fe = jo = None
        if "latents" in want:
            lat = out["latents"] = torch.empty((cfg.n_lat, B, cfg.latent_dim), dtype=torch.float32, device=self.device)
        if "feats" in want:
            fe = out["feats"] = torch.empty((B, T, cfg.vae_nfeats), dtype=torch.float32, device=self.device)
        if "joints" in want:
            jo = out["joints"] = torch.empty((B, T, cfg.njoints, 3), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_sample(self._h, _ptr(c), _ptr(z0), _ptr(ln), B, S, T, _ptr(lat), _ptr(fe),
                                   _ptr(jo), self._stream(), _ptr(sn)), "mldb_sample")
        return out

    # ------------------------------------------------------------------ multi-GPU (one process per GPU)
    def comm_init(self, group=None):
        """Build the handle's NCCL communicator over the ranks of ``group`` (default: the world): rank 0 of
        the group draws the unique id inside the library, torch.distributed only ships its 128 bytes."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        uid = (C.c_ubyte * 128)()
        if rank == 0:
            check(self.lib.mldb_comm_unique_id(uid), "mldb_comm_unique_id")
        box = [bytes(uid)]
        dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        buf = (C.c_ubyte * 128).from_buffer_copy(box[0])
        check(self.lib.mldb_comm_init(self._h, buf, world, rank), "mldb_comm_init")
        return world, rank

    def comm_info(self):
        n, r = C.c_int32(), C.c_int32()
        check(self.lib.mldb_comm_info(self._h, C.byref(n), C.byref(r)), "mldb_comm_info")
        return int(n.value), int(r.value)

    def allgather(self, local: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """ncclAllGather through the C ABI on the current stream: [n, ...] per rank -> [world * n, ...]."""
        world, _ = self.comm_info()
        x = _f32c(local, self.device)
        if out is None:
            out = torch.empty((world * x.shape[0], *x.shape[1:]), dtype=torch.float32, device=self.device)
        check(self.lib.mldb_allgather(self._h, _ptr(x), _ptr(out), x.numel(), self._stream()), "mldb_allgather")
        return out

    def sample_gather(self, cond: torch.Tensor, init_noise: torch.Tensor, lengths, T: Optional[int] = None,
                      out: Optional[torch.Tensor] = None, wait: bool = True, *,
                      step_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """This rank's shard through ``mldb_sample_gather``: joints of ALL ranks ``[world * B, T, J, 3]``.
        ``T`` must be the same on every rank (pad to the global max length).  ``wait=False`` leaves the gather
        running on the side stream (call :meth:`gather_wait` before reading ``out``; alternate two ``out``
        buffers between consecutive calls).  ``step_noise`` is this rank's shard [n_steps, B, n_lat, d]."""
        c, z0 = self._cond(cond), _f32c(init_noise, self.device)
        sn = self._step_noise(step_noise, z0.shape)
        ln = self._lengths(lengths)
        B = z0.shape[0]
        self._check_latent(z0, B, "init_noise")
        self._check_cond(c, 2 * B if self.cfg_on else B)
        self._check_lengths(ln, B)
        S = c.shape[1] if c.dim() == 3 else 1
        if T is None:
            T = int(max(lengths)) if not isinstance(lengths, torch.Tensor) else int(lengths.max())
        world, _ = self.comm_info()
        shape = (world * B, T, self.cfg.njoints, 3)
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=self.device)
        elif tuple(out.shape) != shape or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous float32 {list(shape)} tensor")
        check(self.lib.mldb_sample_gather(self._h, _ptr(c), _ptr(z0), _ptr(ln), B, S, T, _ptr(out), self._stream(),
                                          _ptr(sn)), "mldb_sample_gather")
        if wait:
            self.gather_wait()
        return out

    def gather_wait(self):
        check(self.lib.mldb_gather_wait(self._h, self._stream()), "mldb_gather_wait")

    def sample_host(self, cond_cpu: torch.Tensor, noise_cpu: torch.Tensor, lengths_cpu: torch.Tensor,
                    joints_cpu: torch.Tensor, T: int, *, step_noise: Optional[torch.Tensor] = None):
        """End-to-end through HOST buffers (pinned recommended); asynchronous on the current
        stream - synchronise before reading ``joints_cpu``.  ``step_noise``: contiguous f32 HOST tensor
        [n_steps, B, n_lat, d], as for :meth:`sample`."""
        B = noise_cpu.shape[0]
        if step_noise is not None and (step_noise.device.type != "cpu" or step_noise.dtype != torch.float32
                                       or not step_noise.is_contiguous()):
            raise ValueError("sample_host takes step_noise as a contiguous f32 HOST tensor")
        sn = self._step_noise(step_noise, noise_cpu.shape, device="cpu")
        S = cond_cpu.shape[1] if cond_cpu.dim() == 3 else 1
        for t, dt in ((cond_cpu, torch.float32 if self.cfg.cond_kind == _lib.COND_TEXT else torch.int64),
                      (noise_cpu, torch.float32), (lengths_cpu, torch.int32), (joints_cpu, torch.float32)):
            if t.device.type != "cpu" or t.dtype != dt or not t.is_contiguous():
                raise ValueError("sample_host takes contiguous HOST tensors (cond f32/int64, noise f32, lengths int32, joints f32)")
        self._check_latent(noise_cpu, B, "init_noise")
        self._check_cond(cond_cpu, 2 * B if self.cfg_on else B)
        self._check_lengths(lengths_cpu, B, T)
        world, _ = self.comm_info()
        if joints_cpu.numel() != world * B * T * self.cfg.njoints * 3:
            raise ValueError(f"joints buffer must hold [{world * B}, {T}, {self.cfg.njoints}, 3] floats")
        check(self.lib.mldb_sample_host(self._h, _ptr(cond_cpu), _ptr(noise_cpu), _ptr(lengths_cpu), B, S, T,
                                        _ptr(joints_cpu), self._stream(), _ptr(sn)), "mldb_sample_host")
        return joints_cpu


def make_config(*, condition: str = "text", arch: str = "trans_enc", latent_dim: Sequence[int] = (1, 256),
                ff_size: int = 1024, num_layers: int = 9, num_heads: int = 4, text_encoded_dim: int = 768,
                nclasses: int = 12, nfeats: int = 263, diffusion_only: bool = False,
                flip_sin_to_cos: bool = True, freq_shift: float = 0.0, guidance_scale: float = 7.5,
                vae: str = "mld", vae_layers: Optional[int] = None, vae_heads: int = 4, vae_ff: int = 1024,
                vae_nfeats: Optional[int] = None, scheduler: str = "ddim", num_train_timesteps: int = 1000,
                beta_start: float = 0.00085, beta_end: float = 0.012, steps_offset: int = 1,
                set_alpha_to_one: bool = False, eta: float = 0.0, njoints: int = 22,
                beta_schedule: str = "scaled_linear", clip_sample: bool = False) -> MldbConfig:
    """Build an ``mldb_config`` from the reference's ctor kwargs / yaml params
    (configs/modules/{denoiser,motion_vae,scheduler}.yaml).  ``eta`` (the yaml's scheduler.eta, in [0, 1]),
    ``beta_schedule`` (scaled_linear | linear | squaredcos_cap_v2) and ``clip_sample`` are diffusers'."""
    if beta_schedule not in _lib.BETA_SCHEDULES:
        raise ValueError(f"beta_schedule must be one of {sorted(_lib.BETA_SCHEDULES)}, got {beta_schedule!r}")
    if not 0.0 <= eta <= 1.0:
        raise ValueError(f"eta must lie in [0, 1], got {eta}")
    c = _lib.default_config()
    c.cond_kind = {"text": _lib.COND_TEXT, "action": _lib.COND_ACTION}[condition]
    c.arch = {"trans_enc": _lib.ARCH_TRANS_ENC, "trans_dec": _lib.ARCH_TRANS_DEC}[arch]
    c.n_lat, c.latent_dim = int(latent_dim[0]), int(latent_dim[-1])
    c.ff_size, c.num_layers, c.num_heads = ff_size, num_layers, num_heads
    c.text_dim, c.nclasses, c.nfeats = text_encoded_dim, nclasses, nfeats
    c.diffusion_only = int(diffusion_only)
    c.flip_sin_to_cos, c.freq_shift, c.guidance_scale = int(flip_sin_to_cos), freq_shift, guidance_scale
    c.vae_kind = {"none": _lib.VAE_NONE, "no": _lib.VAE_NONE, "mld": _lib.VAE_MLD, "actor": _lib.VAE_ACTOR}[vae]
    c.vae_layers = vae_layers if vae_layers is not None else (6 if vae == "actor" else 9)
    c.vae_heads, c.vae_ff = vae_heads, vae_ff
    c.vae_nfeats = vae_nfeats if vae_nfeats is not None else nfeats
    c.sched_kind = {"ddim": _lib.SCHED_DDIM, "ddpm": _lib.SCHED_DDPM}[scheduler]
    c.num_train_timesteps, c.beta_start, c.beta_end = num_train_timesteps, beta_start, beta_end
    c.steps_offset, c.set_alpha_to_one, c.eta, c.njoints = steps_offset, int(set_alpha_to_one), eta, njoints
    c.beta_schedule, c.clip_sample = _lib.BETA_SCHEDULES[beta_schedule], int(clip_sample)
    return c
