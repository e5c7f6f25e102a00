"""Seeded synthetic weights and inputs with the reference's state-dict key names and shapes.

There are no checkpoints, CLIP weights or datasets offline, so tests, ``bench.py`` and
``smoke()`` run on random-init weights of the reference architecture.  Keys/shapes follow
the reference modules exactly (``MldDenoiser`` mld_denoiser.py:40-131, ``MldVae``
mld_vae.py:49-114, ``ActorVae`` actor_vae.py:26-51); ``oracle/make_golden.py`` loads these
dicts into the reference's own modules with ``strict=True``, which pins the key contract.
Biases and LayerNorm affines are randomised (the reference initialises them to 0/1) so that
parity tests exercise every term.
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch

Tensor = torch.Tensor


class _Gen:
    def __init__(self, seed: int):
        self.g = torch.Generator().manual_seed(seed)

    def xavier(self, out_f: int, in_f: int) -> Tensor:
        a = math.sqrt(6.0 / (in_f + out_f))
        return (torch.rand(out_f, in_f, generator=self.g) * 2 - 1) * a

    def normal(self, *shape, std=1.0) -> Tensor:
        return torch.randn(*shape, generator=self.g) * std

    def uniform(self, *shape) -> Tensor:
        return torch.rand(*shape, generator=self.g)


def _attn(sd: Dict[str, Tensor], g: _Gen, p: str, d: int):
    sd[p + "in_proj_weight"] = g.xavier(3 * d, d)
    sd[p + "in_proj_bias"] = g.normal(3 * d, std=0.02)
    sd[p + "out_proj.weight"] = g.xavier(d, d)
    sd[p + "out_proj.bias"] = g.normal(d, std=0.02)


def _ln(sd, g: _Gen, p: str, d: int):
    sd[p + "weight"] = 1.0 + g.normal(d, std=0.1)
    sd[p + "bias"] = g.normal(d, std=0.05)


def _ffn(sd, g: _Gen, p: str, d: int, ff: int):
    sd[p + "linear1.weight"] = g.xavier(ff, d)
    sd[p + "linear1.bias"] = g.normal(ff, std=0.02)
    sd[p + "linear2.weight"] = g.xavier(d, ff)
    sd[p + "linear2.bias"] = g.normal(d, std=0.02)


def _enc_layer(sd, g, p, d, ff):
    _attn(sd, g, p + "self_attn.", d)
    _ffn(sd, g, p, d, ff)
    _ln(sd, g, p + "norm1.", d)
    _ln(sd, g, p + "norm2.", d)


def _dec_layer(sd, g, p, d, ff):
    _attn(sd, g, p + "self_attn.", d)
    _attn(sd, g, p + "multihead_attn.", d)
    _ffn(sd, g, p, d, ff)
    _ln(sd, g, p + "norm1.", d)
    _ln(sd, g, p + "norm2.", d)
    _ln(sd, g, p + "norm3.", d)


def _skip_stack(sd, g, p, d, ff, num_layers, layer_fn):
    nb = (num_layers - 1) // 2
    _ln(sd, g, p + "norm.", d)
    for i in range(nb):
        layer_fn(sd, g, f"{p}input_blocks.{i}.", d, ff)
    layer_fn(sd, g, f"{p}middle_block.", d, ff)
    for i in range(nb):
        layer_fn(sd, g, f"{p}output_blocks.{i}.", d, ff)
    for i in range(nb):
        sd[f"{p}linear_blocks.{i}.weight"] = g.xavier(d, 2 * d)
        sd[f"{p}linear_blocks.{i}.bias"] = g.normal(d, std=0.02)


def denoiser_state_dict(seed: int = 1234, condition: str = "text", arch: str = "trans_enc",
                        d: int = 256, ff: int = 1024, num_layers: int = 9,
                        text_dim: int = 768, nclasses: int = 12, nfeats: int = 263,
                        diffusion_only: bool = False) -> Dict[str, Tensor]:
    """State dict of ``MldDenoiser`` (text / action; skip trans_enc / no-VAE trans_dec)."""
    g, sd = _Gen(seed), {}
    if diffusion_only:
        sd["pose_embd.weight"] = g.xavier(d, nfeats)
        sd["pose_embd.bias"] = g.normal(d, std=0.02)
        sd["pose_proj.weight"] = g.xavier(nfeats, d)
        sd["pose_proj.bias"] = g.normal(nfeats, std=0.02)
    tdim = text_dim if condition == "text" else d
    sd["time_embedding.linear_1.weight"] = g.xavier(d, tdim)
    sd["time_embedding.linear_1.bias"] = g.normal(d, std=0.02)
    sd["time_embedding.linear_2.weight"] = g.xavier(d, d)
    sd["time_embedding.linear_2.bias"] = g.normal(d, std=0.02)
    if condition == "text":
        sd["emb_proj.1.weight"] = g.xavier(d, text_dim)
        sd["emb_proj.1.bias"] = g.normal(d, std=0.02)
    else:
        sd["emb_proj.action_embedding"] = g.xavier(nclasses, d)
    sd["query_pos.pe"] = g.uniform(500, 1, d)
    sd["mem_pos.pe"] = g.uniform(500, 1, d)
    if arch == "trans_enc":
        _skip_stack(sd, g, "encoder.", d, ff, num_layers, _enc_layer)
    else:
        for i in range(num_layers):
            _dec_layer(sd, g, f"decoder.layers.{i}.", d, ff)
        _ln(sd, g, "decoder.norm.", d)
    return sd


def mld_vae_state_dict(seed: int = 4321, nfeats: int = 263, d: int = 256, ff: int = 1024,
                       num_layers: int = 9, n_lat: int = 1) -> Dict[str, Tensor]:
    """State dict of ``MldVae`` (arch encoder_decoder, learned PE, MLP_DIST False)."""
    g, sd = _Gen(seed), {}
    sd["global_motion_token"] = g.normal(2 * n_lat, d)
    sd["query_pos_encoder.pe"] = g.uniform(500, 1, d)
    sd["query_pos_decoder.pe"] = g.uniform(500, 1, d)
    _skip_stack(sd, g, "encoder.", d, ff, num_layers, _enc_layer)
    _skip_stack(sd, g, "decoder.", d, ff, num_layers, _dec_layer)
    sd["skel_embedding.weight"] = g.xavier(d, nfeats)
    sd["skel_embedding.bias"] = g.normal(d, std=0.02)
    sd["final_layer.weight"] = g.xavier(nfeats, d)
    sd["final_layer.bias"] = g.normal(nfeats, std=0.02)
    return sd


def sine_pe_table(n: int, d: int) -> Tensor:
    """The ``PositionalEncoding`` buffer (position_encoding_layer.py:14-20), rows [n, d]."""
    pe = torch.zeros(n, d)
    position = torch.arange(0, n, dtype=torch.float).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d, 2).float() * (-math.log(10000.0) / d))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def actor_vae_state_dict(seed: int = 777, nfeats: int = 150, d: int = 256, ff: int = 1024,
                         num_layers: int = 6, with_encoder: bool = True) -> Dict[str, Tensor]:
    """State dict of ``ActorVae`` (torch nn.TransformerEncoder/Decoder stacks, sine PE)."""
    g, sd = _Gen(seed), {}
    pe = sine_pe_table(5000, d).unsqueeze(1)
    if with_encoder:
        sd["encoder.mu_token"] = g.normal(d)
        sd["encoder.logvar_token"] = g.normal(d)
        sd["encoder.skel_embedding.weight"] = g.xavier(d, nfeats)
        sd["encoder.skel_embedding.bias"] = g.normal(d, std=0.02)
        sd["encoder.sequence_pos_encoding.pe"] = pe.clone()
        for i in range(num_layers):
            _enc_layer(sd, g, f"encoder.seqTransEncoder.layers.{i}.", d, ff)
    sd["decoder.sequence_pos_encoding.pe"] = pe.clone()
    for i in range(num_layers):
        _dec_layer(sd, g, f"decoder.seqTransDecoder.layers.{i}.", d, ff)
    sd["decoder.final_layer.weight"] = g.xavier(nfeats, d)
    sd["decoder.final_layer.bias"] = g.normal(nfeats, std=0.02)
    return sd


def text_context(B: int, S: int, seed: int = 1, text_dim: int = 768) -> Tensor:
    """Synthetic CLIP output ``[2B, S, 768]`` for CFG: the uncond half first
    (mld.py:225-230), all uncond rows equal (every "" prompt encodes identically)."""
    g = torch.Generator().manual_seed(seed)
    uncond = torch.randn(1, S, text_dim, generator=g).expand(B, S, text_dim)
    cond = torch.randn(B, S, text_dim, generator=g)
    return torch.cat([uncond, cond], 0).contiguous()


def init_noise(B: int, n_lat: int = 1, d: int = 256, seed: int = 2) -> Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, n_lat, d, generator=g)


def ragged_lengths(B: int, lo: int = 40, hi: int = 196, seed: int = 3) -> List[int]:
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(lo, hi + 1, (B,), generator=g) // 4 * 4).tolist()


def mean_std(nfeats: int = 263, seed: int = 5):
    """Synthetic dataset statistics (``Mean.npy`` / ``Std.npy`` are absent offline) with
    HumanML3D-like magnitudes: per-frame root rotation / translation velocities of a few
    hundredths (rad, m), root height ~0.9 m, joint offsets of decimetres.  feats2joints
    integrates the velocities over up to 196 frames, so the magnitudes matter for how the
    1e-3 joint-position gate conditions the path (see DESIGN.md)."""
    g = torch.Generator().manual_seed(seed)
    mean = torch.randn(nfeats, generator=g) * 0.05
    std = 0.2 + 0.8 * torch.rand(nfeats, generator=g)
    mean[0], std[0] = 0.0, 0.03                      # root angular velocity (rad/frame)
    mean[1:3] = torch.tensor([0.0, 0.02])
    std[1:3] = 0.03                                  # root linear velocity xz (m/frame)
    mean[3], std[3] = 0.9, 0.1                       # root height
    n_ric = min(nfeats, 67) - 4
    if n_ric > 0:
        mean[4:4 + n_ric] = torch.randn(n_ric, generator=g) * 0.3
        std[4:4 + n_ric] = 0.1 + 0.2 * torch.rand(n_ric, generator=g)
    return mean, std


def clip_text_state_dict(seed: int = 4242, vocab_size: int = 49408, max_positions: int = 77, hidden: int = 768,
                         layers: int = 12, ff: int = 3072, projection_dim: int = 768, **_unused) -> Dict[str, Tensor]:
    """State dict of the CLIP text tower as ``MldTextEncoder.state_dict()`` names it (mld_clip.py:26-27: its
    ``text_model`` is a ``CLIPModel``): ``text_model.text_model.*`` and ``text_model.text_projection.weight``.
    Stripping the leading ``text_model.`` gives the keys of transformers' ``CLIPTextModelWithProjection``.  The
    default shape is CLIP ViT-L/14's text tower; smaller shapes are for fast tests (``heads`` does not change the
    weights and is accepted for symmetry with the text config)."""
    g, sd = _Gen(seed), {}
    p = "text_model.text_model."
    sd[p + "embeddings.token_embedding.weight"] = g.normal(vocab_size, hidden, std=0.02)
    sd[p + "embeddings.position_embedding.weight"] = g.normal(max_positions, hidden, std=0.01)
    for i in range(layers):
        q = f"{p}encoder.layers.{i}."
        for name in ("k_proj", "v_proj", "q_proj", "out_proj"):
            sd[f"{q}self_attn.{name}.weight"] = g.xavier(hidden, hidden)
            sd[f"{q}self_attn.{name}.bias"] = g.normal(hidden, std=0.02)
        _ln(sd, g, q + "layer_norm1.", hidden)
        sd[q + "mlp.fc1.weight"] = g.xavier(ff, hidden)
        sd[q + "mlp.fc1.bias"] = g.normal(ff, std=0.02)
        sd[q + "mlp.fc2.weight"] = g.xavier(hidden, ff)
        sd[q + "mlp.fc2.bias"] = g.normal(hidden, std=0.02)
        _ln(sd, g, q + "layer_norm2.", hidden)
    _ln(sd, g, p + "final_layer_norm.", hidden)
    sd["text_model.text_projection.weight"] = g.xavier(projection_dim, hidden)
    return sd


def clip_text_ids(n: int, L: int = 77, seed: int = 7, eos_lo: int = 8, eos_hi: int = 30, vocab_size: int = 49408,
                  bos: int = 49406, eos: int = 49407) -> Tensor:
    """Tokenizer-shaped id rows ``[n, L]`` (int64): bos, random word ids, eos at a seeded position in
    [eos_lo, eos_hi], then eos padding (CLIP's pad token is its eos token)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, min(bos, vocab_size), (n, L), generator=g)
    pos = torch.randint(eos_lo, eos_hi + 1, (n,), generator=g).clamp(max=L - 1)
    ids[:, 0] = bos
    ids[torch.arange(L).expand(n, L) >= pos[:, None]] = eos
    return ids


# ---------------------------------------------------------------------------- T2M evaluator (finest.tar layout)
T2M_DIMS = dict(dim_word=300, dim_pos_ohot=15, dim_text_hidden=512, dim_coemb_hidden=512, dim_pose=259,
                dim_move_hidden=512, dim_move_latent=512, dim_motion_hidden=1024, dim_motion_latent=512)


def _t2m_uniform(g: _Gen, bound: float, *shape) -> Tensor:
    return (g.uniform(*shape) * 2 - 1) * bound


def _t2m_linear(sd, g: _Gen, p: str, out_f: int, in_f: int, k: int = 1):
    """torch's default Linear / Conv1d init: weight and bias U(-1/sqrt(fan_in), 1/sqrt(fan_in))."""
    b = 1.0 / math.sqrt(in_f * k)
    sd[p + "weight"] = _t2m_uniform(g, b, out_f, in_f, k) if k > 1 else _t2m_uniform(g, b, out_f, in_f)
    sd[p + "bias"] = _t2m_uniform(g, b, out_f)


def _t2m_bigru(sd, g: _Gen, in_f: int, H: int, out: int):
    """nn.GRU(in_f, H, bidirectional) (default init U(-1/sqrt(H), 1/sqrt(H))), the learned initial state
    ``hidden`` (torch.randn, as the reference) and the BiGRUCo output_net."""
    b = 1.0 / math.sqrt(H)
    for sfx in ("", "_reverse"):
        sd["gru.weight_ih_l0" + sfx] = _t2m_uniform(g, b, 3 * H, in_f)
        sd["gru.weight_hh_l0" + sfx] = _t2m_uniform(g, b, 3 * H, H)
        sd["gru.bias_ih_l0" + sfx] = _t2m_uniform(g, b, 3 * H)
        sd["gru.bias_hh_l0" + sfx] = _t2m_uniform(g, b, 3 * H)
    _t2m_linear(sd, g, "output_net.0.", H, 2 * H)
    _ln(sd, g, "output_net.1.", H)
    _t2m_linear(sd, g, "output_net.3.", out, H)
    sd["hidden"] = g.normal(2, 1, H)


def t2m_state_dicts(seed: int = 2468, **dims) -> Dict[str, Dict[str, Tensor]]:
    """The three evaluator state dicts under finest.tar's keys ``text_encoder``, ``movement_encoder`` and
    ``motion_encoder`` (mld.py:176-181), shaped by ``T2M_DIMS`` (configs/base.yaml model.t2m_*; dim_pose is
    NFEATS - 4).  Linear, Conv1d and GRU weights follow torch's default init; the LayerNorm affine is randomised as
    elsewhere in this module so that parity tests exercise every term."""
    d = {**T2M_DIMS, **dims}
    g = _Gen(seed)
    text: Dict[str, Tensor] = {}
    _t2m_linear(text, g, "pos_emb.", d["dim_word"], d["dim_pos_ohot"])
    _t2m_linear(text, g, "input_emb.", d["dim_text_hidden"], d["dim_word"])
    _t2m_bigru(text, g, d["dim_text_hidden"], d["dim_text_hidden"], d["dim_coemb_hidden"])
    move: Dict[str, Tensor] = {}
    _t2m_linear(move, g, "main.0.", d["dim_move_hidden"], d["dim_pose"], 4)
    _t2m_linear(move, g, "main.3.", d["dim_move_latent"], d["dim_move_hidden"], 4)
    _t2m_linear(move, g, "out_net.", d["dim_move_latent"], d["dim_move_latent"])
    motion: Dict[str, Tensor] = {}
    _t2m_linear(motion, g, "input_emb.", d["dim_motion_hidden"], d["dim_move_latent"])
    _t2m_bigru(motion, g, d["dim_motion_hidden"], d["dim_motion_hidden"], d["dim_motion_latent"])
    return {"text_encoder": text, "movement_encoder": move, "motion_encoder": motion}


def t2m_text_inputs(B: int, L: int = 22, seed: int = 11, dim_word: int = 300, dim_pos_ohot: int = 15):
    """GloVe-shaped word vectors ``[B, L, 300]`` (element std ~0.4, as GloVe 300d) and one-hot POS rows
    ``[B, L, 15]`` (one random category per token, padding tokens included, as the dataset pads with a word)."""
    g = torch.Generator().manual_seed(seed)
    word = torch.randn(B, L, dim_word, generator=g) * 0.4
    cat = torch.randint(0, dim_pos_ohot, (B, L), generator=g)
    pos = torch.nn.functional.one_hot(cat, dim_pos_ohot).float()
    return word, pos


def t2m_mean_std(nfeats: int = 263, seed: int = 6):
    """Synthetic evaluator statistics (``mean_eval`` / ``std_eval``, the t2m model's Mean.npy / Std.npy): the
    dataset statistics of :func:`mean_std` perturbed, so that ``renorm4t2m`` maps zero padding rows to non-zero."""
    mean, std = mean_std(nfeats)
    g = torch.Generator().manual_seed(seed)
    return mean + 0.1 * std * torch.randn(nfeats, generator=g), std * (0.8 + 0.4 * torch.rand(nfeats, generator=g))


def t2m_feats(B: int, T: int, lengths: List[int], seed: int = 12, nfeats: int = 263) -> Tensor:
    """Dataset-normalised motion features ``[B, T, nfeats]``: N(0, 1) rows up to each length, zero padding after
    (the HumanML3D loader pads normalised motions with zeros)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, nfeats, generator=g)
    for b, n in enumerate(lengths):
        x[b, n:] = 0.0
    return x


def renorm4t2m(feats: Tensor, mean: Tensor, std: Tensor, mean_eval: Tensor, std_eval: Tensor) -> Tensor:
    """HumanML3DDataModule.renorm4t2m (mld/data/HumanML3D.py:54-62)."""
    feats = feats * std.to(feats) + mean.to(feats)
    return (feats - mean_eval.to(feats)) / std_eval.to(feats)


A2M_DIMS = {"input_size": 72, "hidden_size": 128, "hidden_layer": 2, "output_size": 12}   # metrics/gru.py:32-36


def a2m_state_dict(seed: int = 1357, **dims) -> Dict[str, Tensor]:
    """``MotionDiscriminator``'s state dict (the keys of HumanAct12's ``a2m_checkpoint["model"]``), shaped by
    ``A2M_DIMS``, with torch's default init: GRU weights and biases U(-1/sqrt(H), 1/sqrt(H)), Linear
    U(-1/sqrt(fan_in), 1/sqrt(fan_in))."""
    d = {**A2M_DIMS, **dims}
    g = _Gen(seed)
    H = d["hidden_size"]
    b = 1.0 / math.sqrt(H)
    sd: Dict[str, Tensor] = {}
    for k in range(d["hidden_layer"]):
        sd[f"recurrent.weight_ih_l{k}"] = _t2m_uniform(g, b, 3 * H, d["input_size"] if k == 0 else H)
        sd[f"recurrent.weight_hh_l{k}"] = _t2m_uniform(g, b, 3 * H, H)
        sd[f"recurrent.bias_ih_l{k}"] = _t2m_uniform(g, b, 3 * H)
        sd[f"recurrent.bias_hh_l{k}"] = _t2m_uniform(g, b, 3 * H)
    _t2m_linear(sd, g, "linear1.", 30, H)
    _t2m_linear(sd, g, "linear2.", d["output_size"], 30)
    return sd


def a2m_motions(B: int, T: int = 60, seed: int = 21, njoints: int = 24, nfeats: int = 3) -> Tensor:
    """Smooth synthetic joint trajectories ``[B, njoints, nfeats, T]`` (what ``feats2joints_eval`` hands the
    classifier): a per-joint offset of ~0.5 m plus three sinusoids per coordinate with random frequency and phase."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T, dtype=torch.float32) / 30.0                          # 30 fps
    base = torch.randn(B, njoints, nfeats, 1, generator=g) * 0.5
    x = base.expand(B, njoints, nfeats, T).clone()
    for _ in range(3):
        amp = torch.rand(B, njoints, nfeats, 1, generator=g) * 0.2
        freq = 0.2 + torch.rand(B, njoints, nfeats, 1, generator=g) * 2.0
        phase = torch.rand(B, njoints, nfeats, 1, generator=g) * 2 * math.pi
        x = x + amp * torch.sin(2 * math.pi * freq * t + phase)
    return x


# ---------------------------------------------------------------------------- UESTC action classifier (STGCN)
STGCN_DIMS = {"in_channels": 6, "num_class": 40}                              # metrics/stgcn.py:32-40
STGCN_CHANNELS = (64, 64, 64, 64, 128, 128, 128, 256, 256, 256)
STGCN_STRIDES = (1, 1, 1, 1, 2, 1, 1, 2, 1, 1)


def stgcn_residual(i: int, in_channels: int = 6) -> str:
    """The residual of st_gcn block i: "none" (block 0), "identity", or "conv" (1 x 1 stride-s conv + BN)."""
    if i == 0:
        return "none"
    cin = STGCN_CHANNELS[i - 1]
    return "identity" if cin == STGCN_CHANNELS[i] and STGCN_STRIDES[i] == 1 else "conv"


def _stgcn_bn(sd, g: _Gen, p: str, n: int):
    """Eval-mode BatchNorm with non-trivial statistics: running_var spread over two decades."""
    sd[p + "weight"] = 0.5 + g.uniform(n)
    sd[p + "bias"] = g.normal(n, std=0.1)
    sd[p + "running_mean"] = g.normal(n, std=0.2)
    sd[p + "running_var"] = 10.0 ** (g.uniform(n) * 2 - 1)
    sd[p + "num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)


def stgcn_state_dict(seed: int = 2025, **dims) -> Dict[str, Tensor]:
    """``STGCN``'s state dict (the keys of ``uestc_rot6d_stgcn.tar``), shaped by ``STGCN_DIMS``: convolutions with
    torch's default init U(-1/sqrt(fan_in), 1/sqrt(fan_in)), BatchNorms with spread statistics, edge importances in
    [0.8, 1.2] and ``A`` from SMPL's parent table."""
    from .graph import smpl_adjacency
    d = {**STGCN_DIMS, **dims}
    g = _Gen(seed)
    cin0 = d["in_channels"]
    sd: Dict[str, Tensor] = {"A": smpl_adjacency()}
    _stgcn_bn(sd, g, "data_bn.", 24 * cin0)
    for i, co in enumerate(STGCN_CHANNELS):
        ci = STGCN_CHANNELS[i - 1] if i else cin0
        p = f"st_gcn_networks.{i}."
        _t2m_linear(sd, g, p + "gcn.conv.", 3 * co, ci)
        sd[p + "gcn.conv.weight"] = sd[p + "gcn.conv.weight"].reshape(3 * co, ci, 1, 1)
        _stgcn_bn(sd, g, p + "tcn.0.", co)
        b = 1.0 / math.sqrt(co * 9)
        sd[p + "tcn.2.weight"] = _t2m_uniform(g, b, co, co, 9, 1)
        sd[p + "tcn.2.bias"] = _t2m_uniform(g, b, co)
        _stgcn_bn(sd, g, p + "tcn.3.", co)
        if stgcn_residual(i, cin0) == "conv":
            _t2m_linear(sd, g, p + "residual.0.", co, ci)
            sd[p + "residual.0.weight"] = sd[p + "residual.0.weight"].reshape(co, ci, 1, 1)
            _stgcn_bn(sd, g, p + "residual.1.", co)
    for i in range(len(STGCN_CHANNELS)):
        sd[f"edge_importance.{i}"] = 0.8 + 0.4 * g.uniform(3, 24, 24)
    _t2m_linear(sd, g, "fcn.", d["num_class"], 256)
    sd["fcn.weight"] = sd["fcn.weight"].reshape(d["num_class"], 256, 1, 1)
    return sd


def uestc_motions(B: int, T: int = 60, seed: int = 31, njoints: int = 24) -> Tensor:
    """Smooth rot6d-like motions ``[B, njoints, 6, T]`` (what ``UESTCMetrics.update`` hands the classifier): per joint,
    the first two columns of a rotation about a fixed random axis whose angle is an offset plus three sinusoids."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(T, dtype=torch.float64) / 30.0                          # 30 fps
    axis = torch.randn(B, njoints, 3, 1, generator=g, dtype=torch.float64)
    axis = axis / axis.norm(dim=2, keepdim=True)
    ang = (torch.rand(B, njoints, 1, generator=g, dtype=torch.float64) * 2 - 1) * math.pi
    for _ in range(3):
        amp = torch.rand(B, njoints, 1, generator=g, dtype=torch.float64) * 0.5
        freq = 0.2 + torch.rand(B, njoints, 1, generator=g, dtype=torch.float64) * 2.0
        phase = torch.rand(B, njoints, 1, generator=g, dtype=torch.float64) * 2 * math.pi
        ang = ang + amp * torch.sin(2 * math.pi * freq * t + phase)
    kx, ky, kz = axis[:, :, 0], axis[:, :, 1], axis[:, :, 2]             # [B, J, 1]
    c, s = torch.cos(ang), torch.sin(ang)                                # [B, J, T]
    C1 = 1 - c
    # Rodrigues: the first two columns of R = cI + s[k]x + (1 - c) k k^T
    col0 = torch.stack([c + kx * kx * C1, kz * s + ky * kx * C1, -ky * s + kz * kx * C1], 2)
    col1 = torch.stack([-kz * s + kx * ky * C1, c + ky * ky * C1, kx * s + kz * ky * C1], 2)
    return torch.cat([col0, col1], 2).float()                          # [B, J, 6, T]


SMPL_PARENTS = (-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21)   # SMPL's kintree


def smpl_model(seed: int = 99, V: int = 333, dense_every: int = 37) -> Dict[str, Tensor]:
    """A seeded synthetic SMPL model in the layout ``mld_b200.smpl.load_smpl`` returns: SMPL's public parent table, a
    body-sized ``v_template`` [V, 3] (metres), ``J_regressor`` [24, V] with sparse convex rows (6 vertices each),
    ``lbs_weights`` [V, 24] whose rows sum to 1 with 1 to 4 non-zeros, except every ``dense_every``-th row which
    weighs all 24 joints, and ``posedirs`` [207, 3 V] of size about 1e-2."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor([-0.45, -1.15, -0.15]), torch.tensor([0.45, 0.55, 0.15])
    vt = lo + (hi - lo) * torch.rand(V, 3, generator=g)
    jr = torch.zeros(24, V)
    for j in range(24):
        idx = torch.randperm(V, generator=g)[:min(6, V)]
        w = torch.rand(len(idx), generator=g) + 0.1
        jr[j, idx] = w / w.sum()
    lw = torch.zeros(V, 24)
    for v in range(V):
        k = 24 if dense_every and v % dense_every == 0 else 1 + int(torch.randint(0, 4, (1,), generator=g))
        idx = torch.randperm(24, generator=g)[:k]
        w = torch.rand(k, generator=g) + 0.05
        lw[v, idx] = w / w.sum()
    posedirs = torch.randn(207, 3 * V, generator=g) * 1e-2
    return {"v_template": vt, "posedirs": posedirs, "J_regressor": jr, "lbs_weights": lw,
            "parents": torch.tensor(SMPL_PARENTS, dtype=torch.int64)}


def write_smpl_pkl(path: str, model: Dict[str, Tensor], array=None):
    """Write ``model`` (``smpl_model``'s layout) as ``SMPL_NEUTRAL.pkl`` is laid out: ``posedirs`` [V, 3, 207],
    ``weights``, ``kintree_table`` [2, 24] (row 0 the parents, the root's 4294967295), a scipy sparse
    ``J_regressor``, zero ``shapedirs`` [V, 3, 10] and ``f``.  ``array`` wraps every dense array (a chumpy stand-in)."""
    import pickle

    import numpy as np
    import scipy.sparse
    wrap = array or (lambda a: a)
    V = model["v_template"].shape[0]
    parents = model["parents"].numpy().astype(np.int64).copy()
    parents[0] = 4294967295
    data = {
        "v_template": wrap(model["v_template"].double().numpy()),
        "posedirs": wrap(model["posedirs"].double().numpy().T.reshape(V, 3, 207)),
        "J_regressor": scipy.sparse.csc_matrix(model["J_regressor"].double().numpy()),
        "weights": wrap(model["lbs_weights"].double().numpy()),
        "kintree_table": np.stack([parents, np.arange(24, dtype=np.int64)]),
        "shapedirs": wrap(np.zeros((V, 3, 10))),
        "f": np.zeros((1, 3), dtype=np.uint32),
    }
    with open(path, "wb") as f:
        pickle.dump(data, f, protocol=2)


def smpl_feats(B: int, T: int = 60, seed: int = 51) -> Tensor:
    """Rot6d features ``[B, T, 150]`` as ``MLD`` holds them (``view(B, T, 6, 25)``): ``uestc_motions``'s smooth
    rotations for the 24 joints and a smooth root translation (metres) in column 24."""
    rot = uestc_motions(B, T, seed=seed)                                   # [B, 24, 6, T]
    g = torch.Generator().manual_seed(seed + 1)
    t = torch.arange(T, dtype=torch.float32) / 30.0
    trans = torch.randn(B, 3, 1, generator=g) * 0.3 + torch.randn(B, 3, 1, generator=g) * 0.5 * t
    x = torch.zeros(B, T, 6, 25)
    x[..., :24] = rot.permute(0, 3, 2, 1)
    x[:, :, :3, 24] = trans.permute(0, 2, 1)
    return x.reshape(B, T, 150)
