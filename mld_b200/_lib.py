"""ctypes binding of ``libmldb200.so`` (C ABI in ``include/mldb.h``).

The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no
Python/CPU fallback: a missing library is an ImportError with the build command, and every
non-zero status from the C side becomes a ``RuntimeError`` carrying ``mldb_last_error()``.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmldb200.so")

MLDB_ABI_VERSION = 4
COND_TEXT, COND_ACTION = 0, 1
ARCH_TRANS_ENC, ARCH_TRANS_DEC = 0, 1
VAE_NONE, VAE_MLD, VAE_ACTOR = 0, 1, 2
SCHED_DDIM, SCHED_DDPM = 0, 1
# diffusers beta_schedule names -> MLDB_BETA_*
BETA_SCHEDULES = {"scaled_linear": 0, "linear": 1, "squaredcos_cap_v2": 2}
DTYPE_F32 = 0
# mldb_kernel_stats indices (MLDB_KSTAT_* in include/mldb.h)
KSTAT_NAMES = ("gemm_tc", "gemm_ln_tc", "ffn_tc", "attn_tc", "attn_mma", "attn_simt", "gemm_simt", "ln_simt",
               "ln_unfused", "misc", "text_ln", "gru_tc")
# CLIP text tower (mldb_text_config, mldb_text_encode)
MLDB_TEXT_ABI_VERSION = 1
TEXT_HIDDEN, TEXT_POOLED = 0, 1
# BERT text tower (mldb_bert_config, mldb_bert_encode)
MLDB_BERT_ABI_VERSION = 1
BERT_DISTILBERT, BERT_BERT = 0, 1
# T2M evaluator (mldb_t2m_config, mldb_t2m_*)
MLDB_T2M_ABI_VERSION = 1
T2M_TEXT, T2M_MOVEMENT, T2M_MOTION = 1, 2, 4
# HumanAct12 action classifier (mldb_a2m_config, mldb_a2m_classify)
MLDB_A2M_ABI_VERSION = 1
# UESTC action classifier (mldb_stgcn_config, mldb_stgcn_classify)
MLDB_STGCN_ABI_VERSION = 1
# SMPL layer (mldb_smpl_config, mldb_smpl_forward)
MLDB_SMPL_ABI_VERSION = 1
SMPL_JOINTS, SMPL_VERTICES = 0, 1
# APE / AVE metric (mldb_ape_ave)
MLDB_APE_AVE_ABI_VERSION = 1
JOINTS_HUMANML3D, JOINTS_MMM = 0, 1


class MldbConfig(C.Structure):
    """``mldb_config`` (include/mldb.h)."""
    _fields_ = [
        ("abi_version", C.c_int32),
        ("cond_kind", C.c_int32), ("arch", C.c_int32), ("latent_dim", C.c_int32),
        ("n_lat", C.c_int32), ("num_heads", C.c_int32), ("ff_size", C.c_int32),
        ("num_layers", C.c_int32), ("text_dim", C.c_int32), ("nclasses", C.c_int32),
        ("nfeats", C.c_int32), ("diffusion_only", C.c_int32), ("flip_sin_to_cos", C.c_int32),
        ("freq_shift", C.c_float), ("guidance_scale", C.c_float),
        ("vae_kind", C.c_int32), ("vae_layers", C.c_int32), ("vae_heads", C.c_int32),
        ("vae_ff", C.c_int32), ("vae_nfeats", C.c_int32),
        ("sched_kind", C.c_int32), ("num_train_timesteps", C.c_int32),
        ("beta_start", C.c_double), ("beta_end", C.c_double), ("steps_offset", C.c_int32),
        ("set_alpha_to_one", C.c_int32), ("eta", C.c_float), ("njoints", C.c_int32),
        ("beta_schedule", C.c_int32), ("clip_sample", C.c_int32),
    ]


class MldbTextConfig(C.Structure):
    """``mldb_text_config`` (include/mldb.h)."""
    _fields_ = [
        ("abi_version", C.c_int32), ("vocab_size", C.c_int32), ("max_positions", C.c_int32),
        ("hidden", C.c_int32), ("heads", C.c_int32), ("layers", C.c_int32), ("ff", C.c_int32),
        ("projection_dim", C.c_int32), ("eos_token_id", C.c_int32), ("ln_eps", C.c_float),
    ]


class MldbBertConfig(C.Structure):
    """``mldb_bert_config`` (include/mldb.h)."""
    _fields_ = [
        ("abi_version", C.c_int32), ("family", C.c_int32), ("vocab_size", C.c_int32), ("max_positions", C.c_int32),
        ("type_vocab", C.c_int32), ("hidden", C.c_int32), ("heads", C.c_int32), ("layers", C.c_int32),
        ("ff", C.c_int32), ("ln_eps", C.c_float),
    ]


class MldbT2mConfig(C.Structure):
    """``mldb_t2m_config`` (include/mldb.h)."""
    _fields_ = [
        ("abi_version", C.c_int32), ("parts", C.c_int32), ("dim_word", C.c_int32), ("dim_pos_ohot", C.c_int32),
        ("dim_text_hidden", C.c_int32), ("dim_coemb_hidden", C.c_int32), ("dim_pose", C.c_int32),
        ("dim_move_hidden", C.c_int32), ("dim_move_latent", C.c_int32), ("dim_motion_hidden", C.c_int32),
        ("dim_motion_latent", C.c_int32),
    ]


class MldbA2mConfig(C.Structure):
    """``mldb_a2m_config`` (include/mldb.h)."""
    _fields_ = [
        ("abi_version", C.c_int32), ("input_size", C.c_int32), ("hidden_size", C.c_int32),
        ("hidden_layer", C.c_int32), ("output_size", C.c_int32),
    ]


class MldbStgcnConfig(C.Structure):
    """``mldb_stgcn_config`` (include/mldb.h)."""
    _fields_ = [("abi_version", C.c_int32), ("in_channels", C.c_int32), ("num_class", C.c_int32)]


class MldbSmplConfig(C.Structure):
    """``mldb_smpl_config`` (include/mldb.h)."""
    _fields_ = [("abi_version", C.c_int32), ("num_vertices", C.c_int32)]


class MldbGemmRowsArgs(C.Structure):
    """``mldb_gemm_rows_args`` (include/mldb.h)."""
    _fields_ = [
        ("A", C.c_void_p), ("W", C.c_void_p), ("bias", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("R", C.c_void_p), ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("K1", C.c_int32),
        ("act", C.c_int32), ("use_tc", C.c_int32), ("a_kind", C.c_int32),
        ("in_group", C.c_int32), ("out_group", C.c_int32), ("out_off", C.c_int32),
        ("addtab", C.c_void_p), ("tab_rows", C.c_int32), ("zero_lengths", C.c_void_p),
        ("vec_f32", C.c_int32), ("split_out", C.c_int32),
        ("out", C.c_void_p), ("out_rows", C.c_int32), ("out_cols", C.c_int32), ("out_col0", C.c_int32),
    ]


class MldbLnArgs(C.Structure):
    """``mldb_ln_args`` (include/mldb.h)."""
    _fields_ = [
        ("c", C.c_void_p), ("ldc", C.c_int32), ("res", C.c_void_p), ("rowvec", C.c_void_p), ("rv_group", C.c_int32),
        ("gamma", C.c_void_p), ("beta", C.c_void_p), ("M_in", C.c_int32), ("M", C.c_int32), ("d", C.c_int32),
        ("sel_group", C.c_int32), ("in_group", C.c_int32), ("act", C.c_int32), ("split_out", C.c_int32),
        ("out", C.c_void_p), ("ld_out", C.c_int32),
    ]


# name -> (restype, argtypes); every symbol include/mldb.h declares
_P = C.c_void_p
_SIGNATURES = {
    "mldb_default_config": (None, [C.POINTER(MldbConfig)]),
    "mldb_create": (C.c_int, [C.POINTER(MldbConfig), C.c_int, C.POINTER(_P)]),
    "mldb_destroy": (None, [_P]),
    "mldb_load_tensor": (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), C.c_int32, C.c_int32]),
    "mldb_finalize_weights": (C.c_int, [_P, _P]),
    "mldb_set_mean_std": (C.c_int, [_P, _P, _P, C.c_int32]),
    "mldb_scheduler_table": (C.c_int, [C.POINTER(MldbConfig), _P]),
    "mldb_scheduler_timesteps": (C.c_int, [C.POINTER(MldbConfig), C.c_int32, _P]),
    "mldb_scheduler_set_timesteps": (C.c_int, [_P, C.c_int32, _P]),
    "mldb_scheduler_step": (C.c_int, [_P, _P, C.c_int64, _P, _P, C.c_int64, _P, _P]),
    "mldb_denoise": (C.c_int, [_P, _P, C.c_int64, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mldb_diffusion_reverse": (C.c_int, [_P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mldb_vae_decode": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P]),
    "mldb_vae_encode": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P, _P]),
    "mldb_feats2joints": (C.c_int, [_P, _P, C.c_int32, C.c_int32, _P, _P]),
    "mldb_sample": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P]),
    "mldb_sample_host": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P]),
    "mldb_profile_op": (C.c_int, [_P, C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float)]),
    "mldb_profile_steps": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, _P]),
    "mldb_debug_timeline": (C.c_int, [C.c_int32, _P, C.c_int32, C.POINTER(C.c_int32)]),
    "mldb_debug_gemm": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mldb_debug_gemm_rows": (C.c_int, [_P, C.POINTER(MldbGemmRowsArgs), _P]),
    "mldb_debug_ln": (C.c_int, [_P, C.POINTER(MldbLnArgs), _P]),
    "mldb_debug_rows_to_split": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                           C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int32,
                                           _P]),
    "mldb_debug_ffn": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mldb_debug_tail": (C.c_int, [_P] * 13 + [C.c_int32] * 5 + [_P, _P]),
    "mldb_debug_attention": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_int32, _P, _P]),
    "mldb_debug_attention_causal": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                              C.c_int32, C.c_int32, _P, _P]),
    "mldb_default_text_config": (None, [C.POINTER(MldbTextConfig)]),
    "mldb_text_configure": (C.c_int, [_P, C.POINTER(MldbTextConfig)]),
    "mldb_text_encode": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mldb_default_bert_config": (None, [C.POINTER(MldbBertConfig)]),
    "mldb_bert_configure": (C.c_int, [_P, C.POINTER(MldbBertConfig)]),
    "mldb_bert_encode": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P]),
    "mldb_default_t2m_config": (None, [C.POINTER(MldbT2mConfig)]),
    "mldb_t2m_configure": (C.c_int, [_P, C.POINTER(MldbT2mConfig)]),
    "mldb_t2m_movement": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mldb_t2m_motion": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P]),
    "mldb_t2m_text": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P]),
    "mldb_default_a2m_config": (None, [C.POINTER(MldbA2mConfig)]),
    "mldb_a2m_configure": (C.c_int, [_P, C.POINTER(MldbA2mConfig)]),
    "mldb_a2m_classify": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P, _P]),
    "mldb_default_stgcn_config": (None, [C.POINTER(MldbStgcnConfig)]),
    "mldb_stgcn_configure": (C.c_int, [_P, C.POINTER(MldbStgcnConfig)]),
    "mldb_stgcn_classify": (C.c_int, [_P, _P, C.c_int32, C.c_int32, _P, _P, _P]),
    "mldb_default_smpl_config": (None, [C.POINTER(MldbSmplConfig)]),
    "mldb_smpl_configure": (C.c_int, [_P, C.POINTER(MldbSmplConfig)]),
    "mldb_smpl_forward": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mldb_ape_ave": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mldb_comm_unique_id": (C.c_int, [_P]),
    "mldb_comm_init": (C.c_int, [_P, _P, C.c_int32, C.c_int32]),
    "mldb_comm_attach": (C.c_int, [_P, _P, C.c_int32, C.c_int32]),
    "mldb_comm_info": (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "mldb_allgather": (C.c_int, [_P, _P, _P, C.c_int64, _P]),
    "mldb_sample_gather": (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P]),
    "mldb_gather_wait": (C.c_int, [_P, _P]),
    "mldb_kernel_stats": (C.c_int, [_P, _P, C.c_int32]),
    "mldb_reset_kernel_stats": (C.c_int, [_P]),
    "mldb_last_error": (C.c_char_p, []),
    "mldb_abi_version": (C.c_int, []),
    "mldb_launch_count": (C.c_int64, [_P]),
    "mldb_set_option": (C.c_int, [_P, C.c_char_p, C.c_char_p]),
}

_lib = None


def lib():
    """Load libmldb200.so once; fail loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a). mld_b200 has no CPU or PyTorch fallback.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)      # AttributeError if the ABI lost a symbol
            fn.restype = res
            fn.argtypes = args
        if l.mldb_abi_version() != MLDB_ABI_VERSION:
            raise ImportError("libmldb200.so ABI version mismatch; rebuild")
        _lib = l
    return _lib


def check(status: int, what: str = "mldb"):
    if status != 0:
        msg = lib().mldb_last_error()
        raise RuntimeError(f"{what} failed (status {status}): {msg.decode() if msg else '?'}")


def default_config() -> MldbConfig:
    cfg = MldbConfig()
    lib().mldb_default_config(C.byref(cfg))
    return cfg


def default_text_config() -> MldbTextConfig:
    cfg = MldbTextConfig()
    lib().mldb_default_text_config(C.byref(cfg))
    return cfg


def default_bert_config() -> MldbBertConfig:
    cfg = MldbBertConfig()
    lib().mldb_default_bert_config(C.byref(cfg))
    return cfg


def default_t2m_config() -> MldbT2mConfig:
    cfg = MldbT2mConfig()
    lib().mldb_default_t2m_config(C.byref(cfg))
    return cfg


def default_a2m_config() -> MldbA2mConfig:
    cfg = MldbA2mConfig()
    lib().mldb_default_a2m_config(C.byref(cfg))
    return cfg


def default_stgcn_config() -> MldbStgcnConfig:
    cfg = MldbStgcnConfig()
    lib().mldb_default_stgcn_config(C.byref(cfg))
    return cfg


def default_smpl_config() -> MldbSmplConfig:
    cfg = MldbSmplConfig()
    lib().mldb_default_smpl_config(C.byref(cfg))
    return cfg
