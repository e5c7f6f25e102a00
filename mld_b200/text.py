"""``B200TextEncoder``: drop-in replacement for the reference's CLIP text encoder, selectable through the YAML
``target:`` factory (``instantiate_from_config``, mld/config.py:106-121):

    text_encoder.target:  mld_b200.text.B200TextEncoder     (was mld.models.architectures.mld_clip.MldTextEncoder)

Same ctor kwargs (``modelpath, finetune, last_hidden_state, latent_dim``), same ``state_dict`` keys of the text
tower, same ``forward(texts) -> Tensor``: ``[n, 1, projection_dim]`` (``clip``, the shipped config) or
``[n, L, hidden]`` (``clip_hidden``).  The tokenizer stays on the host (Hugging Face's); everything after the
int64 ids runs in ``libmldb200.so`` (``mldb_text_encode``).  Two exact savings are applied to the host ids before
upload: every distinct id row is encoded once (the B identical "" rows of classifier-free guidance), and in
``clip`` mode only the first ``max(eos_pos) + 1`` columns are sent - under the causal mask no later token reaches
a pooled row.  Inference only.
"""
from __future__ import annotations

from dataclasses import asdict, dataclass
from typing import Dict, List, Optional

import torch

from . import _lib
from .modules import _EngineModule, _register_tree
from .engine import make_config

TOWER_PREFIXES = ("text_model.text_model.", "text_model.text_projection.")


@dataclass
class ClipTextConfig:
    """The text tower's shape (``mldb_text_config``); defaults are CLIP ViT-L/14 (openai/clip-vit-large-patch14)."""
    vocab_size: int = 49408
    max_positions: int = 77
    hidden: int = 768
    heads: int = 12
    layers: int = 12
    ff: int = 3072
    projection_dim: int = 768
    eos_token_id: int = 49407
    ln_eps: float = 1e-5

    def to_c(self) -> _lib.MldbTextConfig:
        c = _lib.default_text_config()
        for k, v in asdict(self).items():
            setattr(c, k, v)
        return c


def eos_positions(ids: torch.Tensor, eos_token_id: int) -> torch.Tensor:
    """Position of the pooled token per row, transformers' rule: the first id equal to ``eos_token_id`` (0 when
    absent); ``argmax(ids)`` under the legacy ``eos_token_id == 2``.  Both agree on CLIP vocabularies."""
    ids32 = ids.to(torch.int32)
    if eos_token_id == 2:
        return ids32.argmax(dim=-1)
    return (ids32 == eos_token_id).int().argmax(dim=-1)


def plan_ids(ids: torch.Tensor, pooled: bool, eos_token_id: int):
    """Host-side savings: ``(rows, inverse)`` with ``rows`` the distinct id rows (truncated to
    ``max(eos_pos) + 1`` columns when ``pooled``) and ``rows[inverse] `` the original rows' encodings."""
    rows, inverse = torch.unique(ids, dim=0, return_inverse=True)
    if pooled:
        rows = rows[:, :int(eos_positions(rows, eos_token_id).max()) + 1].contiguous()
    return rows, inverse


def check_ids(ids, vocab_size: int, max_positions: int) -> torch.Tensor:
    ids = torch.as_tensor(ids)
    if ids.dtype.is_floating_point or ids.dtype == torch.bool:
        raise TypeError(f"token ids must be integers, got {ids.dtype}")
    if ids.dim() != 2 or ids.shape[0] < 1 or not 1 <= ids.shape[1] <= max_positions:
        raise ValueError(f"ids must be [n, L] with 1 <= L <= {max_positions}, got {tuple(ids.shape)}")
    ids = ids.to(device="cpu", dtype=torch.int64)
    if int(ids.min()) < 0 or int(ids.max()) >= vocab_size:
        raise ValueError(f"token ids must lie in [0, {vocab_size})")
    return ids


class B200TextEncoder(_EngineModule):
    """``MldTextEncoder`` (mld/models/architectures/mld_clip.py:13-97), CLIP text models only."""
    _prefix = "text_encoder."

    def __init__(self, modelpath: Optional[str] = None, finetune: bool = False, last_hidden_state: bool = False,
                 latent_dim: list = [1, 256], *, state_dict: Optional[Dict[str, torch.Tensor]] = None,
                 tokenizer=None, config: Optional[ClipTextConfig] = None) -> None:
        super().__init__()
        if finetune:
            raise NotImplementedError("B200TextEncoder is inference only: finetune must be False")
        if state_dict is None:
            if modelpath is None:
                raise ValueError("give modelpath (a Hugging Face CLIP model) or use B200TextEncoder.from_state_dict")
            if "clip" not in modelpath:
                # the reference also accepts "bert" paths (mld_bert); only the CLIP tower is built here
                raise ValueError(f"Model {modelpath} not supported")                  # mld_clip.py:49
            state_dict, tokenizer, config = _load_hf(modelpath)
        self.latent_dim = latent_dim
        self.tokenizer = tokenizer
        self.text_cfg = config or ClipTextConfig()
        self.name = "clip_hidden" if last_hidden_state else "clip"                    # mld_clip.py:38-44
        self.text_encoded_dim = self.text_cfg.hidden
        self.max_length = self.text_cfg.max_positions
        _register_tree(self, _tower(state_dict))

    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], tokenizer=None,
                        config: Optional[ClipTextConfig] = None, last_hidden_state: bool = False,
                        latent_dim: list = [1, 256]) -> "B200TextEncoder":
        """Build from ``MldTextEncoder`` text-tower keys (an optional ``text_encoder.`` prefix is stripped).
        ``tokenizer``: anything with Hugging Face's ``__call__(texts, padding="max_length", truncation=True,
        max_length=L, return_tensors="pt").input_ids``; only :meth:`forward` needs it."""
        return cls(None, False, last_hidden_state, latent_dim, state_dict=state_dict, tokenizer=tokenizer,
                   config=config)

    def _make_config(self):
        return make_config(num_layers=0, vae="none")                # a handle that holds only the text tower

    def _configure_engine(self, eng):
        eng.text_configure(self.text_cfg.to_c())

    @property
    def pooled(self) -> bool:
        return self.name == "clip"

    def encode_ids(self, ids) -> torch.Tensor:
        """int64 ids [n, L] -> ``[n, 1, projection_dim]`` (clip) or ``[n, L, hidden]`` (clip_hidden) on the module's
        device.  Out-of-range ids raise before anything is launched."""
        c = self.text_cfg
        ids = check_ids(ids, c.vocab_size, c.max_positions)
        eng = self.engine()
        rows, inverse = plan_ids(ids, self.pooled, c.eos_token_id)
        out = eng.text_encode(rows, _lib.TEXT_POOLED if self.pooled else _lib.TEXT_HIDDEN)
        out = out.index_select(0, inverse.to(out.device))
        return out.unsqueeze(1) if self.pooled else out

    def forward(self, texts: List[str]) -> torch.Tensor:
        if self.tokenizer is None:
            raise RuntimeError("no tokenizer: build with modelpath or pass tokenizer=, or call encode_ids(ids)")
        ids = self.tokenizer(texts, padding="max_length", truncation=True, max_length=self.max_length,
                             return_tensors="pt").input_ids                              # mld_clip.py:56-66
        return self.encode_ids(ids[:, :self.max_length])


def _tower(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The text-tower tensors of an ``MldTextEncoder`` state dict; the ``position_ids`` buffer of older
    transformers checkpoints is dropped after checking that it is ``arange``."""
    out = {}
    for k, v in sd.items():
        if k.startswith("text_encoder."):
            k = k[len("text_encoder."):]
        if not k.startswith(TOWER_PREFIXES):
            continue
        if k.endswith("embeddings.position_ids"):
            if not torch.equal(v.reshape(-1).long(), torch.arange(v.numel())):
                raise ValueError(f"{k} is not arange: custom position ids are not supported")
            continue
        out[k] = v.detach().float()
    return out


def _load_hf(modelpath: str):
    """Tokenizer, text-tower weights and config of a Hugging Face CLIP model (needs transformers)."""
    from transformers import AutoModel, AutoTokenizer
    tok = AutoTokenizer.from_pretrained(modelpath)
    model = AutoModel.from_pretrained(modelpath)
    tc = model.config.text_config
    if getattr(tc, "hidden_act", "quick_gelu") != "quick_gelu":
        raise NotImplementedError(f"text tower activation {tc.hidden_act}: only quick_gelu (CLIP) is built")
    cfg = ClipTextConfig(vocab_size=tc.vocab_size, max_positions=tc.max_position_embeddings, hidden=tc.hidden_size,
                         heads=tc.num_attention_heads, layers=tc.num_hidden_layers, ff=tc.intermediate_size,
                         projection_dim=model.config.projection_dim, eos_token_id=tc.eos_token_id,
                         ln_eps=tc.layer_norm_eps)
    sd = {"text_model." + k: v for k, v in model.state_dict().items()
          if k.startswith(("text_model.", "text_projection."))}
    return sd, tok, cfg
