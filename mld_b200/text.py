"""``B200TextEncoder``: drop-in replacement for the reference's text encoder, selectable through the YAML
``target:`` factory (``instantiate_from_config``, mld/config.py:106-121):

    text_encoder.target:  mld_b200.text.B200TextEncoder     (was mld.models.architectures.mld_clip.MldTextEncoder)

Same ctor kwargs (``modelpath, finetune, last_hidden_state, latent_dim``), same ``state_dict`` keys of the text
tower, same ``forward(texts) -> Tensor``: ``[n, 1, projection_dim]`` (``clip``, the shipped config),
``[n, L, hidden]`` (``clip_hidden``) or, for a ``"bert"`` model path (DistilBERT or BERT), ``[n, L, hidden]``
(``bert``: every position of the right-padded batch, padding positions included).  The tokenizer stays on the host
(Hugging Face's); everything after the int64 ids runs in ``libmldb200.so`` (``mldb_text_encode`` /
``mldb_bert_encode``).  Exact savings are applied to the host ids before upload: every distinct id row (with its
length, for BERT) is encoded once (the B identical "" rows of classifier-free guidance), and in ``clip`` mode only the
first ``max(eos_pos) + 1`` columns are sent - under the causal mask no later token reaches a pooled row.  Inference
only.
"""
from __future__ import annotations

import os
from dataclasses import asdict, dataclass
from typing import Dict, List, Optional, Union

import torch

from . import _lib
from .modules import _EngineModule, _register_tree
from .engine import make_config

TOWER_PREFIXES = ("text_model.text_model.", "text_model.text_projection.")
BERT_PREFIXES = ("text_model.",)                 # the whole AutoModel: DistilBertModel / BertModel


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


@dataclass
class BertTextConfig:
    """The BERT tower's shape (``mldb_bert_config``); defaults are distilbert-base-uncased.  ``family``:
    ``"distilbert"`` or ``"bert"``; ``type_vocab`` counts BERT's token-type rows (unused for DistilBERT)."""
    family: str = "distilbert"
    vocab_size: int = 30522
    max_positions: int = 512
    type_vocab: int = 2
    hidden: int = 768
    heads: int = 12
    layers: int = 6
    ff: int = 3072
    ln_eps: float = 1e-12

    def to_c(self) -> _lib.MldbBertConfig:
        c = _lib.default_bert_config()
        for k, v in asdict(self).items():
            setattr(c, k, {"distilbert": _lib.BERT_DISTILBERT, "bert": _lib.BERT_BERT}[v] if k == "family" else v)
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


def mask_lengths(mask, n: int, L: int) -> torch.Tensor:
    """Real tokens per row of a right-padded attention mask [n, L] (each row: ones, then zeros, at least one one);
    None stands for all ones.  Any other mask raises ValueError."""
    if mask is None:
        return torch.full((n,), L, dtype=torch.int64)
    m = torch.as_tensor(mask).to("cpu")
    if tuple(m.shape) != (n, L):
        raise ValueError(f"attention_mask must be [{n}, {L}], got {tuple(m.shape)}")
    if not bool(((m == 0) | (m == 1)).all()):
        raise ValueError("attention_mask must hold 0 and 1 only")
    m = m.to(torch.int64)
    lengths = m.sum(1)
    if not torch.equal(m, (torch.arange(L)[None] < lengths[:, None]).to(torch.int64)) or int(lengths.min()) < 1:
        raise ValueError("attention_mask rows must be right-padded prefixes of ones, each with at least one token")
    return lengths


def plan_bert_rows(ids: torch.Tensor, lengths: torch.Tensor):
    """``(rows, row_lengths, inverse)``: the distinct (id row, length) pairs, and ``rows[inverse]`` the original
    rows; a row's encoding depends on nothing else, so encoding the distinct ones and gathering is exact."""
    keyed, inverse = torch.unique(torch.cat([ids, lengths[:, None]], 1), dim=0, return_inverse=True)
    return keyed[:, :-1].contiguous(), keyed[:, -1].contiguous(), inverse


class B200TextEncoder(_EngineModule):
    """``MldTextEncoder`` (mld/models/architectures/mld_clip.py:13-97): CLIP text models, and DistilBERT / BERT
    models (``name == "bert"``)."""
    _prefix = "text_encoder."

    def __init__(self, modelpath: Optional[str] = None, finetune: bool = False, last_hidden_state: bool = False,
                 latent_dim: list = [1, 256], *, state_dict: Optional[Dict[str, torch.Tensor]] = None,
                 tokenizer=None, config: Union[ClipTextConfig, BertTextConfig, None] = None) -> None:
        super().__init__()
        if finetune:
            raise NotImplementedError("B200TextEncoder is inference only: finetune must be False")
        if state_dict is None:
            if modelpath is None:
                raise ValueError("give modelpath (a Hugging Face CLIP or BERT model) or use "
                                 "B200TextEncoder.from_state_dict")
            if "clip" in modelpath:                                                    # mld_clip.py:38-49
                state_dict, tokenizer, config = _load_hf(modelpath)
            elif "bert" in modelpath:
                state_dict, tokenizer, config = _load_hf_bert(modelpath)
            else:
                raise ValueError(f"Model {modelpath} not supported")
        self.latent_dim = latent_dim
        self.tokenizer = tokenizer
        self.text_cfg = config or ClipTextConfig()
        if isinstance(self.text_cfg, BertTextConfig):
            self.name = "bert"                                   # last_hidden_state is ignored, as in the reference
        else:
            self.name = "clip_hidden" if last_hidden_state else "clip"
        self.text_encoded_dim = self.text_cfg.hidden
        self.max_length = self.text_cfg.max_positions
        _register_tree(self, _tower(state_dict, BERT_PREFIXES if self.name == "bert" else TOWER_PREFIXES))

    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], tokenizer=None,
                        config: Union[ClipTextConfig, BertTextConfig, None] = None, last_hidden_state: bool = False,
                        latent_dim: list = [1, 256]) -> "B200TextEncoder":
        """Build from ``MldTextEncoder`` text-tower keys (an optional ``text_encoder.`` prefix is stripped); a
        :class:`BertTextConfig` selects the BERT tower (keys ``text_model.`` + the Hugging Face model's).
        ``tokenizer``: anything with Hugging Face's ``__call__`` as :meth:`forward` makes it (CLIP:
        ``padding="max_length", truncation=True, max_length=L, return_tensors="pt"`` -> ``.input_ids``; BERT:
        ``return_tensors="pt", padding=True`` -> ``["input_ids"]``, ``["attention_mask"]``, optional
        ``["token_type_ids"]``); only :meth:`forward` needs it."""
        return cls(None, False, last_hidden_state, latent_dim, state_dict=state_dict, tokenizer=tokenizer,
                   config=config)

    def _make_config(self):
        return make_config(num_layers=0, vae="none")                # a handle that holds only the text tower

    def _configure_engine(self, eng):
        if self.name == "bert":
            eng.bert_configure(self.text_cfg.to_c())
        else:
            eng.text_configure(self.text_cfg.to_c())

    @property
    def pooled(self) -> bool:
        return self.name == "clip"

    def encode_ids(self, ids, attention_mask=None) -> torch.Tensor:
        """int64 ids [n, L] -> ``[n, 1, projection_dim]`` (clip) or ``[n, L, hidden]`` (clip_hidden, bert) on the
        module's device.  ``attention_mask`` (bert only; None: all ones) must be right-padded.  Out-of-range ids, a
        bad mask and L > max_positions raise before anything is launched."""
        c = self.text_cfg
        ids = check_ids(ids, c.vocab_size, c.max_positions)
        if self.name == "bert":
            lengths = mask_lengths(attention_mask, *ids.shape)
            eng = self.engine()
            rows, row_lengths, inverse = plan_bert_rows(ids, lengths)
            out = eng.bert_encode(rows, row_lengths)
            return out.index_select(0, inverse.to(out.device))
        if attention_mask is not None:
            raise ValueError("attention_mask applies to the bert tower only (CLIP runs unmasked, as the reference)")
        eng = self.engine()
        rows, inverse = plan_ids(ids, self.pooled, c.eos_token_id)
        out = eng.text_encode(rows, _lib.TEXT_POOLED if self.pooled else _lib.TEXT_HIDDEN)
        out = out.index_select(0, inverse.to(out.device))
        return out.unsqueeze(1) if self.pooled else out

    def forward(self, texts: List[str]) -> torch.Tensor:
        if self.tokenizer is None:
            raise RuntimeError("no tokenizer: build with modelpath or pass tokenizer=, or call encode_ids(ids)")
        if self.name == "bert":
            enc = self.tokenizer(texts, return_tensors="pt", padding=True)             # mld_clip.py:65-68
            types = enc.get("token_type_ids")
            if types is not None and bool(torch.as_tensor(types).any()):
                raise ValueError("token_type_ids must be zero (single sentences)")
            return self.encode_ids(enc["input_ids"], enc.get("attention_mask"))
        ids = self.tokenizer(texts, padding="max_length", truncation=True, max_length=self.max_length,
                             return_tensors="pt").input_ids                              # mld_clip.py:56-66
        return self.encode_ids(ids[:, :self.max_length])


def _tower(sd: Dict[str, torch.Tensor], prefixes=TOWER_PREFIXES) -> Dict[str, torch.Tensor]:
    """The text-tower tensors (keys under ``prefixes``) of an ``MldTextEncoder`` state dict; the ``position_ids``
    buffer of older transformers checkpoints is dropped after checking that it is ``arange``."""
    out = {}
    for k, v in sd.items():
        if k.startswith("text_encoder."):
            k = k[len("text_encoder."):]
        if not k.startswith(prefixes):
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


def bert_config_from_hf(hf) -> BertTextConfig:
    """The :class:`BertTextConfig` of a transformers ``DistilBertConfig`` / ``BertConfig``; NotImplementedError for
    anything this tower does not build."""
    mt = getattr(hf, "model_type", None)
    if mt == "distilbert":
        if hf.sinusoidal_pos_embds:
            raise NotImplementedError("DistilBERT with sinusoidal_pos_embds=True: only learned positions are built")
        if hf.activation != "gelu":
            raise NotImplementedError(f"DistilBERT activation {hf.activation}: only gelu (exact) is built")
        return BertTextConfig(family="distilbert", vocab_size=hf.vocab_size, max_positions=hf.max_position_embeddings,
                              hidden=hf.dim, heads=hf.n_heads, layers=hf.n_layers, ff=hf.hidden_dim,
                              ln_eps=1e-12)                                 # DistilBERT's LayerNorms: eps 1e-12 fixed
    if mt == "bert":
        if hf.hidden_act != "gelu":
            raise NotImplementedError(f"BERT hidden_act {hf.hidden_act}: only gelu (exact) is built")
        if getattr(hf, "position_embedding_type", "absolute") != "absolute":
            raise NotImplementedError(f"BERT position_embedding_type {hf.position_embedding_type}: only absolute")
        if getattr(hf, "is_decoder", False) or getattr(hf, "add_cross_attention", False):
            raise NotImplementedError("decoder BERT configs are not built: the text encoder is an encoder")
        return BertTextConfig(family="bert", vocab_size=hf.vocab_size, max_positions=hf.max_position_embeddings,
                              type_vocab=hf.type_vocab_size, hidden=hf.hidden_size, heads=hf.num_attention_heads,
                              layers=hf.num_hidden_layers, ff=hf.intermediate_size, ln_eps=hf.layer_norm_eps)
    raise NotImplementedError(f"model_type {mt!r}: only distilbert and bert are built")


def _load_hf_bert(modelpath: str):
    """Tokenizer, weights and config of a locally saved Hugging Face DistilBERT / BERT model (needs transformers)."""
    if not os.path.isdir(modelpath):
        raise ValueError(f"{modelpath} is not a directory: give a locally saved Hugging Face model")
    from transformers import AutoConfig, AutoModel, AutoTokenizer
    cfg = bert_config_from_hf(AutoConfig.from_pretrained(modelpath, local_files_only=True))
    tok = AutoTokenizer.from_pretrained(modelpath, local_files_only=True)
    model = AutoModel.from_pretrained(modelpath, local_files_only=True)
    return {"text_model." + k: v for k, v in model.state_dict().items()}, tok, cfg
