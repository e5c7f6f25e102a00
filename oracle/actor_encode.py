"""CPU restatement of ActorVae's encoder (TEST INFRASTRUCTURE ONLY), in the style of ``oracle/mld_oracle.py``
and built from its primitives.

``ActorAgnosticEncoder.forward`` (mld/models/architectures/actor_vae.py:120-170) in eval mode, up to the
distribution parameters.  It runs in the state dict's dtype, so a float64 copy of the state dict gives the float64
reference.  Pinned against the reference's own ``ActorVae.encode`` through tests/golden/vae_actor_encode.npz (see
``oracle/make_golden_actor_encode.py``).
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from oracle.mld_oracle import SD, Tensor, VaeCfg, encoder_layer_post, lengths_to_mask, linear


def plain_encoder(x: Tensor, sd: SD, p: str, num_layers: int, nhead: int,
                  kpm: Optional[Tensor] = None, act: str = "gelu") -> Tensor:
    """torch's nn.TransformerEncoder without a final norm (actor_vae.py:111-119): post-norm
    layers in sequence, no skip connections."""
    for i in range(num_layers):
        x = encoder_layer_post(x, sd, f"{p}layers.{i}.", nhead, kpm, act)
    return x


def actor_encode(sd: SD, cfg: VaeCfg, feats: Tensor, lengths: Sequence[int]):
    """feats [B, T, nfeats] -> (mu, logvar), each [1, B, d]: ``final[0]`` / ``final[1]`` of the encoder
    (actor_vae.py:169).  ``dist = Normal(mu[0], logvar[0].exp().pow(0.5))`` and the rsample of
    ``sample_from_distribution`` (:238-258) are torch RNG and left to the caller."""
    B, T, _ = feats.shape
    mask = lengths_to_mask(lengths, T)
    e = "encoder."
    feats = feats.to(sd[e + "skel_embedding.weight"].dtype)
    x = linear(feats, sd[e + "skel_embedding.weight"], sd[e + "skel_embedding.bias"]).permute(1, 0, 2)   # :136-139
    tokens = torch.stack((sd[e + "mu_token"], sd[e + "logvar_token"]))[:, None, :].expand(2, B, -1)       # :144-149
    keep = torch.cat((torch.ones(B, 2, dtype=torch.bool), mask), 1)                                       # :150-153
    xseq = torch.cat((tokens, x), 0) + sd[e + "sequence_pos_encoding.pe"][: T + 2]                        # :165
    final = plain_encoder(xseq, sd, e + "seqTransEncoder.", cfg.num_layers, cfg.num_heads, ~keep,
                          cfg.activation)                                                                 # :166
    return final[0:1], final[1:2]
