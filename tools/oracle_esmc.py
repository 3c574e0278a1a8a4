"""fp32 restatement of the ESM C forward pass (esmc-300m / esmc-600m), the reference the native ESMC trunk is tested
against.  TEST INFRASTRUCTURE ONLY.

Source: the published ``esm`` package (EvolutionaryScale, v3.1): esm/models/esmc.py (ESMC.forward: embed, the
transformer stack, ``ESMCOutput.embeddings`` = the stack's final LayerNorm), esm/layers/blocks.py
(UnifiedTransformerBlock: x + attn(x) / s, x + ffn(x) / s with s = sqrt(L / 36); the FFN is LayerNorm, one Linear to
2I, SwiGLU = silu(first half) * second half, Linear back), esm/layers/attention.py (MultiHeadAttention: LayerNorm +
one q | k | v Linear, q_ln / k_ln = LayerNorm over the whole d_model-wide q / k row without bias, rotary, scaled
dot-product attention with the key-padding mask, out_proj) and esm/layers/rotary.py (halves convention, base 10000,
positions 0..S-1).  The package is not installed here, so parity with it is NOT pinned: this module restates it, and
the loader (embed/encoders/weights.py: esmc_config) refuses any checkpoint whose keys or shapes differ from the layout
restated here.  head_dim 64, eps 1e-5 and the SwiGLU half order are fixed, as the weights cannot show them.
"""

from __future__ import annotations

import math
from typing import Mapping

import torch
import torch.nn.functional as F  # noqa: N812

HEAD_DIM = 64
EPS = 1e-5
THETA = 10000.0


def rotary_tables(s: int, d: int = HEAD_DIM, theta: float = THETA) -> tuple[torch.Tensor, torch.Tensor]:
    """cos / sin [s, d/2] at positions 0..s-1: angle(p, i) = p / theta^(2i/d)."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float32) / d))
    ang = torch.outer(torch.arange(s, dtype=torch.float32), inv_freq)
    return ang.cos(), ang.sin()


def rotate(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """Halves rotation of x [B, S, heads, d] with tables [S, d/2]."""
    half = x.shape[-1] // 2
    x1, x2 = x[..., :half], x[..., half:]
    c, s = cos[None, :, None, :], sin[None, :, None, :]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1)


def num_layers(sd: Mapping[str, torch.Tensor]) -> int:
    n = 0
    while f'transformer.blocks.{n}.attn.layernorm_qkv.1.weight' in sd:
        n += 1
    return n


@torch.no_grad()
def esmc_forward(sd: Mapping[str, torch.Tensor], input_ids: torch.Tensor, attention_mask: torch.Tensor,
                 layers: int | None = None, every_depth: bool = False) -> torch.Tensor | list[torch.Tensor]:
    """``ESMCOutput.embeddings`` [B, S, H] in fp32: the first ``layers`` blocks (all by default) and the final norm;
    with ``every_depth`` the list of the final norm after each block.
    ``attention_mask`` is the key-padding mask (ESMC.forward: input_ids != <pad>).  Runs on input_ids' device."""
    dev = input_ids.device
    sd = {k: v.detach().to(dev, torch.float32) for k, v in sd.items() if not k.startswith('sequence_head.')}
    n = num_layers(sd)
    s = math.sqrt(n / 36)
    x = sd['embed.weight'][input_ids]
    b, seq, h = x.shape
    heads = h // HEAD_DIM
    cos, sin = (t.to(dev) for t in rotary_tables(seq))
    bias = torch.zeros(b, 1, 1, seq, device=dev)
    bias.masked_fill_(attention_mask.to(dev)[:, None, None, :] == 0, float('-inf'))
    states = []
    for layer in range(n if layers is None else layers):
        p = f'transformer.blocks.{layer}.'
        y = F.layer_norm(x, (h,), sd[p + 'attn.layernorm_qkv.0.weight'], sd[p + 'attn.layernorm_qkv.0.bias'], EPS)
        q, k, v = (y @ sd[p + 'attn.layernorm_qkv.1.weight'].T).split(h, dim=-1)
        q = F.layer_norm(q, (h,), sd[p + 'attn.q_ln.weight'], None, EPS)
        k = F.layer_norm(k, (h,), sd[p + 'attn.k_ln.weight'], None, EPS)
        q = rotate(q.reshape(b, seq, heads, HEAD_DIM), cos, sin).transpose(1, 2)
        k = rotate(k.reshape(b, seq, heads, HEAD_DIM), cos, sin).transpose(1, 2)
        v = v.reshape(b, seq, heads, HEAD_DIM).transpose(1, 2)
        att = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(HEAD_DIM) + bias, dim=-1)
        att = torch.nan_to_num(att)   # a fully padded row attends to nothing (its values are unspecified anyway)
        ctx = (att @ v).transpose(1, 2).reshape(b, seq, h)
        x = x + (ctx @ sd[p + 'attn.out_proj.weight'].T) / s
        y = F.layer_norm(x, (h,), sd[p + 'ffn.0.weight'], sd[p + 'ffn.0.bias'], EPS)
        gate, up = (y @ sd[p + 'ffn.1.weight'].T).chunk(2, dim=-1)
        x = x + ((F.silu(gate) * up) @ sd[p + 'ffn.3.weight'].T) / s
        if every_depth:
            states.append(F.layer_norm(x, (h,), sd['transformer.norm.weight'], None, EPS))
    return states if every_depth else F.layer_norm(x, (h,), sd['transformer.norm.weight'], None, EPS)
