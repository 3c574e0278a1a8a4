"""fp32 CPU restatement of the forward pass the reference triggers for Qwen3 checkpoints (Qwen3-Embedding).

distllm's AutoEncoder.encode (distllm/embed/encoders/auto.py:119-138) calls
``AutoModel(**batch, output_hidden_states=True)`` and returns ``hidden_states[-1]``; for a ``Qwen3Model`` that is
the output of the final RMSNorm.  Restated from transformers 5.5, transformers/models/qwen3/modeling_qwen3.py:

    RMSNorm      :50-64    x * rsqrt(mean(x^2) + eps), statistics in fp32, then * weight
    MLP          :70-83    down(silu(gate(x)) * up(x)), no biases
    rotary       :86-181   cos/sin of pos * theta^(-2i/d), halves convention (rotate_half)
    attention    :222-291  q/k/v projections without bias; q_norm / k_norm (RMSNorm over head_dim, one gain
                           vector each) on every q and k head (:248-249, :263-264) BEFORE rotary (:268);
                           grouped-query, scores scaled by d^-0.5, causal + key-padding mask, o_proj
    blocks       :294-335  pre-norm: x += attn(norm(x)); x += mlp(norm(x))
    model        :357-439  embed_tokens, position_ids = arange(S) for every row, final norm

It is oracle/mistral.py's block with the two head norms; the helpers are that file's.  The checkpoints this
project accepts have no sliding-window layers (weights.qwen3_desc rejects them), so every layer is fully causal.
Plain torch ops on CPU in fp32; the state dict uses HF parameter names.  TEST INFRASTRUCTURE ONLY.
"""

from __future__ import annotations

from typing import Mapping

import torch
import torch.nn.functional as F  # noqa: N812

from oracle.mistral import _rms
from oracle.mistral import _rotate
from oracle.mistral import _sd
from oracle.mistral import rope_theta_of
from oracle.mistral import visibility


@torch.no_grad()
def qwen3_forward(
    state_dict: Mapping[str, torch.Tensor],
    hf_config,
    input_ids: torch.Tensor,
    attention_mask: torch.Tensor,
    return_all: bool = False,
):
    """Last hidden state ``[B,S,H]`` fp32 (== ``Qwen3Model(...).last_hidden_state``).

    ``return_all``: list over l = 1..L of ``final_norm(residual stream after l layers)`` -- what a model truncated
    to l layers would return (the per-layer drift report compares against these)."""
    sd = _sd(state_dict)
    eps = hf_config.rms_norm_eps
    heads, kv_heads = hf_config.num_attention_heads, hf_config.num_key_value_heads
    b, s = input_ids.shape
    d = hf_config.head_dim
    theta = rope_theta_of(hf_config)
    vis = visibility(attention_mask, None)
    dead = ~vis.any(-1, keepdim=True)  # [B,1,S,1] query rows without a visible key (left padding)

    x = sd['embed_tokens.weight'][input_ids]
    states = []
    for layer in range(hf_config.num_hidden_layers):
        p = f'layers.{layer}.'
        y = _rms(x, sd[p + 'input_layernorm.weight'], eps)
        q = _rms(F.linear(y, sd[p + 'self_attn.q_proj.weight']).view(b, s, heads, d),
                 sd[p + 'self_attn.q_norm.weight'], eps).transpose(1, 2)
        k = _rms(F.linear(y, sd[p + 'self_attn.k_proj.weight']).view(b, s, kv_heads, d),
                 sd[p + 'self_attn.k_norm.weight'], eps).transpose(1, 2)
        v = F.linear(y, sd[p + 'self_attn.v_proj.weight']).view(b, s, kv_heads, d).transpose(1, 2)
        q, k = _rotate(q, theta), _rotate(k, theta)
        k = k.repeat_interleave(heads // kv_heads, dim=1)
        v = v.repeat_interleave(heads // kv_heads, dim=1)
        scores = (q @ k.transpose(-1, -2)) * d ** -0.5
        scores = scores.masked_fill(~vis, float('-inf'))
        prob = torch.softmax(scores, dim=-1).masked_fill(dead, 0.0)
        ctx = (prob @ v).transpose(1, 2).reshape(b, s, heads * d)
        x = x + F.linear(ctx, sd[p + 'self_attn.o_proj.weight'])
        y = _rms(x, sd[p + 'post_attention_layernorm.weight'], eps)
        gate = F.linear(y, sd[p + 'mlp.gate_proj.weight'])
        up = F.linear(y, sd[p + 'mlp.up_proj.weight'])
        x = x + F.linear(F.silu(gate) * up, sd[p + 'mlp.down_proj.weight'])
        if return_all:
            states.append(_rms(x, sd['norm.weight'], eps))
    return states if return_all else _rms(x, sd['norm.weight'], eps)
