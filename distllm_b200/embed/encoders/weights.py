"""Weight layout handed to ``b2e_encoder_create`` (the order IS the ABI, see include/b2e.h).

BERT (``B2E_ARCH_BERT``), 5 + 12*L device tensors:

    0 word_embeddings [V,H] f32      1 position_embeddings [P,H] f32   2 token_type_embeddings [T,H] f32
    3 embeddings.LayerNorm.weight    4 embeddings.LayerNorm.bias       (f32 [H])
    per layer l, base = 5 + 12*l:
      +0 Wqkv [3H,H] 16-bit (rows: query | key | value)   +1 bqkv [3H] f32
      +2 Wo   [H,H]  16-bit                               +3 bo   [H]  f32
      +4 attention.output.LayerNorm.weight  +5 .bias    (f32)
      +6 W1   [I,H]  16-bit (intermediate.dense)          +7 b1   [I]  f32
      +8 W2   [H,I]  16-bit (output.dense)                +9 b2   [H]  f32
      +10 output.LayerNorm.weight           +11 .bias   (f32)

Names on the right are HF ``BertModel`` state-dict keys (transformers/models/bert/modeling_bert.py).
Matrices keep nn.Linear's [out_features, in_features] layout, which is the K-major B operand the
wgmma GEMM wants, so no transposes are needed.

Every list builder takes ``matrix``: the conversion of ONE checkpoint matrix to its device form.  By default that is
the build's 16-bit storage type (:func:`to_storage`); :func:`nf4_matrix` gives an :class:`Nf4Matrix` instead
(``b2e_encoder_create_nf4``).  The layout steps that follow -- row concatenation, the gate/up interleave, zero
padding -- apply to both forms alike (:func:`cat_rows`, :func:`interleave_gate_up`, :func:`pad_rows`,
:func:`pad_cols`), so an NF4 slot dequantises to exactly the 16-bit slot.
"""

from __future__ import annotations

from typing import Callable
from typing import Mapping
from typing import NamedTuple

import torch

from distllm_b200 import _native


HALF_MAX = 65504.0


def to_storage(t: torch.Tensor, device: torch.device, dtype: torch.dtype) -> torch.Tensor:
    """Checkpoint matrix (fp32 / bf16 / fp16) -> contiguous device tensor of the library build's 16-bit storage
    type.  float16 saturates at +-65504 (weights never get near it; the clamp only keeps a broken checkpoint
    from turning into inf)."""
    x = t.detach().to(device=device, dtype=torch.float32)
    if dtype == torch.float16:
        x = x.clamp(-HALF_MAX, HALF_MAX)
    return x.to(dtype).contiguous()


class Nf4Matrix(NamedTuple):
    """One NF4 weight matrix [N, K] in the device format (embed/encoders/nf4.py: nf4_quantize)."""

    codes: torch.Tensor    # uint8 [N, K/2]
    absmax: torch.Tensor   # fp32 [K/64, N]


Matrix = 'torch.Tensor | Nf4Matrix'
NF4_ZERO = 0x77   # two NF4 codes 7 (0.0): padding, with scale 0


def storage_matrix(device: torch.device, dtype: torch.dtype) -> Callable[[torch.Tensor], torch.Tensor]:
    return lambda t: to_storage(t, device, dtype)


def nf4_matrix(device: torch.device) -> Callable[[torch.Tensor], Nf4Matrix]:
    """Quantise one checkpoint matrix on ``device``: only its fp32 copy and the codes / scales live there."""
    from distllm_b200.embed.encoders.nf4 import nf4_quantize

    def convert(t: torch.Tensor) -> Nf4Matrix:
        return Nf4Matrix(*nf4_quantize(t.detach().to(device=device, dtype=torch.float32)))

    return convert


def cat_rows(mats: list) -> Matrix:
    if isinstance(mats[0], Nf4Matrix):
        return Nf4Matrix(torch.cat([m.codes for m in mats]), torch.cat([m.absmax for m in mats], dim=1))
    return torch.cat(mats)


def row_slice(m: Matrix, start: int, stop: int) -> Matrix:
    if isinstance(m, Nf4Matrix):
        return Nf4Matrix(m.codes[start:stop], m.absmax[:, start:stop])
    return m[start:stop]


def pad_rows(m: Matrix, n: int) -> Matrix:
    """n zero rows below."""
    if isinstance(m, Nf4Matrix):
        codes = torch.full((n, m.codes.shape[1]), NF4_ZERO, dtype=torch.uint8, device=m.codes.device)
        absmax = m.absmax.new_zeros((m.absmax.shape[0], n))
        return Nf4Matrix(torch.cat([m.codes, codes]), torch.cat([m.absmax, absmax], dim=1))
    return torch.cat([m, m.new_zeros((n, m.shape[1]))])


def pad_cols(m: Matrix, n: int) -> Matrix:
    """n zero columns on the right (NF4: whole 64-column blocks)."""
    if isinstance(m, Nf4Matrix):
        if n % 64:
            raise ValueError(f'NF4 column padding {n} is not a multiple of 64')
        codes = torch.full((m.codes.shape[0], n // 2), NF4_ZERO, dtype=torch.uint8, device=m.codes.device)
        absmax = m.absmax.new_zeros((n // 64, m.absmax.shape[1]))
        return Nf4Matrix(torch.cat([m.codes, codes], dim=1), torch.cat([m.absmax, absmax]))
    return torch.cat([m, m.new_zeros((m.shape[0], n))], dim=1)


def device_weight_bytes(weights: list) -> dict[str, int]:
    """Device bytes of a weight list: ``matrix`` (16-bit matrices, or NF4 codes + scales) and ``other`` (fp32
    embedding tables, norms, biases)."""
    matrix = other = 0
    for w in weights:
        if isinstance(w, Nf4Matrix):
            matrix += w.codes.nbytes + w.absmax.nbytes
        elif w.dtype in (torch.float16, torch.bfloat16):
            matrix += w.nbytes
        else:
            other += w.nbytes
    return {'matrix': matrix, 'other': other}


def bert_desc(hf_config) -> _native.ModelDesc:
    """Translate a HF ``BertConfig`` into the C ``B2EModelDesc``; reject what is not built."""
    if getattr(hf_config, 'position_embedding_type', 'absolute') not in (None, 'absolute'):
        raise NotImplementedError('only absolute position embeddings are supported')
    act = getattr(hf_config, 'hidden_act', 'gelu')
    if act != 'gelu':
        raise NotImplementedError(f"hidden_act={act!r}: only erf-GELU ('gelu') is built")
    heads = hf_config.num_attention_heads
    return _native.ModelDesc(
        arch=_native.ARCH_BERT,
        num_layers=hf_config.num_hidden_layers,
        hidden=hf_config.hidden_size,
        heads=heads,
        kv_heads=heads,
        head_dim=hf_config.hidden_size // heads,
        intermediate=hf_config.intermediate_size,
        vocab=hf_config.vocab_size,
        max_pos=hf_config.max_position_embeddings,
        type_vocab=hf_config.type_vocab_size,
        eps=float(hf_config.layer_norm_eps),
        rope_theta=0.0,
        sliding_window=0,
        reserved=0,
    )


def roberta_desc(hf_config) -> _native.ModelDesc:
    """HF ``RobertaConfig`` / ``XLMRobertaConfig`` -> ``B2EModelDesc``: the BERT block and weight layout, with
    ``reserved = pad_token_id + 1`` selecting RoBERTa's position ids (pos = cumsum(m) * m + padding_idx with
    m = ids != padding_idx, transformers/models/xlm_roberta/modeling_xlm_roberta.py:
    create_position_ids_from_input_ids).  The token-type table is read as in BERT, whatever its size."""
    pos_type = getattr(hf_config, 'position_embedding_type', 'absolute')
    if pos_type not in (None, 'absolute'):
        raise NotImplementedError(f'position_embedding_type={pos_type!r}: only absolute position embeddings are '
                                  f'built for RoBERTa / XLM-RoBERTa')
    pad = getattr(hf_config, 'pad_token_id', None)
    if pad is None or pad < 0:
        raise NotImplementedError('RoBERTa / XLM-RoBERTa position ids follow pad_token_id, which this config does '
                                  'not set')
    if pad + 1 >= hf_config.max_position_embeddings:
        raise NotImplementedError(f'pad_token_id={pad} leaves no position row of the '
                                  f'{hf_config.max_position_embeddings}-row table for a token')
    desc = bert_desc(hf_config)
    desc.reserved = int(pad) + 1
    return desc


def roberta_max_length(hf_config) -> int:
    """Longest row RoBERTa positions can index: its last token reads row padding_idx + S of the
    max_position_embeddings-row table (514 -> 512, BGE-M3's 8194 -> 8192)."""
    return hf_config.max_position_embeddings - hf_config.pad_token_id - 1


def bert_weight_list(
    state_dict: Mapping[str, torch.Tensor],
    num_layers: int,
    device: torch.device,
    dtype: torch.dtype = torch.float16,
    matrix: Callable[[torch.Tensor], Matrix] | None = None,
) -> list:
    """HF BertModel state dict -> contiguous device tensors in ABI order."""
    sd = {k[5:] if k.startswith('bert.') else k: v for k, v in state_dict.items()}
    b16 = matrix or storage_matrix(device, dtype)

    def f32(key: str) -> torch.Tensor:
        return sd[key].detach().to(device=device, dtype=torch.float32).contiguous()

    out = [
        f32('embeddings.word_embeddings.weight'),
        f32('embeddings.position_embeddings.weight'),
        f32('embeddings.token_type_embeddings.weight'),
        f32('embeddings.LayerNorm.weight'),
        f32('embeddings.LayerNorm.bias'),
    ]
    for layer in range(num_layers):
        p = f'encoder.layer.{layer}.'
        qkv_w = cat_rows([b16(sd[p + f'attention.self.{n}.weight']) for n in ('query', 'key', 'value')])
        qkv_b = torch.cat([sd[p + f'attention.self.{n}.bias'] for n in ('query', 'key', 'value')])
        out += [
            qkv_w,
            qkv_b.detach().to(device=device, dtype=torch.float32).contiguous(),
            b16(sd[p + 'attention.output.dense.weight']),
            f32(p + 'attention.output.dense.bias'),
            f32(p + 'attention.output.LayerNorm.weight'),
            f32(p + 'attention.output.LayerNorm.bias'),
            b16(sd[p + 'intermediate.dense.weight']),
            f32(p + 'intermediate.dense.bias'),
            b16(sd[p + 'output.dense.weight']),
            f32(p + 'output.dense.bias'),
            f32(p + 'output.LayerNorm.weight'),
            f32(p + 'output.LayerNorm.bias'),
        ]
    return out


def random_bert_state_dict(hf_config, seed: int = 0, device: torch.device | str = 'cpu',
                           std: float | None = None) -> dict[str, torch.Tensor]:
    """Seeded random weights with HF BertModel names/shapes (normal(0, initializer_range),
    LayerNorm weight 1 / bias 0 -- HF's ``_init_weights``), generated directly on ``device``.

    Used for synthetic-weight benchmarking where no checkpoint can be downloaded.
    """
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    std = hf_config.initializer_range if std is None else std
    h, i = hf_config.hidden_size, hf_config.intermediate_size

    def normal(*shape: int) -> torch.Tensor:
        return torch.randn(*shape, generator=gen, device=device, dtype=torch.float32) * std

    sd = {
        'embeddings.word_embeddings.weight': normal(hf_config.vocab_size, h),
        'embeddings.position_embeddings.weight': normal(hf_config.max_position_embeddings, h),
        'embeddings.token_type_embeddings.weight': normal(hf_config.type_vocab_size, h),
        'embeddings.LayerNorm.weight': torch.ones(h, device=device),
        'embeddings.LayerNorm.bias': torch.zeros(h, device=device),
    }
    for layer in range(hf_config.num_hidden_layers):
        p = f'encoder.layer.{layer}.'
        for name, (o, k) in {
            'attention.self.query': (h, h),
            'attention.self.key': (h, h),
            'attention.self.value': (h, h),
            'attention.output.dense': (h, h),
            'intermediate.dense': (i, h),
            'output.dense': (h, i),
        }.items():
            sd[p + name + '.weight'] = normal(o, k)
            # HF zero-initialises biases; small non-zero values exercise the bias epilogues
            sd[p + name + '.bias'] = normal(o)
        for name in ('attention.output.LayerNorm', 'output.LayerNorm'):
            sd[p + name + '.weight'] = torch.ones(h, device=device)
            sd[p + name + '.bias'] = torch.zeros(h, device=device)
    return sd


# --------------------------------------------------------------------------- ESM-2
# ``B2E_ARCH_ESM2``, 3 + 12*L device tensors (HF EsmModel / EsmForMaskedLM names, ``esm.`` prefix
# stripped; transformers/models/esm/modeling_esm.py):
#
#     0 embeddings.word_embeddings [V,H] f32
#     1 encoder.emb_layer_norm_after.weight   2 .bias                         (f32 [H])
#     per layer l, base = 3 + 12*l (pre-LayerNorm blocks):
#       +0 attention.LayerNorm.weight  +1 .bias                 (LN before self-attention)
#       +2 Wqkv [3H,H] 16-bit (query | key | value)               +3 bqkv [3H] f32
#       +4 attention.output.dense.weight [H,H] 16-bit             +5 .bias
#       +6 LayerNorm.weight            +7 .bias                 (LN before the feed-forward)
#       +8 intermediate.dense.weight [I,H] 16-bit                 +9 .bias
#       +10 output.dense.weight [H,I] 16-bit                      +11 .bias
#
# ``B2EModelDesc.reserved`` carries ``mask_token_id + 1`` when ``token_dropout`` is on (0 = off).


def esm_desc(hf_config) -> _native.ModelDesc:
    """Translate a HF ``EsmConfig`` (ESM-2 family) into the C ``B2EModelDesc``."""
    if getattr(hf_config, 'position_embedding_type', 'absolute') != 'rotary':
        raise NotImplementedError('only rotary ESM-2 checkpoints are supported')
    if getattr(hf_config, 'emb_layer_norm_before', False):
        raise NotImplementedError('emb_layer_norm_before=True (ESM-1b style) is not built')
    heads = hf_config.num_attention_heads
    token_dropout = bool(getattr(hf_config, 'token_dropout', False))
    return _native.ModelDesc(
        arch=_native.ARCH_ESM2,
        num_layers=hf_config.num_hidden_layers,
        hidden=hf_config.hidden_size,
        heads=heads,
        kv_heads=heads,
        head_dim=hf_config.hidden_size // heads,
        intermediate=hf_config.intermediate_size,
        vocab=hf_config.vocab_size,
        max_pos=hf_config.max_position_embeddings,
        type_vocab=0,
        eps=float(hf_config.layer_norm_eps),
        rope_theta=10000.0,
        sliding_window=0,
        reserved=(int(hf_config.mask_token_id) + 1) if token_dropout else 0,
    )


def esm_weight_list(
    state_dict: Mapping[str, torch.Tensor],
    num_layers: int,
    device: torch.device,
    dtype: torch.dtype = torch.float16,
) -> list[torch.Tensor]:
    """HF EsmModel/EsmForMaskedLM state dict -> contiguous device tensors in ABI order."""
    sd = {k[4:] if k.startswith('esm.') else k: v for k, v in state_dict.items()}

    def f32(key: str) -> torch.Tensor:
        return sd[key].detach().to(device=device, dtype=torch.float32).contiguous()

    def b16(t: torch.Tensor) -> torch.Tensor:
        return to_storage(t, device, dtype)

    out = [
        f32('embeddings.word_embeddings.weight'),
        f32('encoder.emb_layer_norm_after.weight'),
        f32('encoder.emb_layer_norm_after.bias'),
    ]
    for layer in range(num_layers):
        p = f'encoder.layer.{layer}.'
        qkv_w = torch.cat([sd[p + f'attention.self.{n}.weight'] for n in ('query', 'key', 'value')])
        qkv_b = torch.cat([sd[p + f'attention.self.{n}.bias'] for n in ('query', 'key', 'value')])
        out += [
            f32(p + 'attention.LayerNorm.weight'),
            f32(p + 'attention.LayerNorm.bias'),
            b16(qkv_w),
            qkv_b.detach().to(device=device, dtype=torch.float32).contiguous(),
            b16(sd[p + 'attention.output.dense.weight']),
            f32(p + 'attention.output.dense.bias'),
            f32(p + 'LayerNorm.weight'),
            f32(p + 'LayerNorm.bias'),
            b16(sd[p + 'intermediate.dense.weight']),
            f32(p + 'intermediate.dense.bias'),
            b16(sd[p + 'output.dense.weight']),
            f32(p + 'output.dense.bias'),
        ]
    return out


def random_esm_state_dict(hf_config, seed: int = 0, device: torch.device | str = 'cpu',
                          std: float | None = None) -> dict[str, torch.Tensor]:
    """Seeded random ESM-2 weights with HF EsmModel names (no ``esm.`` prefix)."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    std = getattr(hf_config, 'initializer_range', 0.02) if std is None else std
    h, i = hf_config.hidden_size, hf_config.intermediate_size

    def normal(*shape: int) -> torch.Tensor:
        return torch.randn(*shape, generator=gen, device=device, dtype=torch.float32) * std

    def ln(prefix: str, sd: dict) -> None:
        # non-trivial LayerNorm parameters so that both gamma and beta paths are exercised
        sd[prefix + '.weight'] = 1.0 + normal(h)
        sd[prefix + '.bias'] = normal(h)

    sd: dict[str, torch.Tensor] = {'embeddings.word_embeddings.weight': normal(hf_config.vocab_size, h)}
    ln('encoder.emb_layer_norm_after', sd)
    for layer in range(hf_config.num_hidden_layers):
        p = f'encoder.layer.{layer}.'
        for name, (o, k) in {
            'attention.self.query': (h, h),
            'attention.self.key': (h, h),
            'attention.self.value': (h, h),
            'attention.output.dense': (h, h),
            'intermediate.dense': (i, h),
            'output.dense': (h, i),
        }.items():
            sd[p + name + '.weight'] = normal(o, k)
            sd[p + name + '.bias'] = normal(o)
        ln(p + 'attention.LayerNorm', sd)
        ln(p + 'LayerNorm', sd)
    return sd


# ------------------------------------------------------------------------------ Mistral family
# Mistral (``B2E_ARCH_MISTRAL``), 2 + 6*L device tensors (no biases anywhere):
#
#     0 embed_tokens [V,H] f32          1 norm.weight [H] f32 (final RMSNorm)
#     per layer l, base = 2 + 6*l:
#       +0 input_layernorm.weight [H] f32
#       +1 Wqkv [(heads + 2*kv_heads)*d, H] 16-bit (rows: q_proj | k_proj | v_proj)
#       +2 Wo   [H, heads*d] 16-bit
#       +3 post_attention_layernorm.weight [H] f32
#       +4 Wgu  [2I, H] 16-bit: gate_proj and up_proj interleaved in blocks of 64 rows
#               (rows [128t, 128t+64) = gate rows [64t, 64t+64); rows [128t+64, 128t+128) = up rows
#               [64t, 64t+64)), so that one GEMM tile holds gate and up of the same 64 outputs and
#               the SwiGLU product is taken in the epilogue
#       +5 Wd   [H, I] 16-bit (down_proj)
#
# Names are HF ``MistralModel`` state-dict keys (transformers/models/mistral/modeling_mistral.py).

GATE_UP_BLOCK = 64


def rope_theta_of(hf_config) -> float:
    params = getattr(hf_config, 'rope_parameters', None)
    if params and 'rope_theta' in params:
        return float(params['rope_theta'])
    return float(getattr(hf_config, 'rope_theta', 10000.0))


def mistral_desc(hf_config) -> _native.ModelDesc:
    """Translate a HF ``MistralConfig`` into the C ``B2EModelDesc``."""
    heads = hf_config.num_attention_heads
    head_dim = getattr(hf_config, 'head_dim', None) or hf_config.hidden_size // heads
    if getattr(hf_config, 'hidden_act', 'silu') != 'silu':
        raise NotImplementedError(f'hidden_act={hf_config.hidden_act!r}: only SwiGLU (silu) is built')
    window = getattr(hf_config, 'sliding_window', None)
    return _native.ModelDesc(
        arch=_native.ARCH_MISTRAL,
        num_layers=hf_config.num_hidden_layers,
        hidden=hf_config.hidden_size,
        heads=heads,
        kv_heads=hf_config.num_key_value_heads,
        head_dim=head_dim,
        intermediate=hf_config.intermediate_size,
        vocab=hf_config.vocab_size,
        max_pos=hf_config.max_position_embeddings,
        type_vocab=0,
        eps=float(hf_config.rms_norm_eps),
        rope_theta=rope_theta_of(hf_config),
        sliding_window=int(window) if window else 0,
        reserved=0,
    )


def interleave_gate_up(gate: Matrix, up: Matrix) -> Matrix:
    """[I,H], [I,H] -> [2I,H] in the block-interleaved row order the SwiGLU epilogue expects."""
    if isinstance(gate, Nf4Matrix):
        return Nf4Matrix(interleave_gate_up(gate.codes, up.codes),
                         interleave_gate_up(gate.absmax.t(), up.absmax.t()).t().contiguous())
    i, h = gate.shape
    if i % GATE_UP_BLOCK:
        raise ValueError(f'intermediate_size {i} must be a multiple of {GATE_UP_BLOCK}')
    g = gate.reshape(i // GATE_UP_BLOCK, 1, GATE_UP_BLOCK, h)
    u = up.reshape(i // GATE_UP_BLOCK, 1, GATE_UP_BLOCK, h)
    return torch.cat([g, u], dim=1).reshape(2 * i, h)


def mistral_weight_list(
    state_dict: Mapping[str, torch.Tensor],
    num_layers: int,
    device: torch.device,
    dtype: torch.dtype = torch.float16,
    matrix: Callable[[torch.Tensor], Matrix] | None = None,
) -> list:
    """HF MistralModel (or ...ForCausalLM) state dict -> contiguous device tensors in ABI order."""
    sd = {k[6:] if k.startswith('model.') else k: v for k, v in state_dict.items()}
    b16 = matrix or storage_matrix(device, dtype)

    def f32(key: str) -> torch.Tensor:
        return sd[key].detach().to(device=device, dtype=torch.float32).contiguous()

    out = [f32('embed_tokens.weight'), f32('norm.weight')]
    for layer in range(num_layers):
        p = f'layers.{layer}.'
        out += [
            f32(p + 'input_layernorm.weight'),
            cat_rows([b16(sd[p + f'self_attn.{n}_proj.weight']) for n in ('q', 'k', 'v')]),
            b16(sd[p + 'self_attn.o_proj.weight']),
            f32(p + 'post_attention_layernorm.weight'),
            interleave_gate_up(b16(sd[p + 'mlp.gate_proj.weight']), b16(sd[p + 'mlp.up_proj.weight'])),
            b16(sd[p + 'mlp.down_proj.weight']),
        ]
    return out


def random_mistral_state_dict(hf_config, seed: int = 0, device: torch.device | str = 'cpu',
                              std: float | None = None,
                              dtype: torch.dtype = torch.float32) -> dict[str, torch.Tensor]:
    """Seeded random Mistral weights with HF MistralModel names (no ``model.`` prefix)."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    std = getattr(hf_config, 'initializer_range', 0.02) if std is None else std
    h, i = hf_config.hidden_size, hf_config.intermediate_size
    heads, kv = hf_config.num_attention_heads, hf_config.num_key_value_heads
    d = getattr(hf_config, 'head_dim', None) or h // heads

    def normal(*shape: int) -> torch.Tensor:
        return (torch.randn(*shape, generator=gen, device=device, dtype=torch.float32) * std).to(dtype)

    sd: dict[str, torch.Tensor] = {'embed_tokens.weight': normal(hf_config.vocab_size, h)}
    sd['norm.weight'] = (1.0 + normal(h).float()).to(dtype)
    for layer in range(hf_config.num_hidden_layers):
        p = f'layers.{layer}.'
        sd[p + 'self_attn.q_proj.weight'] = normal(heads * d, h)
        sd[p + 'self_attn.k_proj.weight'] = normal(kv * d, h)
        sd[p + 'self_attn.v_proj.weight'] = normal(kv * d, h)
        sd[p + 'self_attn.o_proj.weight'] = normal(h, heads * d)
        sd[p + 'mlp.gate_proj.weight'] = normal(i, h)
        sd[p + 'mlp.up_proj.weight'] = normal(i, h)
        sd[p + 'mlp.down_proj.weight'] = normal(h, i)
        sd[p + 'input_layernorm.weight'] = (1.0 + normal(h).float()).to(dtype)
        sd[p + 'post_attention_layernorm.weight'] = (1.0 + normal(h).float()).to(dtype)
    return sd


# ------------------------------------------------------------------------------ Qwen3
# Qwen3 (``B2E_ARCH_QWEN3``), 2 + 8*L device tensors: Mistral's slots (HF ``Qwen3Model`` uses the same names), and
# per layer two more:
#       +6 self_attn.q_norm.weight [128] f32 (RMSNorm of every q head, before rotary)
#       +7 self_attn.k_norm.weight [128] f32 (RMSNorm of every k head, before rotary)
# Names are HF ``Qwen3Model`` state-dict keys (transformers/models/qwen3/modeling_qwen3.py).


def qwen3_desc(hf_config) -> _native.ModelDesc:
    """Translate a HF ``Qwen3Config`` into the C ``B2EModelDesc``; reject what is not built."""
    if getattr(hf_config, 'attention_bias', False):
        raise NotImplementedError('Qwen3: attention_bias=True is not built (built: q/k/v/o projections without '
                                  'bias, as every Qwen3-Embedding checkpoint)')
    types = list(getattr(hf_config, 'layer_types', None) or [])
    if 'sliding_attention' in types:
        raise NotImplementedError(f'Qwen3: sliding_attention layers (use_sliding_window) are not built (built: '
                                  f'full causal attention in every layer; layer_types {types})')
    params = getattr(hf_config, 'rope_parameters', None) or {}
    if params.get('rope_type', 'default') != 'default':
        raise NotImplementedError(f'Qwen3: rope_type {params["rope_type"]!r} is not built (built: default rotary)')
    if getattr(hf_config, 'hidden_act', 'silu') != 'silu':
        raise NotImplementedError(f'Qwen3: hidden_act={hf_config.hidden_act!r} is not built (built: SwiGLU, silu)')
    desc = mistral_desc(hf_config)
    desc.arch = _native.ARCH_QWEN3
    desc.sliding_window = 0
    return desc


def qwen3_weight_list(
    state_dict: Mapping[str, torch.Tensor],
    num_layers: int,
    device: torch.device,
    dtype: torch.dtype = torch.float16,
    matrix: Callable[[torch.Tensor], Matrix] | None = None,
) -> list:
    """HF Qwen3Model (or ...ForCausalLM, ``model.`` prefix) state dict -> contiguous device tensors in ABI order."""
    sd = {k[6:] if k.startswith('model.') else k: v for k, v in state_dict.items()}
    mistral = mistral_weight_list(sd, num_layers, device, dtype, matrix)
    out = mistral[:2]
    for layer in range(num_layers):
        p = f'layers.{layer}.self_attn.'
        out += mistral[2 + 6 * layer:8 + 6 * layer]
        out += [sd[p + n].detach().to(device=device, dtype=torch.float32).contiguous()
                for n in ('q_norm.weight', 'k_norm.weight')]
    return out


def random_qwen3_state_dict(hf_config, seed: int = 0, device: torch.device | str = 'cpu',
                            std: float | None = None,
                            dtype: torch.dtype = torch.float32) -> dict[str, torch.Tensor]:
    """Seeded random Qwen3 weights with HF Qwen3Model names (no ``model.`` prefix): Mistral's, then q_norm / k_norm
    gains 1 + N(0, std) from a second generator (HF initialises them to ones, which would hide a missing or swapped
    gain)."""
    sd = random_mistral_state_dict(hf_config, seed=seed, device=device, std=std, dtype=dtype)
    gen = torch.Generator(device=device)
    gen.manual_seed(seed + 1)
    std = getattr(hf_config, 'initializer_range', 0.02) if std is None else std
    d = hf_config.head_dim
    for layer in range(hf_config.num_hidden_layers):
        for n in ('q_norm', 'k_norm'):
            g = 1.0 + torch.randn(d, generator=gen, device=device, dtype=torch.float32) * std
            sd[f'layers.{layer}.self_attn.{n}.weight'] = g.to(dtype)
    return sd


# ------------------------------------------------------------------------------ ModernBERT
# ModernBERT (``B2E_ARCH_MODERNBERT``), 5 + 8*L device tensors (HF ``ModernBertModel`` names, ``model.`` prefix
# stripped; transformers/models/modernbert/modeling_modernbert.py):
#
#     0 embeddings.tok_embeddings [V,H] f32      1 embeddings.norm.weight   2 embeddings.norm.bias
#     3 final_norm.weight                         4 final_norm.bias           (f32 [H]; absent biases -> zeros)
#     per layer l, base = 5 + 8*l (pre-LayerNorm blocks; layer 0 has no attn_norm: slots hold ones / zeros):
#       +0 attn_norm.weight   +1 attn_norm.bias
#       +2 attn.Wqkv [3H,H] 16-bit (rows: q | k | v, heads of 64)      +3 attn.Wo [H,H] 16-bit
#       +4 mlp_norm.weight    +5 mlp_norm.bias
#       +6 mlp.Wi [2I,H] 16-bit: the ``input`` half (rows [0,I), the one that goes through GELU) and the ``gate``
#          half (rows [I,2I)) interleaved in blocks of 64 rows, so that the GeGLU product is taken in the GEMM
#          epilogue (``interleave_gate_up(input, gate)``)
#       +7 mlp.Wo [H,I] 16-bit


def modernbert_layer_pattern(hf_config) -> int:
    """``global_every``: layer l is a full-attention layer iff l % global_every == 0 (the published checkpoints:
    3).  Other ``layer_types`` layouts are not built."""
    types = list(hf_config.layer_types)
    for every in range(1, len(types) + 1):
        if all((t == 'full_attention') == (i % every == 0) for i, t in enumerate(types)):
            return every
    raise NotImplementedError(f'layer_types {types} is not "full attention every n-th layer"')


def modernbert_padded_intermediate(intermediate_size: int) -> int:
    """The gated GEMM epilogue pairs 128 input with 128 gate columns: intermediate_size is zero-padded to the
    next multiple of 128 (ModernBERT-large: 2624 -> 2688; gelu(0) * 0 = 0 feeds zero columns of mlp.Wo)."""
    return (intermediate_size + 127) // 128 * 128


def modernbert_desc(hf_config) -> _native.ModelDesc:
    """Translate a HF ``ModernBertConfig`` into the C ``B2EModelDesc``; reject what is not built."""
    if getattr(hf_config, 'hidden_activation', 'gelu') != 'gelu':
        raise NotImplementedError(f'hidden_activation={hf_config.hidden_activation!r}: only erf-GELU is built')
    if getattr(hf_config, 'attention_bias', False) or getattr(hf_config, 'mlp_bias', False):
        raise NotImplementedError('ModernBERT checkpoints with Linear biases are not built')
    heads = hf_config.num_attention_heads
    params = hf_config.rope_parameters
    for kind in ('full_attention', 'sliding_attention'):
        if params[kind].get('rope_type', 'default') != 'default':
            raise NotImplementedError(f'rope_type {params[kind]["rope_type"]!r} is not built')
    return _native.ModelDesc(
        arch=_native.ARCH_MODERNBERT,
        num_layers=hf_config.num_hidden_layers,
        hidden=hf_config.hidden_size,
        heads=heads,
        kv_heads=heads,
        head_dim=hf_config.hidden_size // heads,
        intermediate=modernbert_padded_intermediate(hf_config.intermediate_size),
        vocab=hf_config.vocab_size,
        max_pos=hf_config.max_position_embeddings,
        type_vocab=0,
        eps=float(hf_config.norm_eps),
        rope_theta=float(params['full_attention']['rope_theta']),
        sliding_window=int(hf_config.sliding_window),     # = local_attention // 2: |i - j| <= sliding_window
        reserved=0,
        rope_theta_local=float(params['sliding_attention']['rope_theta']),
        global_every=modernbert_layer_pattern(hf_config),
    )


def modernbert_weight_list(
    state_dict: Mapping[str, torch.Tensor],
    num_layers: int,
    device: torch.device,
    dtype: torch.dtype = torch.bfloat16,
    matrix: Callable[[torch.Tensor], Matrix] | None = None,
) -> list:
    """HF ModernBertModel (or ...ForMaskedLM) state dict -> contiguous device tensors in ABI order."""
    sd = {k[6:] if k.startswith('model.') else k: v for k, v in state_dict.items()}
    hidden = sd['embeddings.norm.weight'].shape[0]
    b16 = matrix or storage_matrix(device, dtype)

    def f32(key: str, default: float | None = None) -> torch.Tensor:
        if key not in sd:
            if default is None:
                raise KeyError(key)
            return torch.full((hidden,), default, dtype=torch.float32, device=device)
        return sd[key].detach().to(device=device, dtype=torch.float32).contiguous()

    out = [
        f32('embeddings.tok_embeddings.weight'),
        f32('embeddings.norm.weight'), f32('embeddings.norm.bias', 0.0),
        f32('final_norm.weight'), f32('final_norm.bias', 0.0),
    ]
    for layer in range(num_layers):
        p = f'layers.{layer}.'
        wi = b16(sd[p + 'mlp.Wi.weight'])
        wo_mlp = b16(sd[p + 'mlp.Wo.weight'])
        inter = sd[p + 'mlp.Wi.weight'].shape[0] // 2
        pad = modernbert_padded_intermediate(inter) - inter
        w_in, w_gate = row_slice(wi, 0, inter), row_slice(wi, inter, 2 * inter)
        if pad:
            w_in, w_gate = pad_rows(w_in, pad), pad_rows(w_gate, pad)
            wo_mlp = pad_cols(wo_mlp, pad)
        out += [
            f32(p + 'attn_norm.weight', 1.0), f32(p + 'attn_norm.bias', 0.0),   # layer 0: Identity (unused)
            b16(sd[p + 'attn.Wqkv.weight']),
            b16(sd[p + 'attn.Wo.weight']),
            f32(p + 'mlp_norm.weight'), f32(p + 'mlp_norm.bias', 0.0),
            interleave_gate_up(w_in, w_gate),
            wo_mlp,
        ]
    return out


def random_modernbert_state_dict(hf_config, seed: int = 0, device: torch.device | str = 'cpu',
                                 std: float | None = None) -> dict[str, torch.Tensor]:
    """Seeded random ModernBERT weights with HF ModernBertModel names (no biases, as the published models)."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    std = getattr(hf_config, 'initializer_range', 0.02) if std is None else std
    h, i = hf_config.hidden_size, hf_config.intermediate_size

    def normal(*shape: int) -> torch.Tensor:
        return torch.randn(*shape, generator=gen, device=device, dtype=torch.float32) * std

    sd: dict[str, torch.Tensor] = {'embeddings.tok_embeddings.weight': normal(hf_config.vocab_size, h)}
    sd['embeddings.norm.weight'] = 1.0 + normal(h)
    sd['final_norm.weight'] = 1.0 + normal(h)
    for layer in range(hf_config.num_hidden_layers):
        p = f'layers.{layer}.'
        if layer > 0:
            sd[p + 'attn_norm.weight'] = 1.0 + normal(h)
        sd[p + 'attn.Wqkv.weight'] = normal(3 * h, h)
        sd[p + 'attn.Wo.weight'] = normal(h, h)
        sd[p + 'mlp_norm.weight'] = 1.0 + normal(h)
        sd[p + 'mlp.Wi.weight'] = normal(2 * i, h)
        sd[p + 'mlp.Wo.weight'] = normal(h, i)
    return sd


# ------------------------------------------------------------------------------ LoRA under NF4 storage
# ``b2e_encoder_create_nf4_lora`` takes per GEMM slot (4 per layer, the absmax order: Wqkv, Wo, W1, W2) the factors of
# the slot's low-rank term, delta(slot) = B_cat . A_cat:
#
#   A_cat  16-bit [round_up(R, 128), K]: the A rows of the slot's adapted modules stacked (Q | K | V, gate | up), zero
#          rows below; ModernBERT's mlp.Wo gets the zero columns of its padded K
#   B_cat  16-bit [N, round_up(R, 64)]: module i's s_i B_i in the rows of its outputs and the columns of its A rows
#          (s folded in fp32 before the storage rounding), then the slot's row layout -- Q | K | V, the gate/up
#          interleave of interleave_gate_up, ModernBERT's padded Wi halves -- and zero columns on the right
#
# so that the NF4 GEMM's tail k-blocks add U . B_cat^T with U = X . A_cat^T, R = the sum of the modules' ranks.


def _lora_slots(arch: str, hf_config, layer: int) -> list[tuple[list[tuple[str, int]], int, str]]:
    """The four GEMM slots of ``layer``: ([(module, output rows)], K, row layout)."""
    h = hf_config.hidden_size
    if arch == 'bert':
        p, i = f'encoder.layer.{layer}.', hf_config.intermediate_size
        return [([(p + f'attention.self.{n}', h) for n in ('query', 'key', 'value')], h, 'cat'),
                ([(p + 'attention.output.dense', h)], h, 'cat'),
                ([(p + 'intermediate.dense', i)], h, 'cat'),
                ([(p + 'output.dense', h)], i, 'cat')]
    if arch in ('mistral', 'qwen3'):
        p, i = f'layers.{layer}.', hf_config.intermediate_size
        heads, kv = hf_config.num_attention_heads, hf_config.num_key_value_heads
        d = getattr(hf_config, 'head_dim', None) or h // heads
        return [([(p + 'self_attn.q_proj', heads * d), (p + 'self_attn.k_proj', kv * d),
                  (p + 'self_attn.v_proj', kv * d)], h, 'cat'),
                ([(p + 'self_attn.o_proj', h)], heads * d, 'cat'),
                ([(p + 'mlp.gate_proj', i), (p + 'mlp.up_proj', i)], h, 'gate_up'),
                ([(p + 'mlp.down_proj', h)], i, 'cat')]
    if arch == 'modernbert':
        p, i = f'layers.{layer}.', hf_config.intermediate_size
        return [([(p + 'attn.Wqkv', 3 * h)], h, 'cat'),
                ([(p + 'attn.Wo', h)], h, 'cat'),
                ([(p + 'mlp.Wi', 2 * i)], h, 'geglu'),
                ([(p + 'mlp.Wo', h)], i, 'pad_k')]
    raise NotImplementedError(f'{arch}: no quantised configuration, so no unmerged LoRA path')


_MODEL_PREFIX = {'bert': 'bert.', 'mistral': 'model.', 'qwen3': 'model.', 'modernbert': 'model.'}


def lora_slot_factors(arch: str, hf_config, lora: Mapping[str, tuple[torch.Tensor, torch.Tensor, float]],
                      device: torch.device, dtype: torch.dtype) -> list[tuple[torch.Tensor, torch.Tensor, int] | None]:
    """LoRA modules ``{module: (A [r, in], B [out, r], s)}`` (state-dict names) -> per slot (A_cat, B_cat, R) with
    R = round_up(sum of ranks, 64), or None for a slot without an adapter; in ``dtype`` on ``device``."""
    pre = _MODEL_PREFIX[arch]
    lo = {k[len(pre):] if k.startswith(pre) else k: v for k, v in lora.items()}
    used = set()
    out: list = []
    for layer in range(hf_config.num_hidden_layers):
        for modules, k, layout in _lora_slots(arch, hf_config, layer):
            present = [(m, rows) for m, rows in modules if m in lo]
            if not present:
                out.append(None)
                continue
            used.update(m for m, _ in present)
            r = sum(lo[m][0].shape[0] for m, _ in present)
            r64, r128 = (r + 63) // 64 * 64, (r + 127) // 128 * 128
            a_cat = torch.zeros((r128, k), dtype=torch.float32, device=device)
            b_full = torch.zeros((sum(rows for _, rows in modules), r64), dtype=torch.float32, device=device)
            row = col = 0
            for m, rows in modules:
                if m in lo:
                    a, b, s = lo[m]
                    ri = a.shape[0]
                    a_cat[col:col + ri] = a.to(device=device, dtype=torch.float32)
                    b_full[row:row + rows, col:col + ri] = s * b.to(device=device, dtype=torch.float32)
                    col += ri
                row += rows
            if layout == 'gate_up':
                half = b_full.shape[0] // 2
                b_full = interleave_gate_up(b_full[:half], b_full[half:])
            elif layout == 'geglu':
                half = b_full.shape[0] // 2
                pad = modernbert_padded_intermediate(half) - half
                b_full = interleave_gate_up(pad_rows(b_full[:half], pad), pad_rows(b_full[half:], pad))
            elif layout == 'pad_k':
                a_cat = pad_cols(a_cat, modernbert_padded_intermediate(k) - k)
            out.append((to_storage(a_cat, device, dtype), to_storage(b_full, device, dtype), r64))
    missing = sorted(set(lo) - used)
    if missing:
        raise ValueError(f'LoRA modules outside the GEMM slots of {arch}: {missing[:8]}')
    return out


# ------------------------------------------------------------------------------ ESM C
# ESM C (``B2E_ARCH_ESMC``), 3 + 10*L device tensors, from the esm package's state dict (esm/models/esmc.py,
# esm/layers/blocks.py, attention.py; ``esmc_{300m,600m}_2024_12_v0.pth``), no Linear biases:
#
#     0 embed.weight [V,H] f32          1 transformer.norm.weight [H] f32    2 zeros [H] (the final norm has no bias)
#     per layer l, base = 3 + 10*l, prefix transformer.blocks.l.:
#       +0 attn.layernorm_qkv.0.weight  +1 .bias       (f32 [H]: LayerNorm before attention)
#       +2 attn.layernorm_qkv.1.weight [3H,H] 16-bit (rows: q | k | v)
#       +3 attn.q_ln.weight  +4 attn.k_ln.weight        (f32 [H]: LayerNorm over the whole q / k row, no bias)
#       +5 attn.out_proj.weight [H,H] 16-bit / s
#       +6 ffn.0.weight  +7 ffn.0.bias                  (f32 [H]: LayerNorm before the FFN)
#       +8 ffn.1.weight [2I,H] 16-bit: rows [0,I) gate (silu), [I,2I) up, interleaved as interleave_gate_up
#       +9 ffn.3.weight [H,I] 16-bit / s
#
# s = sqrt(L / 36) is the blocks' residual scale (x + f(x) / s); it is folded into out_proj and ffn.3 in fp32 before
# the storage rounding (1 for esmc-600m: those weights are untouched).  head_dim is 64, eps 1e-5, rotary base 10000,
# halves convention; none of these is visible in the weights.

ESMC_HEAD_DIM = 64
ESMC_EPS = 1e-5
ESMC_MAX_POS = 2048      # the reference's tokenizer.model_max_length (distllm/embed/encoders/esmc.py:82)
ESMC_LAYER_KEYS = (
    ('attn.layernorm_qkv.0.weight', 'H'), ('attn.layernorm_qkv.0.bias', 'H'), ('attn.layernorm_qkv.1.weight', '3H,H'),
    ('attn.q_ln.weight', 'H'), ('attn.k_ln.weight', 'H'), ('attn.out_proj.weight', 'H,H'),
    ('ffn.0.weight', 'H'), ('ffn.0.bias', 'H'), ('ffn.1.weight', '2I,H'), ('ffn.3.weight', 'H,I'),
)


class EsmcConfig(NamedTuple):
    """The shape of an ESM C checkpoint, read from its tensor shapes (:func:`esmc_config`)."""

    hidden_size: int
    num_hidden_layers: int
    intermediate_size: int
    vocab_size: int
    max_position_embeddings: int = ESMC_MAX_POS


def esmc_residual_scale(num_layers: int) -> float:
    """s = sqrt(L / 36) of esm/layers/blocks.py: each block adds its attention and FFN outputs divided by s."""
    return (num_layers / 36) ** 0.5


def esmc_config(state_dict: Mapping[str, torch.Tensor]) -> EsmcConfig:
    """Shape inference and validation of an ESM C state dict on tensor shapes alone (nothing moves to a device).
    Every expected key must be there with its shape; any other key except ``sequence_head.*`` (the LM head, never
    used) is an error that names it."""
    shapes = {k: tuple(v.shape) for k, v in state_dict.items() if not k.startswith('sequence_head.')}
    if 'embed.weight' not in shapes or len(shapes['embed.weight']) != 2:
        raise ValueError('ESMC checkpoint: no embed.weight [V, H]')
    v, h = shapes['embed.weight']
    layers = 0
    while f'transformer.blocks.{layers}.attn.layernorm_qkv.1.weight' in shapes:
        layers += 1
    if layers == 0:
        raise ValueError('ESMC checkpoint: no transformer.blocks.0')
    w1 = shapes.get('transformer.blocks.0.ffn.1.weight', ())
    if len(w1) != 2 or w1[0] % 2:
        raise ValueError(f'ESMC checkpoint: transformer.blocks.0.ffn.1.weight has shape {w1}, expected [2I, {h}]')
    i = w1[0] // 2
    dims = {'H': h, '3H': 3 * h, '2I': 2 * i, 'I': i}
    want = {'embed.weight': (v, h), 'transformer.norm.weight': (h,)}
    for layer in range(layers):
        for key, shape in ESMC_LAYER_KEYS:
            want[f'transformer.blocks.{layer}.{key}'] = tuple(dims[d] for d in shape.split(','))
    unexpected = sorted(set(shapes) - set(want))
    if unexpected:
        raise ValueError(f'ESMC checkpoint: unexpected keys {unexpected[:8]} (built: the esm package ESMC layout '
                         f'without Linear biases and with full-width q_ln / k_ln)')
    for key, shape in want.items():
        if key not in shapes:
            raise ValueError(f'ESMC checkpoint: missing {key}')
        if shapes[key] != shape:
            raise ValueError(f'ESMC checkpoint: {key} has shape {list(shapes[key])}, expected {list(shape)}')
    return EsmcConfig(hidden_size=h, num_hidden_layers=layers, intermediate_size=i, vocab_size=v)


def esmc_desc(config: EsmcConfig) -> _native.ModelDesc:
    """Translate an :class:`EsmcConfig` into the C ``B2EModelDesc`` (b2e_check_model decides what is built)."""
    h = config.hidden_size
    return _native.ModelDesc(
        arch=_native.ARCH_ESMC,
        num_layers=config.num_hidden_layers,
        hidden=h,
        heads=h // ESMC_HEAD_DIM,
        kv_heads=h // ESMC_HEAD_DIM,
        head_dim=ESMC_HEAD_DIM,
        intermediate=config.intermediate_size,
        vocab=config.vocab_size,
        max_pos=config.max_position_embeddings,
        type_vocab=0,
        eps=ESMC_EPS,
        rope_theta=10000.0,
        sliding_window=0,
        reserved=0,
    )


def esmc_weight_list(
    state_dict: Mapping[str, torch.Tensor],
    num_layers: int,
    device: torch.device,
    dtype: torch.dtype = torch.float16,
    matrix: Callable[[torch.Tensor], Matrix] | None = None,
) -> list:
    """ESM C state dict -> contiguous device tensors in ABI order, with 1/s folded into out_proj and ffn.3."""
    sd = state_dict
    b16 = matrix or storage_matrix(device, dtype)
    s = esmc_residual_scale(num_layers)

    def f32(key: str) -> torch.Tensor:
        return sd[key].detach().to(device=device, dtype=torch.float32).contiguous()

    def scaled(key: str) -> Matrix:
        w = sd[key].detach().to(device=device, dtype=torch.float32)
        return b16(w if s == 1.0 else w / s)

    norm = f32('transformer.norm.weight')
    out = [f32('embed.weight'), norm, torch.zeros_like(norm)]
    for layer in range(num_layers):
        p = f'transformer.blocks.{layer}.'
        w1 = b16(sd[p + 'ffn.1.weight'])
        i = sd[p + 'ffn.1.weight'].shape[0] // 2
        out += [
            f32(p + 'attn.layernorm_qkv.0.weight'), f32(p + 'attn.layernorm_qkv.0.bias'),
            b16(sd[p + 'attn.layernorm_qkv.1.weight']),
            f32(p + 'attn.q_ln.weight'), f32(p + 'attn.k_ln.weight'),
            scaled(p + 'attn.out_proj.weight'),
            f32(p + 'ffn.0.weight'), f32(p + 'ffn.0.bias'),
            interleave_gate_up(row_slice(w1, 0, i), row_slice(w1, i, 2 * i)),
            scaled(p + 'ffn.3.weight'),
        ]
    return out


def random_esmc_state_dict(hidden: int, num_layers: int, intermediate: int, seed: int = 0,
                           device: torch.device | str = 'cpu', std: float = 0.02,
                           vocab: int = 64) -> dict[str, torch.Tensor]:
    """Seeded random ESM C weights with the checkpoint's key names and shapes, including a small ``sequence_head``
    (which the loader skips).  Every norm gain is 1 + N(0, std) and every norm bias N(0, std), so that a missing or
    swapped norm parameter changes the result."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    h, i = hidden, intermediate

    def normal(*shape: int) -> torch.Tensor:
        return torch.randn(*shape, generator=gen, device=device, dtype=torch.float32) * std

    sd: dict[str, torch.Tensor] = {'embed.weight': normal(vocab, h), 'transformer.norm.weight': 1.0 + normal(h)}
    for layer in range(num_layers):
        p = f'transformer.blocks.{layer}.'
        sd[p + 'attn.layernorm_qkv.0.weight'] = 1.0 + normal(h)
        sd[p + 'attn.layernorm_qkv.0.bias'] = normal(h)
        sd[p + 'attn.layernorm_qkv.1.weight'] = normal(3 * h, h)
        sd[p + 'attn.q_ln.weight'] = 1.0 + normal(h)
        sd[p + 'attn.k_ln.weight'] = 1.0 + normal(h)
        sd[p + 'attn.out_proj.weight'] = normal(h, h)
        sd[p + 'ffn.0.weight'] = 1.0 + normal(h)
        sd[p + 'ffn.0.bias'] = normal(h)
        sd[p + 'ffn.1.weight'] = normal(2 * i, h)
        sd[p + 'ffn.3.weight'] = normal(h, i)
    sd['sequence_head.0.weight'] = normal(h, h)
    sd['sequence_head.0.bias'] = normal(h)
    sd['sequence_head.3.weight'] = normal(vocab, h)
    return sd
