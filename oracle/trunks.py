"""Each encoder family's forward pass as the list of steps HF's modules define, run on a set of blocks.

Written from transformers/models/{bert,esm,mistral,qwen3,modernbert}, not from csrc/b2e_api.cu: one function per
family reads the HF state dict, builds every linear layer's weight from the HF tensors itself (q | k | v rows, the
64-row gate/up and input/gate interleave, ModernBERT's zero-padded intermediate width) and calls the blocks in the
order the HF forward pass runs them:

    blocks.embed(ids, mask, types)                      -> (16-bit rows or None, fp32 residual stream or None)
    blocks.linear(x, weights, bias, epi, slot)          -> one GEMM; weights: the HF matrices of the slot and how
                                                           they stack (see ``Linear``)
    blocks.rotary(qkv, layer)                           in place
    blocks.attention(qkv, heads, kv_heads, d, window, causal)
    blocks.norm(kind, xres, add, resid, gamma, beta, out_dtype)
                                                        kind 'post_ln': LayerNorm(add + resid); 'add_ln' / 'add_rms':
                                                        xres += add in place, then LayerNorm / RMSNorm of xres

Two block sets run the same list: ``TorchBlocks`` (fp32 torch on the CPU, checked against the oracles' forward
passes by tests/test_trunks_cpu.py) and the library's own verified kernels (tests/test_gpu_trunks_exact.py).  Rows
are whatever token layout the block set keeps; ``run`` returns the final norm of every depth 1..L (``every_depth``)
or of the last, for each requested output type.  TEST INFRASTRUCTURE ONLY.
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Mapping

import torch
import torch.nn.functional as F  # noqa: N812

GATE_UP_BLOCK = 64
EPI_BIAS, EPI_BIAS_GELU, EPI_SWIGLU, EPI_GEGLU = 'bias', 'bias_gelu', 'swiglu', 'geglu'


@dataclass
class Linear:
    """One GEMM's weight as HF tensors: ``names`` stacked by rows, or (``layout`` 'gate_up') the two halves interleaved
    in blocks of 64 rows; ``pad_rows`` zero rows under each half, ``pad_cols`` zero columns on the right."""

    names: tuple[str, ...]
    layout: str = 'cat'
    pad_rows: int = 0
    pad_cols: int = 0
    split: tuple[int, int] | None = None   # one HF tensor holding both halves: (rows of the first, of the second)


def interleave(first: torch.Tensor, second: torch.Tensor) -> torch.Tensor:
    """Rows [128t, 128t + 64) = first[64t, 64t + 64), rows [128t + 64, 128t + 128) = second[64t, 64t + 64)."""
    i, k = first.shape
    blocks = torch.stack([first.reshape(i // GATE_UP_BLOCK, GATE_UP_BLOCK, k),
                          second.reshape(i // GATE_UP_BLOCK, GATE_UP_BLOCK, k)], dim=1)
    return blocks.reshape(2 * i, k)


def build_weight(lin: Linear, mats: list[torch.Tensor]) -> torch.Tensor:
    """The slot's [N, K] weight from its HF matrices, each already in the block set's form (same dtype)."""
    if lin.layout == 'cat':
        w = torch.cat(mats)
    else:
        first, second = mats if lin.split is None else (mats[0][:lin.split[0]], mats[0][lin.split[0]:])
        if lin.pad_rows:
            first = torch.cat([first, first.new_zeros(lin.pad_rows, first.shape[1])])
            second = torch.cat([second, second.new_zeros(lin.pad_rows, second.shape[1])])
        w = interleave(first, second)
    if lin.pad_cols:
        w = torch.cat([w, w.new_zeros(w.shape[0], lin.pad_cols)], dim=1)
    return w.contiguous()


def _strip(state_dict: Mapping[str, torch.Tensor], prefix: str) -> dict[str, torch.Tensor]:
    return {(k[len(prefix):] if k.startswith(prefix) else k): v for k, v in state_dict.items()}


class Run:
    """Final norms collected per depth."""

    def __init__(self, out_dtypes):
        self.out_dtypes = tuple(out_dtypes)
        self.depths: list[dict] = []

    def add(self, make) -> None:
        self.depths.append({dt: make(dt) for dt in self.out_dtypes})


# ------------------------------------------------------------------------------------------------------ BERT
@torch.no_grad()
def bert(sd, cfg, blocks, ids, mask, types, out_dtypes=(torch.float32,), every_depth=False):
    """modeling_bert.py: BertEmbeddings (word + position + token type, LayerNorm), then per layer BertSelfAttention
    (q | k | v with bias), BertSelfOutput (dense, LayerNorm(dense + input)), BertIntermediate (erf GELU), BertOutput
    (dense, LayerNorm(dense + attention output))."""
    sd = _strip(sd, 'bert.')
    eps, heads, h = cfg.layer_norm_eps, cfg.num_attention_heads, cfg.hidden_size
    d = h // heads
    run = Run(out_dtypes)
    hidden, _ = blocks.embed(ids, mask, types)
    n_layers = cfg.num_hidden_layers
    for l in range(n_layers):
        p = f'encoder.layer.{l}.'
        sa = p + 'attention.self.'
        qkv = blocks.linear(hidden, Linear((sa + 'query.weight', sa + 'key.weight', sa + 'value.weight')),
                            torch.cat([sd[sa + n + '.bias'] for n in ('query', 'key', 'value')]), EPI_BIAS, (l, 0))
        ctx = blocks.attention(qkv, heads, heads, d, 0, False)
        tmp = blocks.linear(ctx, Linear((p + 'attention.output.dense.weight',)), sd[p + 'attention.output.dense.bias'],
                            EPI_BIAS, (l, 1))
        hidden = blocks.norm('post_ln', None, tmp, hidden, sd[p + 'attention.output.LayerNorm.weight'],
                             sd[p + 'attention.output.LayerNorm.bias'], eps, None)
        inter = blocks.linear(hidden, Linear((p + 'intermediate.dense.weight',)), sd[p + 'intermediate.dense.bias'],
                              EPI_BIAS_GELU, (l, 2))
        tmp = blocks.linear(inter, Linear((p + 'output.dense.weight',)), sd[p + 'output.dense.bias'], EPI_BIAS, (l, 3))
        g, b = sd[p + 'output.LayerNorm.weight'], sd[p + 'output.LayerNorm.bias']
        if every_depth or l == n_layers - 1:
            run.add(lambda dt: blocks.norm('post_ln', None, tmp, hidden, g, b, eps, dt))
        if l + 1 < n_layers:
            hidden = blocks.norm('post_ln', None, tmp, hidden, g, b, eps, None)
    return run.depths


# --------------------------------------------------------------------------------------------- pre-norm tail
def _final(blocks, run, kind, xres, tmp, g, b, eps):
    """The final norm over (residual stream + last block output) on a copy of the stream, so that the next layer's
    own norm still folds ``tmp`` in."""
    run.add(lambda dt: blocks.norm(kind, xres.clone(), tmp, None, g, b, eps, dt))


# ------------------------------------------------------------------------------------------------------ ESM-2
@torch.no_grad()
def esm(sd, cfg, blocks, ids, mask, types=None, out_dtypes=(torch.float32,), every_depth=False):
    """modeling_esm.py: EsmEmbeddings (token dropout), then per layer EsmAttention (LayerNorm, q | k | v with bias,
    rotary on q and k, dense), EsmLayer's LayerNorm before EsmIntermediate (erf GELU) and EsmOutput, and
    emb_layer_norm_after over the residual stream."""
    sd = _strip(sd, 'esm.')
    eps, heads, h = cfg.layer_norm_eps, cfg.num_attention_heads, cfg.hidden_size
    d = h // heads
    run = Run(out_dtypes)
    _, xres = blocks.embed(ids, mask, None)
    n_layers = cfg.num_hidden_layers
    tmp = None
    for l in range(n_layers):
        p = f'encoder.layer.{l}.'
        sa = p + 'attention.self.'
        hidden = blocks.norm('add_ln', xres, tmp, None, sd[p + 'attention.LayerNorm.weight'],
                             sd[p + 'attention.LayerNorm.bias'], eps, None)
        qkv = blocks.linear(hidden, Linear((sa + 'query.weight', sa + 'key.weight', sa + 'value.weight')),
                            torch.cat([sd[sa + n + '.bias'] for n in ('query', 'key', 'value')]), EPI_BIAS, (l, 0))
        blocks.rotary(qkv, l)
        ctx = blocks.attention(qkv, heads, heads, d, 0, False)
        tmp = blocks.linear(ctx, Linear((p + 'attention.output.dense.weight',)), sd[p + 'attention.output.dense.bias'],
                            EPI_BIAS, (l, 1))
        hidden = blocks.norm('add_ln', xres, tmp, None, sd[p + 'LayerNorm.weight'], sd[p + 'LayerNorm.bias'], eps, None)
        inter = blocks.linear(hidden, Linear((p + 'intermediate.dense.weight',)), sd[p + 'intermediate.dense.bias'],
                              EPI_BIAS_GELU, (l, 2))
        tmp = blocks.linear(inter, Linear((p + 'output.dense.weight',)), sd[p + 'output.dense.bias'], EPI_BIAS, (l, 3))
        if every_depth or l == n_layers - 1:
            _final(blocks, run, 'add_ln', xres, tmp, sd['encoder.emb_layer_norm_after.weight'],
                   sd['encoder.emb_layer_norm_after.bias'], eps)
    return run.depths


# ------------------------------------------------------------------------------------------- Mistral / Qwen3
@torch.no_grad()
def mistral(sd, cfg, blocks, ids, mask, types=None, out_dtypes=(torch.float32,), every_depth=False):
    """modeling_mistral.py / modeling_qwen3.py: embed_tokens, then per layer input_layernorm, q | k | v (no bias;
    Qwen3: q_norm / k_norm of every head, inside the rotary block), rotary, grouped-query causal attention within
    ``sliding_window``, o_proj, post_attention_layernorm, silu(gate) * up, down_proj; the final norm."""
    sd = _strip(sd, 'model.')
    eps, heads, kv, h = cfg.rms_norm_eps, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.hidden_size
    d = getattr(cfg, 'head_dim', None) or h // heads
    window = getattr(cfg, 'sliding_window', None) or 0
    run = Run(out_dtypes)
    _, xres = blocks.embed(ids, mask, None)
    n_layers = cfg.num_hidden_layers
    tmp = None
    for l in range(n_layers):
        p = f'layers.{l}.'
        sa = p + 'self_attn.'
        hidden = blocks.norm('add_rms', xres, tmp, None, sd[p + 'input_layernorm.weight'], None, eps, None)
        qkv = blocks.linear(hidden, Linear((sa + 'q_proj.weight', sa + 'k_proj.weight', sa + 'v_proj.weight')),
                            None, EPI_BIAS, (l, 0))
        blocks.rotary(qkv, l)
        ctx = blocks.attention(qkv, heads, kv, d, window, True)
        tmp = blocks.linear(ctx, Linear((sa + 'o_proj.weight',)), None, EPI_BIAS, (l, 1))
        hidden = blocks.norm('add_rms', xres, tmp, None, sd[p + 'post_attention_layernorm.weight'], None, eps, None)
        inter = blocks.linear(hidden, Linear((p + 'mlp.gate_proj.weight', p + 'mlp.up_proj.weight'), 'gate_up'),
                              None, EPI_SWIGLU, (l, 2))
        tmp = blocks.linear(inter, Linear((p + 'mlp.down_proj.weight',)), None, EPI_BIAS, (l, 3))
        if every_depth or l == n_layers - 1:
            _final(blocks, run, 'add_rms', xres, tmp, sd['norm.weight'], None, eps)
    return run.depths


qwen3 = mistral


# ------------------------------------------------------------------------------------------------ ModernBERT
def padded_intermediate(i: int) -> int:
    return (i + 127) // 128 * 128


def layer_is_global(cfg, layer: int) -> bool:
    return cfg.layer_types[layer] == 'full_attention'


@torch.no_grad()
def modernbert(sd, cfg, blocks, ids, mask, types=None, out_dtypes=(torch.float32,), every_depth=False):
    """modeling_modernbert.py: ModernBertEmbeddings (gather, LayerNorm), then per layer attn_norm (Identity in layer
    0), Wqkv, rotary with the layer type's table, full or sliding-window (|i - j| <= sliding_window) bidirectional
    attention by ``layer_types``, Wo, mlp_norm, gelu(input) * gate, mlp.Wo; final_norm.  The intermediate width is
    zero-padded to a multiple of 128 (gelu(0) * 0 = 0 feeds zero columns of mlp.Wo)."""
    sd = _strip(sd, 'model.')
    eps, heads, h = cfg.norm_eps, cfg.num_attention_heads, cfg.hidden_size
    d = h // heads
    inter = cfg.intermediate_size
    pad = padded_intermediate(inter) - inter
    run = Run(out_dtypes)
    hidden, xres = blocks.embed(ids, mask, None)
    n_layers = cfg.num_hidden_layers
    zero = torch.zeros(h)

    def bias(name):
        return sd.get(name, zero)

    for l in range(n_layers):
        p = f'layers.{l}.'
        if l > 0:
            hidden = blocks.norm('add_ln', xres, tmp, None, sd[p + 'attn_norm.weight'], bias(p + 'attn_norm.bias'),
                                 eps, None)
        qkv = blocks.linear(hidden, Linear((p + 'attn.Wqkv.weight',)), None, EPI_BIAS, (l, 0))
        blocks.rotary(qkv, l)
        ctx = blocks.attention(qkv, heads, heads, d, 0 if layer_is_global(cfg, l) else int(cfg.sliding_window), False)
        tmp = blocks.linear(ctx, Linear((p + 'attn.Wo.weight',)), None, EPI_BIAS, (l, 1))
        hidden = blocks.norm('add_ln', xres, tmp, None, sd[p + 'mlp_norm.weight'], bias(p + 'mlp_norm.bias'), eps, None)
        act = blocks.linear(hidden, Linear((p + 'mlp.Wi.weight',), 'gate_up', pad_rows=pad, split=(inter, inter)),
                            None, EPI_GEGLU, (l, 2))
        tmp = blocks.linear(act, Linear((p + 'mlp.Wo.weight',), pad_cols=pad), None, EPI_BIAS, (l, 3))
        if every_depth or l == n_layers - 1:
            _final(blocks, run, 'add_ln', xres, tmp, sd['final_norm.weight'], bias('final_norm.bias'), eps)
    return run.depths


FAMILIES = {'bert': bert, 'esm': esm, 'mistral': mistral, 'qwen3': qwen3, 'modernbert': modernbert}


# ------------------------------------------------------------------------------------------ fp32 torch blocks
def _rotate_half(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    x1, x2 = x.chunk(2, dim=-1)
    return x * cos + torch.cat((-x2, x1), dim=-1) * sin


def _rope(s: int, d: int, theta: float) -> tuple[torch.Tensor, torch.Tensor]:
    inv_freq = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.int64).float() / d))
    emb = torch.outer(torch.arange(s).float(), inv_freq)
    emb = torch.cat((emb, emb), dim=-1)
    return emb.cos(), emb.sin()


class TorchBlocks:
    """fp32 torch stand-ins on the CPU in the padded [B*S] layout: every block is the plain formula."""

    def __init__(self, fam: str, sd: Mapping[str, torch.Tensor], cfg, mask: torch.Tensor):
        self.fam, self.cfg, self.mask = fam, cfg, mask
        self.sd = _strip(sd, {'bert': 'bert.', 'esm': 'esm.'}.get(fam, 'model.'))
        self.sd = {k: v.detach().float().cpu() for k, v in self.sd.items()}
        self.b, self.s = mask.shape

    def embed(self, ids, mask, types):
        sd, cfg, s = self.sd, self.cfg, self.s
        if self.fam == 'bert':
            t = torch.zeros_like(ids) if types is None else types
            x = (sd['embeddings.word_embeddings.weight'][ids] + sd['embeddings.token_type_embeddings.weight'][t]
                 + sd['embeddings.position_embeddings.weight'][:s][None])
            x = F.layer_norm(x, (x.shape[-1],), sd['embeddings.LayerNorm.weight'], sd['embeddings.LayerNorm.bias'],
                             cfg.layer_norm_eps)
            return x.reshape(self.b * s, -1), None
        if self.fam == 'esm':
            x = sd['embeddings.word_embeddings.weight'][ids]
            if getattr(cfg, 'token_dropout', False):
                is_mask = ids == cfg.mask_token_id
                x = x.masked_fill(is_mask[..., None], 0.0)
                observed = is_mask.sum(-1).float() / mask.sum(-1)
                x = x * (1 - 0.15 * 0.8) / (1 - observed)[:, None, None]
            x = x * mask[..., None].float()
            return None, x.reshape(self.b * s, -1)
        if self.fam == 'modernbert':
            x = sd['embeddings.tok_embeddings.weight'][ids].reshape(self.b * s, -1)
            x = F.layer_norm(x, (x.shape[-1],), sd['embeddings.norm.weight'], sd.get('embeddings.norm.bias'),
                             cfg.norm_eps)
            return x, x.clone()
        return None, sd['embed_tokens.weight'][ids].reshape(self.b * s, -1)

    def linear(self, x, lin: Linear, bias, epi, slot):
        w = build_weight(lin, [self.sd[n] for n in lin.names])
        y = F.linear(x, w, None if bias is None else bias.float())
        if epi == EPI_BIAS_GELU:
            return F.gelu(y)
        if epi in (EPI_SWIGLU, EPI_GEGLU):
            blk = y.view(y.shape[0], -1, 2, GATE_UP_BLOCK)
            first, second = blk[:, :, 0].reshape(y.shape[0], -1), blk[:, :, 1].reshape(y.shape[0], -1)
            return (F.silu(first) if epi == EPI_SWIGLU else F.gelu(first)) * second
        return y

    def rotary(self, qkv, layer):
        cfg, b, s = self.cfg, self.b, self.s
        if self.fam in ('mistral', 'qwen3'):
            heads, kv = cfg.num_attention_heads, cfg.num_key_value_heads
            d = getattr(cfg, 'head_dim', None) or cfg.hidden_size // heads
            params = getattr(cfg, 'rope_parameters', None) or {}
            theta = float(params.get('rope_theta', getattr(cfg, 'rope_theta', 10000.0)))
            n = heads + kv
        else:
            heads = cfg.num_attention_heads
            d = cfg.hidden_size // heads
            n = 2 * heads
            if self.fam == 'esm':
                theta = 10000.0
            else:
                kind = 'full_attention' if layer_is_global(cfg, layer) else 'sliding_attention'
                theta = float(cfg.rope_parameters[kind]['rope_theta'])
        cos, sin = _rope(s, d, theta)
        x = qkv[:, :n * d].view(b, s, n, d)
        if self.fam == 'qwen3':
            p = f'layers.{layer}.self_attn.'
            eps = cfg.rms_norm_eps
            q, k = x[:, :, :heads], x[:, :, heads:]
            q = self.sd[p + 'q_norm.weight'] * (q * torch.rsqrt(q.pow(2).mean(-1, keepdim=True) + eps))
            k = self.sd[p + 'k_norm.weight'] * (k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + eps))
            x = torch.cat([q, k], dim=2)
        qkv[:, :n * d] = _rotate_half(x, cos[None, :, None], sin[None, :, None]).reshape(b * s, n * d)

    def attention(self, qkv, heads, kv, d, window, causal):
        b, s = self.b, self.s
        q = qkv[:, :heads * d].view(b, s, heads, d).transpose(1, 2)
        k = qkv[:, heads * d:(heads + kv) * d].view(b, s, kv, d).transpose(1, 2).repeat_interleave(heads // kv, 1)
        v = qkv[:, (heads + kv) * d:(heads + 2 * kv) * d].view(b, s, kv, d).transpose(1, 2)
        v = v.repeat_interleave(heads // kv, 1)
        i, j = torch.arange(s)[:, None], torch.arange(s)[None]
        vis = (self.mask != 0)[:, None, None, :].expand(b, 1, s, s)
        if causal:
            vis = vis & (j <= i) & ((i - j < window) if window else True)
        elif window:
            vis = vis & ((i - j).abs() <= window)
        scores = (q @ k.transpose(-1, -2)) / math.sqrt(d)
        prob = torch.softmax(scores.masked_fill(~vis, float('-inf')), -1).nan_to_num(0.0)
        return (prob @ v).transpose(1, 2).reshape(b * s, heads * d)

    def norm(self, kind, xres, add, resid, gamma, beta, eps, out_dtype):
        if kind == 'post_ln':
            return F.layer_norm(add + resid, (add.shape[-1],), gamma.float(), beta.float(), eps)
        if add is not None:
            xres += add
        if kind == 'add_ln':
            return F.layer_norm(xres, (xres.shape[-1],), gamma.float(), None if beta is None else beta.float(), eps)
        return gamma.float() * (xres * torch.rsqrt(xres.pow(2).mean(-1, keepdim=True) + eps))

    def unlayout(self, rows: torch.Tensor) -> torch.Tensor:
        return rows.reshape(self.b, self.s, -1)


# ------------------------------------------------------------------------------------------- test models
def config(fam: str, h: int, layers: int, heads: int | None = None, kv_heads: int | None = None,
           window: int | None = None, intermediate: int | None = None, vocab: int = 300):
    """A small HF config of ``fam``: BERT with two token types, ESM-2 with token dropout, ModernBERT with full
    attention every third layer and ``local_attention`` 128, Mistral / Qwen3 with head_dim 128."""
    import transformers as T

    if fam == 'bert':
        return T.BertConfig(vocab_size=vocab, hidden_size=h, num_hidden_layers=layers, num_attention_heads=heads,
                            intermediate_size=intermediate or 2 * h, max_position_embeddings=512, type_vocab_size=2,
                            layer_norm_eps=1e-12)
    if fam == 'esm':
        return T.EsmConfig(vocab_size=33, hidden_size=h, num_hidden_layers=layers, num_attention_heads=heads,
                           intermediate_size=intermediate or 2 * h, max_position_embeddings=1026,
                           position_embedding_type='rotary', token_dropout=True, mask_token_id=32, pad_token_id=1,
                           layer_norm_eps=1e-5, emb_layer_norm_before=False)
    if fam == 'modernbert':
        return T.ModernBertConfig(vocab_size=vocab, hidden_size=h, num_hidden_layers=layers, num_attention_heads=heads,
                                  intermediate_size=intermediate or 3 * h // 2, max_position_embeddings=512,
                                  local_attention=128, global_attn_every_n_layers=3, norm_eps=1e-5, pad_token_id=0,
                                  bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2)
    cls = T.MistralConfig if fam == 'mistral' else T.Qwen3Config
    extra = {'sliding_window': window} if fam == 'mistral' else {}
    return cls(vocab_size=vocab, hidden_size=h, num_hidden_layers=layers, num_attention_heads=heads,
               num_key_value_heads=kv_heads or heads, head_dim=128, intermediate_size=intermediate or 2 * h,
               max_position_embeddings=512, rms_norm_eps=1e-5, **extra)


NORM_SUFFIXES = ('LayerNorm.weight', 'LayerNorm.bias', 'layer_norm_after.weight', 'layer_norm_after.bias',
                 'layernorm.weight', 'norm.weight', 'norm.bias')


def state_dict(fam: str, cfg, seed: int, device='cpu') -> dict[str, torch.Tensor]:
    """Random weights (weights.random_*_state_dict, std 0.02) in which every norm slot is told apart: each gain drawn
    from +-[0.5, 2] and each bias from N(0, 0.5), per slot and layer; ModernBERT's norms get biases too, and Qwen3's
    q_norm / k_norm gains are drawn the same way."""
    from distllm_b200.embed.encoders import weights as W

    make = {'bert': W.random_bert_state_dict, 'esm': W.random_esm_state_dict, 'mistral': W.random_mistral_state_dict,
            'qwen3': W.random_qwen3_state_dict, 'modernbert': W.random_modernbert_state_dict}[fam]
    sd = make(cfg, seed=seed, device=device, std=0.02)
    g = torch.Generator(device=device).manual_seed(seed + 7)
    for name in sorted(sd):
        if not name.endswith(NORM_SUFFIXES):
            continue
        t = sd[name]
        if name.endswith('bias'):
            sd[name] = torch.randn(t.shape, generator=g, device=device) * 0.5
        else:
            mag = 0.5 + 1.5 * torch.rand(t.shape, generator=g, device=device)
            sign = torch.randint(0, 2, t.shape, generator=g, device=device) * 2 - 1
            sd[name] = (mag * sign).to(t.dtype)
    if fam == 'modernbert':
        h = cfg.hidden_size
        for name in [n for n in sd if n.endswith('norm.weight')]:
            sd[name[:-len('weight')] + 'bias'] = torch.randn(h, generator=g, device=device) * 0.5
    return sd


def oracle_forward(fam: str):
    """The family's CPU oracle forward pass (state dict, config, ids, mask[, types], return_all)."""
    from oracle import bert as obert, esm as oesm, mistral as omistral, modernbert as omodernbert
    from tools import oracle_qwen3

    return {'bert': obert.bert_forward, 'esm': oesm.esm_forward, 'mistral': omistral.mistral_forward,
            'qwen3': oracle_qwen3.qwen3_forward, 'modernbert': omodernbert.modernbert_forward}[fam]
