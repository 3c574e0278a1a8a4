"""PEFT adapter checkpoints (LoRA, IA3) on the native encoders, without peft at run time.

A directory holding ``adapter_config.json`` and no ``config.json`` is an adapter checkpoint, as transformers'
``from_pretrained`` decides: the base model is ``base_model_name_or_path`` and the adapter tensors come from
``adapter_model.safetensors`` (or ``adapter_model.bin``).  Keys lose peft's ``base_model.model.`` prefix (what
transformers' ``load_adapter`` strips) and are then matched to the modules of the base ``AutoModel`` /
``EsmForMaskedLM`` state dict:

  LoRA   ``<module>.lora_A.weight`` [r, in], ``<module>.lora_B.weight`` [out, r]:  y = W x + b + s B A x, with
         s = lora_alpha / r, or lora_alpha / sqrt(r) under ``use_rslora``; r comes from the tensor shapes, so
         ``rank_pattern`` needs no parsing
  IA3    ``<module>.ia3_l``: shape (out, 1) scales the output, bias included (y = l * (W x + b)); shape (1, in) scales
         the input, peft's ``feedforward_modules`` (y = W (l * x) + b).  Decided by the shape: peft's default BERT
         targets make ``output.dense`` match both the attention output and the FFN down projection.

This restates peft's published ``tuners/lora/layer.py`` (``LoraLayer.update_layer``, ``Linear.forward``) and
``tuners/ia3/layer.py`` (``IA3Layer.update_layer``, ``Linear.forward``); peft is absent from this image, so the
parity is UNPINNED, as ``nf4.py``'s is for bitsandbytes.

Every transformer-block linear layer (``nf4.is_quantized_linear``) can carry an adapter.  Tensors on heads that
cannot change the last hidden state (BERT's pooler, ESM-2's LM and contact heads) are ignored and counted; any
other tensor that matches no module is an error naming the keys -- where peft would warn and return the base
model.  What the native encoders do not run (DoRA, ``alpha_pattern``, ``modules_to_save``, trained biases,
embedding LoRA, ``fan_in_fan_out``) is refused with the field that asks for it.

The weights: with 16-bit matrices (and for IA3 always) the adapter is merged in fp32 at load time
(:func:`merge_adapter`) before the storage rounding; under NF4 storage a LoRA adapter stays unmerged and the NF4
GEMM adds ``U . B_cat^T`` itself (``weights.lora_slot_factors``), because ``NF4(W + s B A)`` is not the model the
adapter was trained against.
"""

from __future__ import annotations

import json
import logging
import math
from dataclasses import dataclass
from dataclasses import field
from pathlib import Path
from typing import Mapping

import torch

from distllm_b200.embed.encoders.nf4 import is_quantized_linear

ADAPTER_CONFIG = 'adapter_config.json'
PEFT_PREFIX = 'base_model.model.'
# modules downstream of the last hidden state: an adapter on them changes nothing the encoders return
IGNORED_MODULES = ('pooler.dense', 'lm_head.dense', 'lm_head.decoder', 'contact_head.regression')
_TOKENIZER_FILES = ('tokenizer_config.json', 'tokenizer.json', 'vocab.txt', 'vocab.json', 'tokenizer.model',
                    'spiece.model')

logger = logging.getLogger(__name__)


class AdapterError(ValueError):
    """An adapter checkpoint the native encoders cannot run as the reference would."""


@dataclass
class Adapter:
    """One adapter matched to a base state dict: tensors in fp32, keyed by module name (the state-dict key of the
    module's weight without ``.weight``)."""

    peft_type: str
    lora: dict[str, tuple[torch.Tensor, torch.Tensor, float]] = field(default_factory=dict)  # A [r,in], B [out,r], s
    ia3: dict[str, tuple[torch.Tensor, bool]] = field(default_factory=dict)   # l (flat), scales the input
    ignored: list[str] = field(default_factory=list)                          # modules whose tensors were ignored


def adapter_dir(path: str | Path) -> Path | None:
    """``path`` when it is a local adapter checkpoint (``adapter_config.json`` and no ``config.json``), else None."""
    p = Path(path)
    if (p / ADAPTER_CONFIG).is_file() and not (p / 'config.json').is_file():
        return p
    return None


def read_config(directory: Path) -> dict:
    return json.loads((directory / ADAPTER_CONFIG).read_text())


def resolve(path: str | Path) -> tuple[str, Path | None]:
    """(base checkpoint, adapter directory or None) for ``pretrained_model_name_or_path``."""
    d = adapter_dir(path)
    if d is None:
        return str(path), None
    base = read_config(d).get('base_model_name_or_path')
    if not base:
        raise AdapterError(f'{d / ADAPTER_CONFIG}: base_model_name_or_path is missing')
    return str(base), d


def tokenizer_source(explicit: str | None, path: str | Path, base: str) -> str:
    """The tokenizer the reference loads: ``explicit`` when given; else the adapter directory when it holds tokenizer
    files, the base checkpoint when it does not."""
    if explicit:
        return explicit
    d = adapter_dir(path)
    if d is None or any((d / f).is_file() for f in _TOKENIZER_FILES):
        return str(path)
    return base


def check_config(cfg: dict) -> str:
    """Refuse what the native encoders do not run; returns the peft type."""
    kind = cfg.get('peft_type')
    if kind not in ('LORA', 'IA3'):
        raise AdapterError(f'peft_type {kind!r} is not supported (supported: LORA, IA3)')
    if cfg.get('modules_to_save'):
        raise AdapterError(f'modules_to_save {cfg["modules_to_save"]!r} is not supported (trained copies of whole '
                           f'modules)')
    if cfg.get('fan_in_fan_out'):
        raise AdapterError('fan_in_fan_out: true is not supported (Conv1D-style weights)')
    if kind == 'LORA':
        if cfg.get('use_dora'):
            raise AdapterError('use_dora: true is not supported (DoRA)')
        if cfg.get('alpha_pattern'):
            raise AdapterError(f'alpha_pattern {cfg["alpha_pattern"]!r} is not supported (per-module lora_alpha)')
        if cfg.get('bias', 'none') != 'none':
            raise AdapterError(f'bias {cfg["bias"]!r} is not supported (trained biases); need "none"')
        if cfg.get('lora_bias'):
            raise AdapterError('lora_bias: true is not supported (a bias on lora_B)')
    return kind


def read_tensors(directory: Path) -> dict[str, torch.Tensor]:
    st, binf = directory / 'adapter_model.safetensors', directory / 'adapter_model.bin'
    if st.is_file():
        from safetensors.torch import load_file

        return load_file(str(st))
    if binf.is_file():
        return torch.load(str(binf), map_location='cpu', weights_only=True)
    raise AdapterError(f'{directory}: neither adapter_model.safetensors nor adapter_model.bin')


def lora_scale(cfg: dict, r: int) -> float:
    alpha = float(cfg.get('lora_alpha', 8))
    return alpha / math.sqrt(r) if cfg.get('use_rslora') else alpha / r


def match_adapter(cfg: dict, tensors: Mapping[str, torch.Tensor], state_dict: Mapping[str, torch.Tensor]) -> Adapter:
    """Match adapter tensors to the modules of ``state_dict`` (the base model's) and check every shape."""
    kind = check_config(cfg)
    ad = Adapter(kind)
    by_module: dict[str, dict[str, torch.Tensor]] = {}
    unmatched = []
    for key, t in tensors.items():
        k = key[len(PEFT_PREFIX):] if key.startswith(PEFT_PREFIX) else key
        if '.lora_embedding_' in k:
            raise AdapterError(f'{key}: LoRA on embeddings is not supported')
        if '.lora_magnitude_vector' in k:
            raise AdapterError(f'{key}: DoRA (use_dora) is not supported')
        for suffix in ('.lora_A.weight', '.lora_B.weight', '.lora_B.bias', '.ia3_l'):
            if k.endswith(suffix):
                by_module.setdefault(k[:-len(suffix)], {})[suffix] = t
                break
        else:
            unmatched.append(key)
    for module, parts in by_module.items():
        if '.lora_B.bias' in parts:
            raise AdapterError(f'{module}.lora_B.bias: lora_bias is not supported')
        weight = state_dict.get(module + '.weight')
        if weight is not None and module.endswith(IGNORED_MODULES):
            ad.ignored.append(module)
            continue
        if weight is None or not is_quantized_linear(module + '.weight', weight):
            unmatched += [module + s for s in parts]
            continue
        out_f, in_f = weight.shape
        if kind == 'LORA':
            a, b = parts.get('.lora_A.weight'), parts.get('.lora_B.weight')
            if a is None or b is None or '.ia3_l' in parts:
                raise AdapterError(f'{module}: a LoRA module needs lora_A.weight and lora_B.weight, got {sorted(parts)}')
            r = a.shape[0]
            if tuple(a.shape) != (r, in_f) or tuple(b.shape) != (out_f, r):
                raise AdapterError(f'{module}: lora_A {tuple(a.shape)} / lora_B {tuple(b.shape)} do not fit the '
                                   f'[{out_f}, {in_f}] weight')
            ad.lora[module] = (a.float(), b.float(), lora_scale(cfg, r))
        else:
            if set(parts) != {'.ia3_l'}:
                raise AdapterError(f'{module}: an IA3 module holds ia3_l only, got {sorted(parts)}')
            l = parts['.ia3_l']
            if tuple(l.shape) == (out_f, 1):
                ad.ia3[module] = (l.float().flatten(), False)
            elif tuple(l.shape) == (1, in_f):
                ad.ia3[module] = (l.float().flatten(), True)
            else:
                raise AdapterError(f'{module}.ia3_l: shape {tuple(l.shape)} is neither ({out_f}, 1) nor (1, {in_f})')
    if unmatched:
        raise AdapterError(f'adapter tensors match no transformer-block linear layer of the base model: '
                           f'{sorted(unmatched)[:8]}{" ..." if len(unmatched) > 8 else ""} (the keys must name modules '
                           f'of the base AutoModel / EsmForMaskedLM after stripping {PEFT_PREFIX!r})')
    if ad.ignored:
        logger.warning('adapter: ignored tensors on %d module(s) downstream of the last hidden state: %s',
                       len(ad.ignored), ad.ignored)
    return ad


def load_adapter(directory: Path, state_dict: Mapping[str, torch.Tensor]) -> Adapter:
    return match_adapter(read_config(directory), read_tensors(directory), state_dict)


@torch.no_grad()
def merge_adapter(state_dict: Mapping[str, torch.Tensor], adapter: Adapter) -> dict[str, torch.Tensor]:
    """Copy of ``state_dict`` with the adapter merged in fp32: ``W + s B A`` (LoRA); ``diag(l) W`` and ``l * b``, or
    ``W diag(l)`` (IA3).  The encoders round the result to their storage type as they round any weight."""
    out = dict(state_dict)
    for module, (a, b, s) in adapter.lora.items():
        w = state_dict[module + '.weight']
        out[module + '.weight'] = w.float() + s * (b.to(w.device) @ a.to(w.device))
    for module, (l, on_input) in adapter.ia3.items():
        w = state_dict[module + '.weight']
        if on_input:
            out[module + '.weight'] = w.float() * l.to(w.device)[None, :]
        else:
            out[module + '.weight'] = w.float() * l.to(w.device)[:, None]
            if module + '.bias' in state_dict:   # (the NF4 round trip may have moved the weight, not the bias)
                bias = state_dict[module + '.bias']
                out[module + '.bias'] = bias.float() * l.to(bias.device)
    return out
