"""PEFT adapters (LoRA, IA3) as an adapted fp32 state dict, for the family oracles.

Restates peft's published ``tuners/lora/layer.py`` (``Linear.forward``: ``result = base(x) + lora_B(lora_A(x)) *
scaling``, ``scaling = lora_alpha / r`` or ``lora_alpha / sqrt(r)`` with ``use_rslora``) and ``tuners/ia3/layer.py``
(``Linear.forward``: feed-forward modules scale the input, ``base(x * ia3_l)``; the others the output,
``base(x) * ia3_l``), merged into the weights: in exact arithmetic the merged and unmerged forms are the same model.
The oracles in ``oracle/{bert,esm,mistral,modernbert}.py`` then run on the result unchanged.  peft is not installed
here: the parity with it is unpinned; tests/test_adapters_cpu.py pins this file against forward hooks on HF's own
``nn.Linear`` modules.
"""

from __future__ import annotations

import math

import torch


def adapted_state_dict(state_dict: dict[str, torch.Tensor], tensors: dict[str, torch.Tensor],
                       config: dict) -> dict[str, torch.Tensor]:
    """Base ``state_dict`` + adapter ``tensors`` (peft's saved keys) + ``adapter_config.json`` -> fp32 state dict."""
    sd = {k: v.detach().float().clone() for k, v in state_dict.items()}
    keys = {k.removeprefix('base_model.model.'): v.detach().float() for k, v in tensors.items()}
    alpha = float(config.get('lora_alpha', 8))
    for k, a in keys.items():
        if k.endswith('.lora_A.weight'):
            module = k[:-len('.lora_A.weight')]
            b = keys[module + '.lora_B.weight']
            r = a.shape[0]
            s = alpha / math.sqrt(r) if config.get('use_rslora') else alpha / r
            sd[module + '.weight'] = sd[module + '.weight'] + s * (b @ a)
        elif k.endswith('.ia3_l'):
            module = k[:-len('.ia3_l')]
            # (out, 1) scales the rows of W (the outputs, and so the bias too); (1, in) its columns (the inputs)
            sd[module + '.weight'] = sd[module + '.weight'] * a
            if a.shape[1] == 1 and module + '.bias' in sd:
                sd[module + '.bias'] = sd[module + '.bias'] * a.flatten()
    return sd
