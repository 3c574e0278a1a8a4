"""``esm2`` encoder: HuggingFace ESM-2 checkpoint in, native sm_90a forward pass out.

Drop-in for distllm/embed/encoders/esm2.py:15-134 (same config fields and defaults; ``faesm`` is
accepted and ignored -- the native path replaces both the eager and the flash-attention variants).
``encode`` returns ``hidden_states[-1]`` of ``EsmForMaskedLM``, i.e. the state after
``emb_layer_norm_after``; the unused LM head is never computed.
"""

from __future__ import annotations

from typing import Literal

import torch
from transformers import BatchEncoding
from transformers import PreTrainedTokenizer

from distllm_b200.embed.encoders.native import NativeEsm2Encoder
from distllm_b200.utils import BaseConfig


class Esm2EncoderConfig(BaseConfig):
    """Config for the ESM-2 encoder (fields as in the reference, esm2.py:15-34)."""

    name: Literal['esm2'] = 'esm2'  # type: ignore[assignment]
    # The model id.  The default is the reference's (esm2.py:21); the native kernels are built for
    # 64-wide attention heads and hidden sizes of 256 x {1,2,3,4,5,8,10,16}: of the published ESM-2 family
    # that is facebook/esm2_t33_650M_UR50D (H=1280) and facebook/esm2_t36_3B_UR50D (H=2560).  The 8M / 35M /
    # 150M checkpoints (16-, 24- and 32-wide heads) and the 15B one (128-wide heads) are rejected when the
    # encoder is built, before any weight is loaded; there is no eager fallback.
    pretrained_model_name_or_path: str = 'facebook/esm2_t6_8M_UR50D'
    # The model tokenizer
    tokenizer_path: str | None = None
    # Return half precision (fp16) embeddings (the reference default)
    half_precision: bool = True
    # Kept for compatibility: inference is always in eval mode here
    eval_mode: bool = True
    # Kept for compatibility: there is no tracing compiler in this path
    compile_model: bool = False
    # Kept for compatibility: the native attention kernel is used either way
    faesm: bool = False


class Esm2Encoder:
    """Encoder for ESM-2 checkpoints on the native kernels."""

    def __init__(self, config: Esm2EncoderConfig):
        from transformers import AutoConfig
        from transformers import EsmForMaskedLM
        from transformers import EsmTokenizer

        from distllm_b200.embed.encoders import adapters

        # a PEFT adapter checkpoint runs on its base_model_name_or_path, merged into the 16-bit weights
        base_path, adapter_dir = adapters.resolve(config.pretrained_model_name_or_path)
        hf_config = AutoConfig.from_pretrained(base_path)
        if hf_config.model_type != 'esm':
            raise NotImplementedError(f'model_type={hf_config.model_type!r} is not an ESM checkpoint')
        NativeEsm2Encoder.validate(hf_config)   # unsupported shapes fail here, before the weights load
        model = EsmForMaskedLM.from_pretrained(base_path)
        tokenizer = EsmTokenizer.from_pretrained(
            adapters.tokenizer_source(config.tokenizer_path, config.pretrained_model_name_or_path, base_path),
        )
        # proper truncation, as esm2.py:66
        tokenizer.model_max_length = hf_config.max_position_embeddings

        self.config = config
        state_dict = model.state_dict()
        self.adapter_ignored = []
        if adapter_dir is not None:
            adapter = adapters.load_adapter(adapter_dir, state_dict)
            self.adapter_ignored = list(adapter.ignored)
            state_dict = adapters.merge_adapter(state_dict, adapter)
        self._native = NativeEsm2Encoder(hf_config, state_dict)
        del model, state_dict
        self._tokenizer = tokenizer
        self._dtype = torch.float16 if config.half_precision else torch.float32

    @classmethod
    def from_native(cls, native: NativeEsm2Encoder, tokenizer: PreTrainedTokenizer | None = None,
                    half_precision: bool = False) -> 'Esm2Encoder':
        """Wrap an already-built native encoder (synthetic weights, tests, benchmarks)."""
        self = cls.__new__(cls)
        self.config = None
        self.adapter_ignored = []
        self._native = native
        self._tokenizer = tokenizer
        self._dtype = torch.float16 if half_precision else torch.float32
        return self

    @property
    def dtype(self) -> torch.dtype:
        return self._dtype

    @property
    def device(self) -> torch.device:
        return self._native.device

    @property
    def embedding_size(self) -> int:
        return self._native.hidden_size

    @property
    def tokenizer(self) -> PreTrainedTokenizer:
        return self._tokenizer

    @property
    def native(self) -> NativeEsm2Encoder:
        return self._native

    def encode(self, batch_encoding: BatchEncoding) -> torch.Tensor:
        """Last hidden state ``[B,S,H]`` in ``self.dtype`` (esm2.py:109-134)."""
        hidden = self._native.encode(
            batch_encoding['input_ids'],
            batch_encoding['attention_mask'],
            None,
            out_dtype=torch.float32,
        )
        return hidden if self._dtype == torch.float32 else hidden.to(self._dtype)

    def encode_pooled(self, batch_encoding: BatchEncoding, pool_kind: int, normalize: bool,
                      out: torch.Tensor | None = None) -> torch.Tensor:
        """Fused encode + pool (+ normalise) -> fp32 ``[B,H]`` (used by the native embedders)."""
        return self._native.encode_pooled(
            batch_encoding['input_ids'],
            batch_encoding['attention_mask'],
            None,
            pool_kind,
            normalize,
            out=out,
        )
