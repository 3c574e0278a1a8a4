"""``auto`` encoder: HuggingFace checkpoint in, native sm_90a forward pass out.

Drop-in for distllm/embed/encoders/auto.py:15-138 -- same config fields and defaults, same
properties, ``encode`` returns the last hidden state ``[B,S,H]``.  transformers is used only to read
the checkpoint and to build the tokenizer; the forward pass is libb2e (fp16 tensor-core GEMMs with
fp32 accumulation, fp32 LayerNorm/softmax statistics).  There is no eager/CPU fallback: an
architecture that is not built raises.
"""

from __future__ import annotations

from typing import Literal
from typing import Optional

import torch
from transformers import BatchEncoding
from transformers import PreTrainedTokenizer

from distllm_b200.embed.encoders.native import NativeBertEncoder
from distllm_b200.embed.encoders.native import NativeMistralEncoder
from distllm_b200.embed.encoders.native import NativeModernBertEncoder
from distllm_b200.embed.encoders.native import NativeQwen3Encoder
from distllm_b200.utils import BaseConfig

# HF model_type -> native forward pass (BERT: post-LN encoder; Mistral: pre-RMSNorm decoder blocks
# with rotary, grouped-query causal attention and SwiGLU, used as an encoder by the embedding models;
# ModernBERT: pre-LN encoder with rotary, alternating full / sliding-window attention and GeGLU --
# examples/embed/workstation/modernbert_semchunk.yaml:16-17; Qwen3: the Mistral block with a per-head RMSNorm of q
# and k before rotary -- Qwen3-Embedding 0.6B / 4B / 8B)
_NATIVE_BY_MODEL_TYPE = {'bert': NativeBertEncoder, 'mistral': NativeMistralEncoder,
                         'modernbert': NativeModernBertEncoder, 'qwen3': NativeQwen3Encoder}
_SUPPORTED_MODEL_TYPES = tuple(_NATIVE_BY_MODEL_TYPE)


class AutoEncoderConfig(BaseConfig):
    """Config for the AutoModel-compatible encoder (fields as in the reference, auto.py:15-31)."""

    name: Literal['auto'] = 'auto'  # type: ignore[assignment]
    # The model id
    pretrained_model_name_or_path: str
    # Optional tokenizer
    tokenizer_name: Optional[str] = None  # noqa: UP007
    # Report/return half precision (fp16) embeddings
    half_precision: bool = False
    # Kept for compatibility: inference is always in eval mode here
    eval_mode: bool = True
    # Kept for compatibility: there is no tracing compiler in this path
    compile_model: bool = False
    # The model id may name a PEFT adapter checkpoint (adapter_config.json without config.json, LoRA or IA3): the
    # base model is its base_model_name_or_path, and the tokenizer tokenizer_name, else the adapter directory if it
    # holds tokenizer files, else the base (embed/encoders/adapters.py).
    # NF4 (bitsandbytes) weight quantisation: every transformer-block weight matrix is held on the device in 4-bit
    # NF4 (3.56x less memory than 16 bits) and dequantised inside the GEMMs to exactly dequant(quant(W)).  A LoRA
    # adapter stays unmerged next to the NF4 weights; an IA3 adapter is merged into dequant(quant(W)) at load time,
    # in 16 bits, as with nf4_storage: False
    quantization: bool = True
    # With quantization: False dequantises once at load time into 16-bit matrices instead -- the same results bit for
    # bit, 3.56x the weight memory, and the faster 16-bit GEMM (README: the NF4 GEMM runs at 0.64-0.78x of it)
    nf4_storage: bool = True


class AutoEncoder:
    """Encoder for HF checkpoints of the BERT, ModernBERT, Mistral and Qwen3 families on the native kernels.

    Built shapes (``b2e_check_model``, checked before any weight is loaded): BERT with head_dim 64 or 32 and H in
    256 x {1,2,3,4,5,8,10,16}, 384 or 640 (all-MiniLM-L6-v2, bge-small-en-v1.5, e5-small-v2: 384 = 12 x 32);
    ModernBERT with head_dim 64 at H a multiple of 256; Mistral and Qwen3 with head_dim 128 at a built H that is a
    multiple of 256 (Qwen3-Embedding-0.6B / 4B / 8B: H = 1024 / 2560 / 4096), Qwen3 without sliding-window layers,
    without attention biases and with default rotary."""

    def __init__(self, config: AutoEncoderConfig):
        from transformers import AutoConfig
        from transformers import AutoModel
        from transformers import AutoTokenizer

        from distllm_b200.embed.encoders import adapters

        # a PEFT adapter checkpoint (adapter_config.json, no config.json) runs on its base_model_name_or_path
        base_path, adapter_dir = adapters.resolve(config.pretrained_model_name_or_path)
        hf_config = AutoConfig.from_pretrained(base_path)
        if hf_config.model_type not in _SUPPORTED_MODEL_TYPES:
            raise NotImplementedError(
                f'model_type={hf_config.model_type!r} has no native sm_90a forward pass yet '
                f'(built: {_SUPPORTED_MODEL_TYPES}); there is no eager fallback.',
            )
        _NATIVE_BY_MODEL_TYPE[hf_config.model_type].validate(hf_config)   # before any weight is loaded
        model = AutoModel.from_pretrained(base_path)
        tokenizer = AutoTokenizer.from_pretrained(
            adapters.tokenizer_source(config.tokenizer_name, config.pretrained_model_name_or_path, base_path),
        )
        # proper truncation, as auto.py:74
        tokenizer.model_max_length = hf_config.max_position_embeddings

        self.config = config
        state_dict = model.state_dict()
        adapter = adapters.load_adapter(adapter_dir, state_dict) if adapter_dir is not None else None
        # modules whose adapter tensors were ignored (heads downstream of the last hidden state)
        self.adapter_ignored = list(adapter.ignored) if adapter is not None else []
        nf4 = False
        if config.quantization:
            # the reference's default (auto.py:44-56): every nn.Linear weight goes through 4-bit NormalFloat with
            # double quantisation and is dequantised in front of each matmul -- what the GEMMs see is
            # dequant(quant(W)) (embed/encoders/nf4.py restates bitsandbytes' published algorithm).  The weights stay
            # in NF4 on the device, quantised one matrix at a time, and the GEMMs dequantise them exactly.  A
            # checkpoint whose quantised matrices are not all in 64-column blocks (no published checkpoint of a built
            # family), or a config with nf4_storage: False, gets dequant(quant(W)) computed here once, in 16 bits: the
            # same results, without the saving.  A LoRA adapter stays outside the quantisation, as in the reference
            # (dequant(NF4(W)) x + s B A x): under NF4 storage the GEMMs add it unmerged, otherwise it is merged in
            # fp32 into dequant(quant(W)).  An IA3 adapter always takes the second path.
            from distllm_b200.embed.encoders.nf4 import is_quantized_linear
            from distllm_b200.embed.encoders.nf4 import nf4_storable
            from distllm_b200.embed.encoders.nf4 import quantize_state_dict_nf4

            nf4 = (config.nf4_storage and (adapter is None or adapter.peft_type == 'LORA')
                   and all(nf4_storable(t) for name, t in state_dict.items() if is_quantized_linear(name, t)))
            if not nf4:
                state_dict = quantize_state_dict_nf4(state_dict, device='cuda' if torch.cuda.is_available() else None)
        lora = None
        if adapter is not None:
            if nf4:
                lora = adapter.lora
            else:
                state_dict = adapters.merge_adapter(state_dict, adapter)
        extra = {'lora': lora} if lora else {}   # without an adapter the encoder is built exactly as before
        self._native = _NATIVE_BY_MODEL_TYPE[hf_config.model_type](hf_config, state_dict, nf4=nf4, **extra)
        del model, state_dict
        self._tokenizer = tokenizer
        self._dtype = torch.float16 if config.half_precision else torch.float32

    @classmethod
    def from_native(cls, native: NativeBertEncoder, tokenizer: PreTrainedTokenizer | None = None,
                    half_precision: bool = False) -> 'AutoEncoder':
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
    def native(self) -> NativeBertEncoder:
        return self._native

    def encode(self, batch_encoding: BatchEncoding) -> torch.Tensor:
        """Last hidden state ``[B,S,H]`` in ``self.dtype`` (auto.py:119-138)."""
        hidden = self._native.encode(
            batch_encoding['input_ids'],
            batch_encoding['attention_mask'],
            batch_encoding.get('token_type_ids'),
            out_dtype=torch.float32,
        )
        return hidden if self._dtype == torch.float32 else hidden.to(self._dtype)

    def encode_pooled(self, batch_encoding: BatchEncoding, pool_kind: int, normalize: bool,
                      out: torch.Tensor | None = None) -> torch.Tensor:
        """Fused encode + pool (+ normalise) -> fp32 ``[B,H]`` (used by the native embedders)."""
        return self._native.encode_pooled(
            batch_encoding['input_ids'],
            batch_encoding['attention_mask'],
            batch_encoding.get('token_type_ids'),
            pool_kind,
            normalize,
            out=out,
        )
