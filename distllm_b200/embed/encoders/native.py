"""Owner of one ``B2EEncoder`` handle: weights on the device + the native forward entry points."""

from __future__ import annotations

import ctypes as C
from typing import Mapping

import torch

from distllm_b200 import _native
from distllm_b200.embed.encoders import weights as W


class NativeBertEncoder:
    """Encoder forward pass on libb2e (wgmma GEMMs + fused attention + row kernels).

    Holds the device weight tensors (the C handle only borrows their pointers) and wraps
    ``b2e_encode`` / ``b2e_encode_pooled`` / ``b2e_embed_host``.  ``_DESC`` / ``_WEIGHTS`` pick the
    architecture: BERT here, ESM-2 in the ``NativeEsm2Encoder`` subclass.
    """

    _DESC = staticmethod(W.bert_desc)
    _WEIGHTS = staticmethod(W.bert_weight_list)
    _ARCH = 'bert'    # picks the build of the library (16-bit storage type): _native.storage_for_arch

    def __init__(self, hf_config, state_dict: Mapping[str, torch.Tensor],
                 device: torch.device | str | None = None, storage: str | None = None, nf4: bool = False,
                 lora: Mapping[str, tuple[torch.Tensor, torch.Tensor, float]] | None = None) -> None:
        """``nf4``: hold every weight matrix in 4-bit NF4 (``b2e_encoder_create_nf4``), quantised from
        ``state_dict`` one checkpoint matrix at a time on the device; the results equal bit for bit those of the
        16-bit encoder built from ``nf4.quantize_state_dict_nf4(state_dict)``.

        ``lora`` (NF4 only; ``adapters.Adapter.lora``): LoRA modules kept unmerged, added by the NF4 GEMMs as extra
        k-blocks (``b2e_encoder_create_nf4_lora``, ``weights.lora_slot_factors``)."""
        if nf4 and self._ARCH == 'esm':
            raise NotImplementedError('ESM-2 has no quantised configuration')
        if lora and not nf4:
            raise ValueError('unmerged LoRA needs NF4 storage; merge the adapter into 16-bit weights instead')
        self.storage = storage or _native.storage_for_arch(self._ARCH)
        lib = _native.load(self.storage)
        if not torch.cuda.is_available():
            raise _native.NativeError(
                'no CUDA device: the native encoder has no CPU fallback (sm_90a only)')
        self.device = torch.device(device if device is not None else f'cuda:{torch.cuda.current_device()}')
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.hf_config = hf_config
        self.desc = self._DESC(hf_config)
        # shape validation BEFORE the weights are converted and uploaded (an unsupported checkpoint must
        # not cost gigabytes of transfers first)
        _native.check(lib.b2e_check_model(C.byref(self.desc)), lib)
        self.hidden_size = hf_config.hidden_size
        self.max_positions = hf_config.max_position_embeddings
        extra = {'matrix': W.nf4_matrix(self.device)} if nf4 else {}
        self._weights = self._WEIGHTS(state_dict, hf_config.num_hidden_layers, self.device,
                                      _native.STORAGE_TORCH_DTYPE[self.storage], **extra)
        self.nf4 = nf4
        n = len(self._weights)
        expected = lib.b2e_num_weights(C.byref(self.desc))
        if n != expected:
            raise _native.NativeError(f'weight list has {n} tensors, ABI expects {expected}')
        ptrs = (C.c_void_p * n)(*[(t.codes if isinstance(t, W.Nf4Matrix) else t).data_ptr() for t in self._weights])
        handle = C.c_void_p()
        self._lora = (W.lora_slot_factors(self._ARCH, hf_config, lora, self.device,
                                          _native.STORAGE_TORCH_DTYPE[self.storage]) if lora else [])
        if nf4:
            scales = [t.absmax.data_ptr() for t in self._weights if isinstance(t, W.Nf4Matrix)]
            scale_ptrs = (C.c_void_p * len(scales))(*scales)
            if self._lora:
                k = len(self._lora)
                a_ptrs = (C.c_void_p * k)(*[f[0].data_ptr() if f else None for f in self._lora])
                b_ptrs = (C.c_void_p * k)(*[f[1].data_ptr() if f else None for f in self._lora])
                ranks = (C.c_int * k)(*[f[2] if f else 0 for f in self._lora])
                _native.check(lib.b2e_encoder_create_nf4_lora(
                    C.byref(self.desc), ptrs, n, scale_ptrs, len(scales), a_ptrs, b_ptrs, ranks, k,
                    self.device.index, C.byref(handle)), lib)
            else:
                _native.check(lib.b2e_encoder_create_nf4(C.byref(self.desc), ptrs, n, scale_ptrs, len(scales),
                                                         self.device.index, C.byref(handle)), lib)
        else:
            _native.check(lib.b2e_encoder_create(C.byref(self.desc), ptrs, n, self.device.index,
                                                 C.byref(handle)), lib)
        self._handle = handle
        self._lib = lib

    @classmethod
    def validate(cls, hf_config) -> None:
        """Raise ``NativeError`` / ``NotImplementedError`` when this checkpoint's shape has no native forward
        pass.  Needs no device and no weights: the encoders call it right after reading ``config.json``,
        before ``from_pretrained`` loads a single parameter."""
        desc = cls._DESC(hf_config)
        lib = _native.load(_native.storage_for_arch(cls._ARCH))
        _native.check(lib.b2e_check_model(C.byref(desc)), lib)

    def close(self) -> None:
        if getattr(self, '_handle', None):
            self._lib.b2e_encoder_destroy(self._handle)
            self._handle = None

    def __del__(self) -> None:  # pragma: no cover - interpreter shutdown order
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    # ------------------------------------------------------------------ helpers
    def _prep(self, t: torch.Tensor | None, name: str) -> torch.Tensor | None:
        if t is None:
            return None
        if t.device != self.device:
            t = t.to(self.device)
        if t.dtype != torch.int64:
            t = t.to(torch.int64)
        if not t.is_contiguous():
            t = t.contiguous()
        if t.dim() != 2:
            raise _native.NativeError(f'{name} must be [B,S]')
        return t

    def weight_bytes(self) -> dict[str, int]:
        """Device bytes of the weights: ``matrix`` (16-bit matrices, or NF4 codes + scales) and ``other``."""
        return W.device_weight_bytes(self._weights)

    def lora_bytes(self) -> int:
        """Device bytes of the unmerged LoRA factors (A_cat and B_cat of every adapted slot)."""
        return sum(f[0].nbytes + f[1].nbytes for f in self._lora if f)

    def workspace_bytes(self, batch: int, seq: int) -> int:
        return int(self._lib.b2e_workspace_bytes(self._handle, batch, seq))

    # ------------------------------------------------------------------ forward
    def encode(self, input_ids: torch.Tensor, attention_mask: torch.Tensor,
               token_type_ids: torch.Tensor | None = None,
               out_dtype: torch.dtype = torch.float32) -> torch.Tensor:
        """Final hidden state ``[B,S,H]`` (post final LayerNorm) as fp32 or fp16."""
        ids = self._prep(input_ids, 'input_ids')
        mask = self._prep(attention_mask, 'attention_mask')
        types = self._prep(token_type_ids, 'token_type_ids')
        b, s = ids.shape
        out = torch.empty((b, s, self.hidden_size), dtype=out_dtype, device=self.device)
        with torch.cuda.device(self.device):
            _native.check(self._lib.b2e_encode(
                self._handle, ids.data_ptr(), mask.data_ptr(), _native._ptr(types), b, s,
                out.data_ptr(), _native.dtype_code(out_dtype), _native.stream_ptr(self.device)), self._lib)
        return out

    def encode_pooled(self, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                      token_type_ids: torch.Tensor | None, pool_kind: int, normalize: bool,
                      out: torch.Tensor | None = None) -> torch.Tensor:
        """Forward + fused pooling (+ L2 normalise): fp32 ``[B,H]``; mask is left untouched."""
        ids = self._prep(input_ids, 'input_ids')
        mask = self._prep(attention_mask, 'attention_mask')
        types = self._prep(token_type_ids, 'token_type_ids')
        b, s = ids.shape
        if out is None:
            out = torch.empty((b, self.hidden_size), dtype=torch.float32, device=self.device)
        elif (out.dtype != torch.float32 or not out.is_contiguous() or out.device != self.device
              or tuple(out.shape) != (b, self.hidden_size)):
            raise _native.NativeError('out must be a contiguous fp32 [B,H] tensor on the encoder device')
        with torch.cuda.device(self.device):
            _native.check(self._lib.b2e_encode_pooled(
                self._handle, ids.data_ptr(), mask.data_ptr(), _native._ptr(types), b, s, pool_kind,
                int(normalize), out.data_ptr(), _native.stream_ptr(self.device)), self._lib)
        return out

    def embed_host(self, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                   token_type_ids: torch.Tensor | None, batch: int, pool_kind: int,
                   normalize: bool, out: torch.Tensor | None = None) -> torch.Tensor:
        """Whole batch loop over HOST tensors (pin them for full PCIe speed) -> host fp32 ``[N,H]``.

        One C call: per batch H2D of ids/mask/types, forward, fused pooling, D2H of the pooled rows.
        """
        for t in (input_ids, attention_mask, token_type_ids):
            if t is not None and (t.is_cuda or t.dtype != torch.int64 or not t.is_contiguous()):
                raise _native.NativeError('embed_host expects contiguous int64 host tensors')
        n, s = input_ids.shape
        if out is None:
            out = torch.empty((n, self.hidden_size), dtype=torch.float32,
                              pin_memory=True)
        _native.check(self._lib.b2e_embed_host(
            self._handle, input_ids.data_ptr(), attention_mask.data_ptr(),
            _native._ptr(token_type_ids), n, s, batch, pool_kind, int(normalize), out.data_ptr()), self._lib)
        return out


class NativeEsm2Encoder(NativeBertEncoder):
    """ESM-2 (pre-LayerNorm, rotary, token dropout) on the same kernels; ``token_type_ids`` unused."""

    _DESC = staticmethod(W.esm_desc)
    _WEIGHTS = staticmethod(W.esm_weight_list)
    _ARCH = 'esm'


class NativeMistralEncoder(NativeBertEncoder):
    """Mistral family (pre-RMSNorm blocks, rotary, grouped-query causal attention with optional sliding
    window, SwiGLU) on the wgmma GEMM + the head_dim-128 causal attention kernel; ``token_type_ids``
    unused."""

    _DESC = staticmethod(W.mistral_desc)
    _WEIGHTS = staticmethod(W.mistral_weight_list)
    _ARCH = 'mistral'


class NativeQwen3Encoder(NativeBertEncoder):
    """Qwen3 (Qwen3-Embedding): the Mistral-family trunk with a per-head RMSNorm of q and k before the rotary
    embedding, fused with it in one kernel; ``token_type_ids`` unused."""

    _DESC = staticmethod(W.qwen3_desc)
    _WEIGHTS = staticmethod(W.qwen3_weight_list)
    _ARCH = 'qwen3'


class NativeModernBertEncoder(NativeBertEncoder):
    """ModernBERT (pre-LayerNorm blocks, rotary with one base per layer type, alternating full / sliding-window
    bidirectional attention, GeGLU) on the wgmma GEMMs and the head_dim-64 attention kernel with its
    sliding-window variant; ``token_type_ids`` unused."""

    _DESC = staticmethod(W.modernbert_desc)
    _WEIGHTS = staticmethod(W.modernbert_weight_list)
    _ARCH = 'modernbert'
