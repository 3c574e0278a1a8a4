"""ctypes binding of libb2e.so (the C ABI declared in include/b2e.h).

There is deliberately no fallback: if the library is missing, or a compute call is made without an
sm_90 device, a ``NativeError`` is raised.  Tensors cross the boundary as ``data_ptr()`` integers
plus sizes; the current torch CUDA stream is passed explicitly.
"""

from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import torch

# Two builds of the same sources (distllm_b200/build.py): they differ only in the 16-bit storage type of
# weights and activations.  libb2e.so = IEEE half, libb2e_bf16.so = bfloat16 (b2e_storage_dtype()).
LIB_PATH = Path(__file__).resolve().parent / 'libb2e.so'
LIB_PATHS = {'f16': LIB_PATH, 'bf16': LIB_PATH.with_name('libb2e_bf16.so')}
STORAGE_TORCH_DTYPE = {'f16': torch.float16, 'bf16': torch.bfloat16}
# Which build an encoder family runs on.  With bfloat16 the 12-layer BERT and 33-layer ESM-2 shapes stay well
# inside the 1e-3 cosine tolerance against the fp32 reference; the 32-layer Mistral-7B shape needs half's three extra
# significand bits (tools/drift_report.py measures the drift per layer; tests/test_gpu_config_parity.py holds every
# family to the tolerance at configuration depth).  bench.py's extra.storage_ab times the same GEMM in both builds.
# Qwen3 follows Mistral: Qwen3-Embedding-4B / 8B are 36 layers deep.
# ESM C runs bfloat16, as the reference does: at the esmc-600m shape (36 layers, S = 2048) its pooled rows stay within
# 1 - cos 5.1e-5 of the fp32 restatement (half: 9.6e-7), a twentieth of the tolerance (README, tools/drift_report.py).
# B2E_STORAGE=f16|bf16 overrides for every family.
_STORAGE_BY_ARCH = {'bert': 'bf16', 'esm': 'bf16', 'modernbert': 'bf16', 'mistral': 'f16', 'qwen3': 'f16',
                   'esmc': 'bf16'}


def storage_for_arch(arch: str) -> str:
    import os

    forced = os.environ.get('B2E_STORAGE')
    if forced:
        if forced not in LIB_PATHS:
            raise NativeError(f'B2E_STORAGE={forced!r}: expected one of {sorted(LIB_PATHS)}')
        return forced
    return _STORAGE_BY_ARCH[arch]


def storage_of(dtype: torch.dtype) -> str:
    """The build whose storage type is ``dtype`` (operands of the building-block entry points)."""
    for name, dt in STORAGE_TORCH_DTYPE.items():
        if dt == dtype:
            return name
    raise NativeError(f'no libb2e build stores {dtype}: expected float16 or bfloat16 operands')

ARCH_BERT, ARCH_ESM2, ARCH_MISTRAL, ARCH_MODERNBERT, ARCH_QWEN3, ARCH_ESMC = 0, 1, 2, 3, 4, 5
DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2
POOL_MEAN_REF, POOL_MEAN_PER_ROW, POOL_LAST_TOKEN = 0, 1, 2
EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_RESID, EPI_SWIGLU, EPI_GEGLU = 0, 1, 2, 3, 4

_DTYPE_CODES = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16, torch.float16: DTYPE_F16}

# every symbol include/b2e.h declares (checked by the CPU test-suite)
EXPORTS = (
    'b2e_version',
    'b2e_storage_dtype',
    'b2e_last_error',
    'b2e_num_weights',
    'b2e_check_model',
    'b2e_encoder_create',
    'b2e_encoder_create_nf4',
    'b2e_encoder_create_nf4_lora',
    'b2e_encoder_destroy',
    'b2e_workspace_bytes',
    'b2e_encode',
    'b2e_encode_pooled',
    'b2e_embed_host',
    'b2e_pool_mean',
    'b2e_pool_last_token',
    'b2e_l2_normalize',
    'b2e_adjacent_cosine_dist',
    'b2e_gemm_h16',
    'b2e_gemm_nf4',
    'b2e_gemm_nf4_lora',
    'b2e_attention_d64',
    'b2e_attention_d32',
    'b2e_attention_d64_window',
    'b2e_attention_causal_d128',
    'b2e_qk_norm_rope',
    'b2e_qk_layernorm_rope',
    'b2e_topk_ip',
    'b2e_topk_ip_tc',
    'b2e_max_row_norm',
    'b2e_topk_l2',
    'b2e_topk_l2_tc',
    'b2e_row_norms',
    'b2e_pack_ubinary',
    'b2e_search_ubinary',
    'b2e_layernorm',
)
# profiling hooks declared in include/b2e_debug.h (tools/ only; nothing in the package calls them)
DEBUG_EXPORTS = (
    'b2e_debug_set_att3_clock',
    'b2e_debug_set_clock_buffer',
    'b2e_debug_set_layers',
    'b2e_debug_set_att3_variant',
    'b2e_debug_set_packing',
    'b2e_debug_set_gemm_bn',
    'b2e_debug_gemm_bn',
    'b2e_debug_gemm_rows',
    'b2e_debug_gemm_nf4_lora_rows',
    'b2e_debug_topk_tc_fell_back',
    'b2e_debug_topk_tc_state',
    'b2e_debug_attention_packed',
    'b2e_debug_rotary',
    'b2e_debug_embed',
    'b2e_debug_roberta_positions',
    'b2e_debug_norm',
)


class NativeError(RuntimeError):
    """Raised when libb2e.so is missing or a native call fails."""


class ModelDesc(C.Structure):
    """Mirror of ``B2EModelDesc``."""

    _fields_ = [
        ('arch', C.c_int32),
        ('num_layers', C.c_int32),
        ('hidden', C.c_int32),
        ('heads', C.c_int32),
        ('kv_heads', C.c_int32),
        ('head_dim', C.c_int32),
        ('intermediate', C.c_int32),
        ('vocab', C.c_int32),
        ('max_pos', C.c_int32),
        ('type_vocab', C.c_int32),
        ('eps', C.c_float),
        ('rope_theta', C.c_float),
        ('sliding_window', C.c_int32),
        ('reserved', C.c_int32),
        ('rope_theta_local', C.c_float),
        ('global_every', C.c_int32),
    ]


_libs: dict[str, C.CDLL] = {}


def _declare(lib: C.CDLL) -> None:
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    lib.b2e_version.restype = i32
    lib.b2e_version.argtypes = []
    lib.b2e_storage_dtype.restype = i32
    lib.b2e_storage_dtype.argtypes = []
    lib.b2e_last_error.restype = C.c_char_p
    lib.b2e_last_error.argtypes = []
    lib.b2e_num_weights.restype = i32
    lib.b2e_num_weights.argtypes = [C.POINTER(ModelDesc)]
    lib.b2e_check_model.restype = i32
    lib.b2e_check_model.argtypes = [C.POINTER(ModelDesc)]
    lib.b2e_encoder_create.restype = i32
    lib.b2e_encoder_create.argtypes = [C.POINTER(ModelDesc), C.POINTER(vp), i32, i32, C.POINTER(vp)]
    lib.b2e_encoder_create_nf4.restype = i32
    lib.b2e_encoder_create_nf4.argtypes = [C.POINTER(ModelDesc), C.POINTER(vp), i32, C.POINTER(vp), i32, i32,
                                           C.POINTER(vp)]
    lib.b2e_encoder_create_nf4_lora.restype = i32
    lib.b2e_encoder_create_nf4_lora.argtypes = [C.POINTER(ModelDesc), C.POINTER(vp), i32, C.POINTER(vp), i32,
                                                C.POINTER(vp), C.POINTER(vp), C.POINTER(i32), i32, i32, C.POINTER(vp)]
    lib.b2e_encoder_destroy.restype = None
    lib.b2e_encoder_destroy.argtypes = [vp]
    lib.b2e_workspace_bytes.restype = i64
    lib.b2e_workspace_bytes.argtypes = [vp, i32, i32]
    lib.b2e_encode.restype = i32
    lib.b2e_encode.argtypes = [vp, vp, vp, vp, i32, i32, vp, i32, vp]
    lib.b2e_encode_pooled.restype = i32
    lib.b2e_encode_pooled.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp, vp]
    lib.b2e_embed_host.restype = i32
    lib.b2e_embed_host.argtypes = [vp, vp, vp, vp, i64, i32, i32, i32, i32, vp]
    lib.b2e_pool_mean.restype = i32
    lib.b2e_pool_mean.argtypes = [vp, i32, vp, i32, i32, i32, i32, i32, vp, vp]
    lib.b2e_pool_last_token.restype = i32
    lib.b2e_pool_last_token.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp]
    lib.b2e_l2_normalize.restype = i32
    lib.b2e_l2_normalize.argtypes = [vp, i64, i32, vp]
    lib.b2e_adjacent_cosine_dist.restype = i32
    lib.b2e_adjacent_cosine_dist.argtypes = [vp, i32, i64, i32, vp, vp, vp]
    lib.b2e_gemm_h16.restype = i32
    lib.b2e_gemm_h16.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.b2e_gemm_nf4.restype = i32
    lib.b2e_gemm_nf4.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.b2e_gemm_nf4_lora.restype = i32
    lib.b2e_gemm_nf4_lora.argtypes = [vp, vp, vp, vp, i32, vp, i32, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.b2e_attention_d64.restype = i32
    lib.b2e_attention_d64.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp]
    lib.b2e_attention_d32.restype = i32
    lib.b2e_attention_d32.argtypes = [vp, vp, vp, i32, i32, i32, vp]
    lib.b2e_attention_d64_window.restype = i32
    lib.b2e_attention_d64_window.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp]
    lib.b2e_attention_causal_d128.restype = i32
    lib.b2e_attention_causal_d128.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, vp]
    lib.b2e_qk_norm_rope.restype = i32
    lib.b2e_qk_norm_rope.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, C.c_float, vp, vp, vp]
    lib.b2e_qk_layernorm_rope.restype = i32
    lib.b2e_qk_layernorm_rope.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, C.c_float, vp, vp, vp]
    lib.b2e_topk_ip.restype = i32
    lib.b2e_topk_ip.argtypes = [vp, i32, vp, i32, i64, i32, i32, vp, vp, vp]
    lib.b2e_topk_ip_tc.restype = i32
    lib.b2e_topk_ip_tc.argtypes = [vp, i32, vp, i64, i32, i32, C.c_float, vp, vp, vp]
    lib.b2e_max_row_norm.restype = i32
    lib.b2e_max_row_norm.argtypes = [vp, i64, i32, C.POINTER(C.c_float), vp]
    lib.b2e_topk_l2.restype = i32
    lib.b2e_topk_l2.argtypes = [vp, i32, vp, i64, i32, i32, vp, vp, vp]
    lib.b2e_topk_l2_tc.restype = i32
    lib.b2e_topk_l2_tc.argtypes = [vp, i32, vp, vp, i64, i32, i32, C.c_float, vp, vp, vp]
    lib.b2e_row_norms.restype = i32
    lib.b2e_row_norms.argtypes = [vp, i64, i32, vp, C.POINTER(C.c_float), vp]
    lib.b2e_pack_ubinary.restype = i32
    lib.b2e_pack_ubinary.argtypes = [vp, i64, i32, vp, vp]
    lib.b2e_search_ubinary.restype = i32
    lib.b2e_search_ubinary.argtypes = [vp, i32, vp, i64, i32, i32, i32, vp, vp, vp]
    lib.b2e_layernorm.restype = i32
    lib.b2e_layernorm.argtypes = [vp, vp, vp, vp, i32, i32, C.c_float, i32, vp]


def load(storage: str = 'f16') -> C.CDLL:
    """Load libb2e.so ('f16') or libb2e_bf16.so ('bf16'), once each.  Raises ``NativeError`` when it has not
    been built."""
    if storage in _libs:
        return _libs[storage]
    path = LIB_PATHS[storage]
    if not path.exists():
        raise NativeError(
            f'{path} not found: build it with `python -m distllm_b200.build` '
            '(or __graft_entry__.build()). There is no CPU fallback.',
        )
    try:
        lib = C.CDLL(str(path))
    except OSError as exc:  # pragma: no cover - depends on the box
        raise NativeError(f'cannot load {path}: {exc}') from exc
    _declare(lib)
    want = DTYPE_F16 if storage == 'f16' else DTYPE_BF16
    if lib.b2e_storage_dtype() != want:
        raise NativeError(f'{path} reports storage dtype {lib.b2e_storage_dtype()}, expected {want}')
    _libs[storage] = lib
    return lib


def check(rc: int, lib: C.CDLL | None = None) -> None:
    """Turn a non-zero return code into a NativeError carrying that library's b2e_last_error()."""
    if rc != 0:
        msg = (lib or load()).b2e_last_error()
        raise NativeError(f'libb2e error {rc}: {msg.decode() if msg else "?"}')


def dtype_code(dtype: torch.dtype) -> int:
    try:
        return _DTYPE_CODES[dtype]
    except KeyError:
        raise NativeError(f'unsupported dtype {dtype}') from None


def stream_ptr(device: torch.device | None = None) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def _cuda_contig(t: torch.Tensor, what: str) -> torch.Tensor:
    if not t.is_cuda:
        raise NativeError(f'{what} must be a CUDA tensor (libb2e has no CPU fallback)')
    if not t.is_contiguous():
        raise NativeError(f'{what} must be contiguous')
    return t


# --------------------------------------------------------------------------- thin op wrappers
def gemm_h16(
    a: torch.Tensor,
    w: torch.Tensor,
    bias: torch.Tensor | None,
    resid: torch.Tensor | None = None,
    epilogue: int = EPI_BIAS,
) -> torch.Tensor:
    """out[M,N] = epi(a[M,K] @ w[N,K].T + bias (+ resid)) on the wgmma GEMM; float16 or bfloat16 in/out (the
    matching build of the library is used), fp32 accumulation.  ``EPI_BIAS_RESID`` sums ``acc + bias + resid``
    in fp32; the result is rounded to nearest-even once, and in float16 values beyond +-65504 saturate to
    +-65504 instead of becoming inf.

    ``EPI_SWIGLU``: ``w`` holds gate/up rows interleaved in blocks of 64 (weights.interleave_gate_up)
    and the result is ``silu(gate) * up`` of shape [M, N/2]; ``EPI_GEGLU`` the same with erf-GELU.  The gated
    epilogues take no ``bias``, and only ``EPI_BIAS_RESID`` takes ``resid``: passing one anyway raises
    ``NativeError`` rather than dropping it."""
    if a.dtype != w.dtype:
        raise NativeError(f'gemm_h16: operands differ in dtype ({a.dtype} vs {w.dtype})')
    lib = load(storage_of(a.dtype))
    _cuda_contig(a, 'a'), _cuda_contig(w, 'w')
    if bias is not None:
        _cuda_contig(bias, 'bias')
    m, k = a.shape
    n = w.shape[0]
    n_out = n // 2 if epilogue in (EPI_SWIGLU, EPI_GEGLU) else n
    out = torch.empty((m, n_out), dtype=a.dtype, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.b2e_gemm_h16(a.data_ptr(), w.data_ptr(), _ptr(bias), _ptr(resid),
                               out.data_ptr(), m, n, k, epilogue, stream_ptr(a.device)), lib)
    return out


def gemm_nf4(
    a: torch.Tensor,
    codes: torch.Tensor,
    absmax: torch.Tensor,
    bias: torch.Tensor | None,
    resid: torch.Tensor | None = None,
    epilogue: int = EPI_BIAS,
) -> torch.Tensor:
    """:func:`gemm_h16` with W in NF4 (embed/encoders/nf4.py: nf4_quantize): ``codes`` uint8 [N, K/2] and
    ``absmax`` fp32 [K/64, N].  Equals bit for bit ``gemm_h16`` on the dequantised W in ``a``'s storage type,
    with the same rules for ``bias`` and ``resid``."""
    lib = load(storage_of(a.dtype))
    _cuda_contig(a, 'a'), _cuda_contig(codes, 'codes'), _cuda_contig(absmax, 'absmax')
    if bias is not None:
        _cuda_contig(bias, 'bias')
    m, k = a.shape
    n = codes.shape[0]
    if codes.dtype != torch.uint8 or absmax.dtype != torch.float32:
        raise NativeError('gemm_nf4: codes must be uint8 and absmax float32')
    if tuple(codes.shape) != (n, k // 2) or tuple(absmax.shape) != (k // 64, n):
        raise NativeError(f'gemm_nf4: expected codes [{n}, {k // 2}] and absmax [{k // 64}, {n}] for K = {k}')
    n_out = n // 2 if epilogue in (EPI_SWIGLU, EPI_GEGLU) else n
    out = torch.empty((m, n_out), dtype=a.dtype, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.b2e_gemm_nf4(a.data_ptr(), codes.data_ptr(), absmax.data_ptr(), _ptr(bias), _ptr(resid),
                               out.data_ptr(), m, n, k, epilogue, stream_ptr(a.device)), lib)
    return out


def gemm_nf4_lora(
    a: torch.Tensor,
    codes: torch.Tensor,
    absmax: torch.Tensor,
    u: torch.Tensor,
    b_cat: torch.Tensor,
    bias: torch.Tensor | None,
    resid: torch.Tensor | None = None,
    epilogue: int = EPI_BIAS,
) -> torch.Tensor:
    """:func:`gemm_nf4` plus the low-rank term ``u[:, :R] @ b_cat.T`` inside the same sum (R = ``b_cat.shape[1]``, a
    multiple of 64; ``u`` [M, >= R] may be wider, its row stride is its width).  Equals bit for bit :func:`gemm_h16`
    on ``[a | u[:, :R]]`` and ``[dequant(W) | b_cat]``."""
    lib = load(storage_of(a.dtype))
    for t, what in ((a, 'a'), (codes, 'codes'), (absmax, 'absmax'), (u, 'u'), (b_cat, 'b_cat')):
        _cuda_contig(t, what)
    if bias is not None:
        _cuda_contig(bias, 'bias')
    m, k = a.shape
    n, r = b_cat.shape
    if u.dtype != a.dtype or b_cat.dtype != a.dtype or u.shape[0] != m:
        raise NativeError(f'gemm_nf4_lora: u must be [{m}, >= R] and b_cat [N, R] in {a.dtype}')
    n_out = n // 2 if epilogue in (EPI_SWIGLU, EPI_GEGLU) else n
    out = torch.empty((m, n_out), dtype=a.dtype, device=a.device)
    with torch.cuda.device(a.device):
        check(lib.b2e_gemm_nf4_lora(a.data_ptr(), codes.data_ptr(), absmax.data_ptr(), u.data_ptr(), u.shape[1],
                                    b_cat.data_ptr(), r, _ptr(bias), _ptr(resid), out.data_ptr(), m, n, k,
                                    epilogue, stream_ptr(a.device)), lib)
    return out


def attention_d64(
    qkv: torch.Tensor,
    attention_mask: torch.Tensor,
    batch: int,
    seq: int,
    heads: int,
) -> torch.Tensor:
    """qkv [B*S, 3*heads*64] fp16 -> context [B*S, heads*64] fp16."""
    lib = load(storage_of(qkv.dtype))
    _cuda_contig(qkv, 'qkv'), _cuda_contig(attention_mask, 'attention_mask')
    ctx = torch.zeros((batch * seq, heads * 64), dtype=qkv.dtype, device=qkv.device)
    with torch.cuda.device(qkv.device):
        check(lib.b2e_attention_d64(qkv.data_ptr(), attention_mask.data_ptr(), ctx.data_ptr(), batch,
                                    seq, heads, None, stream_ptr(qkv.device)), lib)
    return ctx


def attention_d32(qkv: torch.Tensor, attention_mask: torch.Tensor, batch: int, seq: int, heads: int) -> torch.Tensor:
    """Head_dim-32 attention (MiniLM / BGE-small / E5-small, ESM-2 150M): qkv [B*S, 3*heads*32] -> [B*S, heads*32]."""
    lib = load(storage_of(qkv.dtype))
    _cuda_contig(qkv, 'qkv'), _cuda_contig(attention_mask, 'attention_mask')
    ctx = torch.zeros((batch * seq, heads * 32), dtype=qkv.dtype, device=qkv.device)
    with torch.cuda.device(qkv.device):
        check(lib.b2e_attention_d32(qkv.data_ptr(), attention_mask.data_ptr(), ctx.data_ptr(), batch, seq, heads,
                                    stream_ptr(qkv.device)), lib)
    return ctx


def attention_d64_window(qkv: torch.Tensor, attention_mask: torch.Tensor, batch: int, seq: int, heads: int,
                         window: int) -> torch.Tensor:
    """Bidirectional sliding-window attention (|i - j| <= window): qkv [B*S, 3*heads*64] fp16 -> [B*S, heads*64]."""
    lib = load(storage_of(qkv.dtype))
    _cuda_contig(qkv, 'qkv'), _cuda_contig(attention_mask, 'attention_mask')
    ctx = torch.zeros((batch * seq, heads * 64), dtype=qkv.dtype, device=qkv.device)
    with torch.cuda.device(qkv.device):
        check(lib.b2e_attention_d64_window(qkv.data_ptr(), attention_mask.data_ptr(), ctx.data_ptr(), batch, seq,
                                           heads, window, stream_ptr(qkv.device)), lib)
    return ctx


def attention_causal_d128(
    qkv: torch.Tensor,
    attention_mask: torch.Tensor,
    batch: int,
    seq: int,
    heads: int,
    kv_heads: int,
    window: int = 0,
) -> torch.Tensor:
    """qkv [B*S, (heads + 2*kv_heads)*128] fp16 (q | k | v, rotary applied) -> [B*S, heads*128] fp16."""
    lib = load(storage_of(qkv.dtype))
    _cuda_contig(qkv, 'qkv'), _cuda_contig(attention_mask, 'attention_mask')
    ctx = torch.zeros((batch * seq, heads * 128), dtype=qkv.dtype, device=qkv.device)
    with torch.cuda.device(qkv.device):
        check(lib.b2e_attention_causal_d128(qkv.data_ptr(), attention_mask.data_ptr(), ctx.data_ptr(),
                                            batch, seq, heads, kv_heads, window, stream_ptr(qkv.device)), lib)
    return ctx


def attention_packed(qkv: torch.Tensor, attention_mask: torch.Tensor, batch: int, seq: int, heads: int,
                     kv_heads: int, head_dim: int, window: int = 0, causal: bool = False) -> torch.Tensor:
    """Debug hook: one attention step in the token layout an encoder derives from the mask (csrc/pack.cuh).  With
    every mask row a non-empty prefix, qkv rows cu[b] + s hold the attended tokens back to back, else qkv is the
    padded [B*S] layout; ctx comes back in the same layout (rows past the last token untouched: zero)."""
    lib = load(storage_of(qkv.dtype))
    _cuda_contig(qkv, 'qkv'), _cuda_contig(attention_mask, 'attention_mask')
    if qkv.shape[0] != batch * seq:
        raise NativeError(f'attention_packed: qkv has {qkv.shape[0]} rows, expected B*S = {batch * seq}')
    i32 = C.c_int
    lib.b2e_debug_attention_packed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, i32, i32, i32, i32, i32, i32,
                                               i32, C.c_void_p]
    ctx = torch.zeros((batch * seq, heads * head_dim), dtype=qkv.dtype, device=qkv.device)
    with torch.cuda.device(qkv.device):
        check(lib.b2e_debug_attention_packed(qkv.data_ptr(), attention_mask.data_ptr(), ctx.data_ptr(), batch, seq,
                                             heads, kv_heads, head_dim, window, int(causal),
                                             stream_ptr(qkv.device)), lib)
    return ctx


def debug_rotary_(enc, layer: int, qkv: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
    """Debug hook: the rotary step of ``layer`` of encoder ``enc`` (embed.encoders.native), in place on qkv
    [B*S, q | k | v columns] in the token layout the encoder derives from ``attention_mask`` (see attention_packed)."""
    lib = enc._lib
    _cuda_contig(qkv, 'qkv'), _cuda_contig(attention_mask, 'attention_mask')
    if attention_mask.dtype != torch.int64:
        raise NativeError('attention_mask must be int64')
    b, s = attention_mask.shape
    if qkv.shape[0] != b * s or qkv.dtype != STORAGE_TORCH_DTYPE[enc.storage]:
        raise NativeError(f'debug_rotary_: qkv must be [B*S = {b * s}, cols] in the encoder storage type')
    lib.b2e_debug_rotary.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    with torch.cuda.device(qkv.device):
        check(lib.b2e_debug_rotary(enc._handle, layer, qkv.data_ptr(), attention_mask.data_ptr(), b, s,
                                   stream_ptr(qkv.device)), lib)
    return qkv


def debug_embed(enc, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                token_type_ids: torch.Tensor | None = None) -> tuple[torch.Tensor | None, torch.Tensor | None]:
    """Debug hook: the embedding step of encoder ``enc`` (embed.encoders.native) in the token layout it derives from
    ``attention_mask`` (see attention_packed): (16-bit rows [B*S, H] or None, fp32 residual stream [B*S, H] or None),
    as the family writes them (BERT the first, ESM-2 / Mistral / Qwen3 the second, ModernBERT both).  Rows the step
    does not write are zero."""
    lib = enc._lib
    for t, what in ((input_ids, 'input_ids'), (attention_mask, 'attention_mask'), (token_type_ids, 'token_type_ids')):
        if t is not None and (_cuda_contig(t, what).dtype != torch.int64 or t.shape != input_ids.shape):
            raise NativeError(f'{what} must be int64 [B, S]')
    b, s = input_ids.shape
    arch, h = enc.desc.arch, enc.desc.hidden
    out16 = (torch.zeros((b * s, h), dtype=STORAGE_TORCH_DTYPE[enc.storage], device=input_ids.device)
             if arch in (ARCH_BERT, ARCH_MODERNBERT) else None)
    xres = torch.zeros((b * s, h), dtype=torch.float32, device=input_ids.device) if arch != ARCH_BERT else None
    lib.b2e_debug_embed.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int] + [C.c_void_p] * 3
    with torch.cuda.device(input_ids.device):
        check(lib.b2e_debug_embed(enc._handle, input_ids.data_ptr(), attention_mask.data_ptr(), _ptr(token_type_ids),
                                  b, s, _ptr(out16), _ptr(xres), stream_ptr(input_ids.device)), lib)
    return out16, xres


def debug_roberta_positions(input_ids: torch.Tensor, padding_idx: int, storage: str = 'f16') -> torch.Tensor:
    """Debug hook: RoBERTa position ids of int64 device ids [B, S] (b2e_debug_roberta_positions) -> int32 [B, S]."""
    lib = load(storage)
    if _cuda_contig(input_ids, 'input_ids').dtype != torch.int64 or input_ids.dim() != 2:
        raise NativeError('input_ids must be int64 [B, S]')
    b, s = input_ids.shape
    pos = torch.empty((b, s), dtype=torch.int32, device=input_ids.device)
    lib.b2e_debug_roberta_positions.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    with torch.cuda.device(input_ids.device):
        check(lib.b2e_debug_roberta_positions(input_ids.data_ptr(), b, s, padding_idx, pos.data_ptr(),
                                              stream_ptr(input_ids.device)), lib)
    return pos


NORM_POST_LN, NORM_ADD_LN, NORM_ADD_RMS = 0, 1, 2   # b2e_debug_norm's kinds


def debug_norm(kind: int, xres: torch.Tensor | None, add: torch.Tensor | None, resid: torch.Tensor | None,
               gamma: torch.Tensor, beta: torch.Tensor | None, eps: float, out_dtype: torch.dtype) -> torch.Tensor:
    """Debug hook: one norm step of the trunks with the caller's gains.  ``NORM_POST_LN``: LayerNorm(add + resid) of
    16-bit rows; ``NORM_ADD_LN`` / ``NORM_ADD_RMS``: ``xres += add`` in place (fp32; ``add`` may be None), then
    LayerNorm / RMSNorm of xres.  Returns [rows, H] in ``out_dtype`` (float32 or the 16-bit storage type)."""
    x = add if kind == NORM_POST_LN else xres
    for t, what in ((xres, 'xres'), (add, 'add'), (resid, 'resid'), (gamma, 'gamma'), (beta, 'beta')):
        if t is not None:
            _cuda_contig(t, what)
    storage = storage_of(add.dtype) if add is not None else storage_of(out_dtype)
    lib = load(storage)
    rows, h = x.shape
    out = torch.empty((rows, h), dtype=out_dtype, device=x.device)
    lib.b2e_debug_norm.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_int, C.c_float,
                                                                         C.c_void_p, C.c_void_p]
    with torch.cuda.device(x.device):
        check(lib.b2e_debug_norm(kind, h, _ptr(xres), _ptr(add), _ptr(resid), gamma.data_ptr(), _ptr(beta),
                                 out.data_ptr(), dtype_code(out_dtype), rows, eps, None, stream_ptr(x.device)), lib)
    return out


def qk_norm_rope_(qkv: torch.Tensor, q_gamma: torch.Tensor, k_gamma: torch.Tensor, cos: torch.Tensor,
                  sin: torch.Tensor, heads: int, kv_heads: int, eps: float, t_real: torch.Tensor | None = None,
                  tok_src: torch.Tensor | None = None) -> torch.Tensor:
    """Qwen3's q/k step in place on qkv [T, (heads + 2*kv_heads)*128] (q | k | v heads): per-head RMSNorm with
    q_gamma / k_gamma (fp32 [128]), then rotary with cos / sin [S, 64] fp32 at position tok_src[t] % S (or t % S).
    ``t_real``: int32 device tensor whose first element replaces T as the row count."""
    lib = load(storage_of(qkv.dtype))
    for t, what in ((qkv, 'qkv'), (q_gamma, 'q_gamma'), (k_gamma, 'k_gamma'), (cos, 'cos'), (sin, 'sin')):
        _cuda_contig(t, what)
    for t, what in ((t_real, 't_real'), (tok_src, 'tok_src')):
        if t is not None and (_cuda_contig(t, what).dtype != torch.int32):
            raise NativeError(f'{what} must be int32')
    if q_gamma.dtype != torch.float32 or k_gamma.dtype != torch.float32 or cos.dtype != torch.float32 \
            or sin.dtype != torch.float32:
        raise NativeError('gains and rotary tables must be float32')
    if qkv.shape[1] != (heads + 2 * kv_heads) * 128 or cos.shape[1] != 64 or q_gamma.numel() != 128 \
            or k_gamma.numel() != 128:
        raise NativeError('qk_norm_rope_: expected qkv [T, (heads + 2*kv_heads)*128], tables [S, 64], gains [128]')
    with torch.cuda.device(qkv.device):
        check(lib.b2e_qk_norm_rope(qkv.data_ptr(), q_gamma.data_ptr(), k_gamma.data_ptr(), cos.data_ptr(),
                                   sin.data_ptr(), qkv.shape[0], cos.shape[0], heads, kv_heads, eps, _ptr(t_real),
                                   _ptr(tok_src), stream_ptr(qkv.device)), lib)
    return qkv


def qk_layernorm_rope_(qkv: torch.Tensor, q_gamma: torch.Tensor, k_gamma: torch.Tensor, cos: torch.Tensor,
                       sin: torch.Tensor, eps: float, t_real: torch.Tensor | None = None,
                       tok_src: torch.Tensor | None = None) -> torch.Tensor:
    """ESM C's q/k step in place on qkv [T, 3H] (q | k | v, H = 960 or 1152): a LayerNorm without bias over the whole
    q row (gain q_gamma, fp32 [H]) and the whole k row (k_gamma), then rotary per 64-wide head with cos / sin [S, 32]
    fp32 at position tok_src[t] % S (or t % S).  ``t_real``: int32 device tensor whose first element replaces T as
    the row count."""
    lib = load(storage_of(qkv.dtype))
    for t, what in ((qkv, 'qkv'), (q_gamma, 'q_gamma'), (k_gamma, 'k_gamma'), (cos, 'cos'), (sin, 'sin')):
        _cuda_contig(t, what)
    for t, what in ((t_real, 't_real'), (tok_src, 'tok_src')):
        if t is not None and (_cuda_contig(t, what).dtype != torch.int32):
            raise NativeError(f'{what} must be int32')
    if any(t.dtype != torch.float32 for t in (q_gamma, k_gamma, cos, sin)):
        raise NativeError('gains and rotary tables must be float32')
    h = qkv.shape[1] // 3
    if qkv.shape[1] != 3 * h or cos.shape[1] != 32 or q_gamma.numel() != h or k_gamma.numel() != h:
        raise NativeError('qk_layernorm_rope_: expected qkv [T, 3H], tables [S, 32], gains [H]')
    with torch.cuda.device(qkv.device):
        check(lib.b2e_qk_layernorm_rope(qkv.data_ptr(), q_gamma.data_ptr(), k_gamma.data_ptr(), cos.data_ptr(),
                                        sin.data_ptr(), qkv.shape[0], cos.shape[0], h, eps, _ptr(t_real),
                                        _ptr(tok_src), stream_ptr(qkv.device)), lib)
    return qkv


def topk_ip(queries: torch.Tensor, corpus: torch.Tensor, k: int,
            max_norm: float | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """Exact inner-product top-k: queries [Q,H] f32, corpus [N,H] f32|bf16 (CUDA) -> (scores [Q,k] f32,
    indices [Q,k] i64), sorted by descending score.  ``max_norm`` (an upper bound of the corpus rows' Euclidean
    norms, see :func:`max_row_norm`) selects the tensor-core scan for a float32 corpus; the results are the same."""
    lib = load()
    _cuda_contig(queries, 'queries'), _cuda_contig(corpus, 'corpus')
    if queries.dtype != torch.float32:
        raise NativeError('queries must be float32')
    q, h = queries.shape
    n = corpus.shape[0]
    scores = torch.empty((q, k), dtype=torch.float32, device=queries.device)
    indices = torch.empty((q, k), dtype=torch.int64, device=queries.device)
    with torch.cuda.device(queries.device):
        if max_norm is not None and corpus.dtype == torch.float32:
            check(lib.b2e_topk_ip_tc(queries.data_ptr(), q, corpus.data_ptr(), n, h, k, float(max_norm),
                                     scores.data_ptr(), indices.data_ptr(), stream_ptr(queries.device)))
        else:
            check(lib.b2e_topk_ip(queries.data_ptr(), q, corpus.data_ptr(), dtype_code(corpus.dtype), n, h, k,
                                  scores.data_ptr(), indices.data_ptr(), stream_ptr(queries.device)))
    return scores, indices


def max_row_norm(matrix: torch.Tensor) -> float:
    """Largest Euclidean row norm of a float32 CUDA matrix (index-build step of the tensor-core search)."""
    lib = load()
    _cuda_contig(matrix, 'matrix')
    if matrix.dtype != torch.float32:
        raise NativeError('max_row_norm expects float32')
    out = C.c_float(0.0)
    with torch.cuda.device(matrix.device):
        check(lib.b2e_max_row_norm(matrix.data_ptr(), matrix.shape[0], matrix.shape[1], C.byref(out),
                                   stream_ptr(matrix.device)))
    return float(out.value)


def topk_l2(queries: torch.Tensor, corpus: torch.Tensor, k: int, norms: torch.Tensor | None = None,
            max_norm: float | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """Exact squared-L2 top-k: queries [Q,H] f32, corpus [N,H] f32 (CUDA) -> (distances [Q,k] f32, indices [Q,k]
    i64), ascending squared Euclidean distance, ties by ascending index, +inf / -1 past N.  ``norms`` and
    ``max_norm`` (both from :func:`row_norms` on this corpus) select the tensor-core scan; the results are the
    same."""
    lib = load()
    _cuda_contig(queries, 'queries'), _cuda_contig(corpus, 'corpus')
    if queries.dtype != torch.float32 or corpus.dtype != torch.float32:
        raise NativeError('topk_l2 expects float32 queries and corpus')
    if (norms is None) != (max_norm is None):
        raise NativeError('topk_l2: pass both norms and max_norm (row_norms) or neither')
    q, h = queries.shape
    n = corpus.shape[0]
    dist = torch.empty((q, k), dtype=torch.float32, device=queries.device)
    indices = torch.empty((q, k), dtype=torch.int64, device=queries.device)
    with torch.cuda.device(queries.device):
        if norms is not None:
            _cuda_contig(norms, 'norms')
            if norms.dtype != torch.float32 or norms.shape != (n,):
                raise NativeError(f'norms must be float32 [{n}]')
            check(lib.b2e_topk_l2_tc(queries.data_ptr(), q, corpus.data_ptr(), norms.data_ptr(), n, h, k,
                                     float(max_norm), dist.data_ptr(), indices.data_ptr(),
                                     stream_ptr(queries.device)))
        else:
            check(lib.b2e_topk_l2(queries.data_ptr(), q, corpus.data_ptr(), n, h, k, dist.data_ptr(),
                                  indices.data_ptr(), stream_ptr(queries.device)))
    return dist, indices


def row_norms(matrix: torch.Tensor) -> tuple[torch.Tensor, float]:
    """(squared Euclidean norm of every row, fp32 [N] on the device; largest row norm) of a float32 CUDA matrix:
    the index-build step of the tensor-core L2 search."""
    lib = load()
    _cuda_contig(matrix, 'matrix')
    if matrix.dtype != torch.float32:
        raise NativeError('row_norms expects float32')
    norms = torch.empty(matrix.shape[0], dtype=torch.float32, device=matrix.device)
    out = C.c_float(0.0)
    with torch.cuda.device(matrix.device):
        check(lib.b2e_row_norms(matrix.data_ptr(), matrix.shape[0], matrix.shape[1], norms.data_ptr(), C.byref(out),
                                stream_ptr(matrix.device)))
    return norms, float(out.value)


def topk_tc_fell_back() -> bool:
    """Whether this thread's last tensor-core search (inner product or L2) had to redo the call with the exact scan
    (debug hook)."""
    lib = load()
    out = C.c_int(0)
    lib.b2e_debug_topk_tc_fell_back.argtypes = [C.POINTER(C.c_int)]
    check(lib.b2e_debug_topk_tc_fell_back(C.byref(out)))
    return bool(out.value)


TC_QUERY_DTYPE = np.dtype([('r', '<f4'), ('eps', '<f4'), ('thr', '<f4'), ('need', '<i4')])


def topk_tc_state(rows: int) -> dict[str, np.ndarray]:
    """The intermediate state of the last pass (<= 16 queries) of this thread's last tensor-core search (debug
    hook): 'scores' [rows, 16] f32 (the TF32 scan), 'meta' [16] records (r, eps, thr, need), 'hist' [16, 2048],
    'cand' [16, 4096] row ids and 'n_cand' [16], all uint32 but the first two.  Synchronises the device."""
    lib = load()
    out = {'scores': np.empty((rows, 16), np.float32), 'meta': np.empty(16, TC_QUERY_DTYPE),
           'hist': np.empty((16, 2048), np.uint32), 'cand': np.empty((16, 4096), np.uint32),
           'n_cand': np.empty(16, np.uint32)}
    lib.b2e_debug_topk_tc_state.argtypes = [C.c_int64] + [C.c_void_p] * 5
    check(lib.b2e_debug_topk_tc_state(rows, *(a.ctypes.data for a in out.values())), lib)
    return out


def pack_ubinary(embeddings: torch.Tensor) -> torch.Tensor:
    """fp32 [N,H] (CUDA) -> uint8 [N,H/8]: bit = value > 0, first dimension in the most significant bit."""
    lib = load()
    _cuda_contig(embeddings, 'embeddings')
    if embeddings.dtype != torch.float32:
        raise NativeError('pack_ubinary expects float32')
    n, h = embeddings.shape
    out = torch.empty((n, h // 8), dtype=torch.uint8, device=embeddings.device)
    with torch.cuda.device(embeddings.device):
        check(lib.b2e_pack_ubinary(embeddings.data_ptr(), n, h, out.data_ptr(), stream_ptr(embeddings.device)))
    return out


def search_ubinary(queries: torch.Tensor, corpus_bits: torch.Tensor, k: int,
                   rescore_multiplier: int = 2) -> tuple[torch.Tensor, torch.Tensor]:
    """Hamming top-(k * rescore_multiplier) over packed bits + float rescoring: (scores [Q,k] f32,
    indices [Q,k] i64), descending score."""
    lib = load()
    _cuda_contig(queries, 'queries'), _cuda_contig(corpus_bits, 'corpus_bits')
    if queries.dtype != torch.float32 or corpus_bits.dtype != torch.uint8:
        raise NativeError('search_ubinary expects float32 queries and a uint8 packed corpus')
    q, h = queries.shape
    n = corpus_bits.shape[0]
    if corpus_bits.shape[1] * 8 != h:
        raise NativeError(f'corpus has {corpus_bits.shape[1] * 8} bits per row, queries have {h} dimensions')
    scores = torch.empty((q, k), dtype=torch.float32, device=queries.device)
    indices = torch.empty((q, k), dtype=torch.int64, device=queries.device)
    with torch.cuda.device(queries.device):
        check(lib.b2e_search_ubinary(queries.data_ptr(), q, corpus_bits.data_ptr(), n, h, k, rescore_multiplier,
                                     scores.data_ptr(), indices.data_ptr(), stream_ptr(queries.device)))
    return scores, indices


def layernorm(
    x: torch.Tensor,
    gamma: torch.Tensor,
    beta: torch.Tensor,
    eps: float,
    out_dtype: torch.dtype | None = None,
) -> torch.Tensor:
    """LayerNorm of a 16-bit matrix; ``out_dtype``: float32 or (default) the input's own 16-bit type."""
    lib = load(storage_of(x.dtype))
    out_dtype = out_dtype or x.dtype
    _cuda_contig(x, 'x')
    rows, h = x.shape
    out = torch.empty((rows, h), dtype=out_dtype, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.b2e_layernorm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), rows,
                                h, eps, dtype_code(out_dtype), stream_ptr(x.device)), lib)
    return out


def pool_mean(
    hidden: torch.Tensor,
    attention_mask: torch.Tensor,
    pool_kind: int = POOL_MEAN_REF,
    mutate_mask: bool = True,
) -> torch.Tensor:
    """Masked mean over the sequence axis; fp32 [B,H].  Rewrites the mask like the reference."""
    lib = load()
    _cuda_contig(hidden, 'hidden'), _cuda_contig(attention_mask, 'attention_mask')
    if attention_mask.dtype != torch.int64:
        raise NativeError('attention_mask must be int64')
    b, s, h = hidden.shape
    out = torch.empty((b, h), dtype=torch.float32, device=hidden.device)
    with torch.cuda.device(hidden.device):
        check(lib.b2e_pool_mean(hidden.data_ptr(), dtype_code(hidden.dtype), attention_mask.data_ptr(),
                                b, s, h, pool_kind, int(mutate_mask), out.data_ptr(),
                                stream_ptr(hidden.device)))
    return out


def pool_last_token(hidden: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
    lib = load()
    _cuda_contig(hidden, 'hidden'), _cuda_contig(attention_mask, 'attention_mask')
    if attention_mask.dtype != torch.int64:
        raise NativeError('attention_mask must be int64')
    b, s, h = hidden.shape
    out = torch.empty((b, h), dtype=torch.float32, device=hidden.device)
    with torch.cuda.device(hidden.device):
        check(lib.b2e_pool_last_token(hidden.data_ptr(), dtype_code(hidden.dtype),
                                      attention_mask.data_ptr(), b, s, h, out.data_ptr(),
                                      stream_ptr(hidden.device)))
    return out


def l2_normalize_(x: torch.Tensor) -> torch.Tensor:
    lib = load()
    _cuda_contig(x, 'x')
    if x.dtype != torch.float32:
        raise NativeError('l2_normalize_ expects fp32')
    n, h = x.shape
    with torch.cuda.device(x.device):
        check(lib.b2e_l2_normalize(x.data_ptr(), n, h, stream_ptr(x.device)))
    return x


def adjacent_cosine_dist(emb: torch.Tensor, doc_id: torch.Tensor | None = None) -> torch.Tensor:
    """fp32 [N-1]: 1 - cos(emb[i], emb[i+1]); NaN where doc_id changes."""
    lib = load()
    _cuda_contig(emb, 'emb')
    n, h = emb.shape
    out = torch.empty((max(n - 1, 0),), dtype=torch.float32, device=emb.device)
    if doc_id is not None:
        _cuda_contig(doc_id, 'doc_id')
        if doc_id.dtype != torch.int32:
            raise NativeError('doc_id must be int32')
    with torch.cuda.device(emb.device):
        check(lib.b2e_adjacent_cosine_dist(emb.data_ptr(), dtype_code(emb.dtype), n, h,
                                           _ptr(doc_id), out.data_ptr(), stream_ptr(emb.device)))
    return out
