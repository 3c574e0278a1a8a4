"""The C-ABI shared library: loads on a CPU-only box, exports every symbol include/b2e.h declares,
and refuses to compute without a GPU (there is no CPU fallback)."""

from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

import pytest
import torch

from distllm_b200 import _native

HEADER = Path(__file__).resolve().parents[1] / 'include' / 'b2e.h'
DEBUG_HEADER = HEADER.with_name('b2e_debug.h')


def declared_symbols(header: Path = HEADER) -> list[str]:
    text = re.sub(r'/\*.*?\*/', '', header.read_text(), flags=re.S)
    return sorted(set(re.findall(r'\b(b2e_[a-z0-9_]+)\s*\(', text)))


def test_every_exported_b2e_symbol_is_declared_in_a_header():
    """`nm -D` of the shipped library: the b2e_* dynamic symbols are exactly b2e.h (the reference-facing
    ABI) plus b2e_debug.h (profiling hooks for tools/)."""
    import shutil
    import subprocess

    nm = shutil.which('nm')
    if nm is None:
        pytest.skip('binutils nm not available')
    for path in _native.LIB_PATHS.values():      # both builds (half / bfloat16 storage) export the same ABI
        out = subprocess.run([nm, '-D', '--defined-only', str(path)], capture_output=True, text=True,
                             check=True).stdout
        exported = {line.split()[-1] for line in out.splitlines() if line.split()[-1].startswith('b2e_')}
        assert exported == set(declared_symbols()) | set(declared_symbols(DEBUG_HEADER)), path
    assert set(declared_symbols(DEBUG_HEADER)) == set(_native.DEBUG_EXPORTS)


def test_check_model_rejects_unsupported_shapes_before_any_upload():
    """b2e_check_model needs neither a device nor weights (ADVICE r1: the default ESM-2 checkpoint, H=320
    with 16-wide heads, must fail before its parameters are converted and uploaded)."""
    lib = _native.load()
    ok = _native.ModelDesc(arch=_native.ARCH_ESM2, num_layers=33, hidden=1280, heads=20, kv_heads=20,
                           head_dim=64, intermediate=5120, vocab=33, max_pos=1026)
    assert lib.b2e_check_model(C.byref(ok)) == 0
    big = _native.ModelDesc(arch=_native.ARCH_ESM2, num_layers=36, hidden=2560, heads=40, kv_heads=40,
                            head_dim=64, intermediate=10240, vocab=33, max_pos=1026)
    assert lib.b2e_check_model(C.byref(big)) == 0   # esm2_t36_3B
    tiny = _native.ModelDesc(arch=_native.ARCH_ESM2, num_layers=6, hidden=320, heads=20, kv_heads=20,
                             head_dim=16, intermediate=1280, vocab=33, max_pos=1026)
    assert lib.b2e_check_model(C.byref(tiny)) == 3
    assert b'head_dim 64' in lib.b2e_last_error()
    odd = _native.ModelDesc(arch=_native.ARCH_BERT, num_layers=2, hidden=1536 + 256, heads=28, kv_heads=28,
                            head_dim=64, intermediate=4096, vocab=100, max_pos=64)
    assert lib.b2e_check_model(C.byref(odd)) == 3 and b'hidden size 1792' in lib.b2e_last_error()
    mistral = _native.ModelDesc(arch=_native.ARCH_MISTRAL, num_layers=32, hidden=4096, heads=32, kv_heads=8,
                                head_dim=128, intermediate=14336, vocab=32000, max_pos=4096)
    assert lib.b2e_check_model(C.byref(mistral)) == 0
    mistral.head_dim = 64
    assert lib.b2e_check_model(C.byref(mistral)) == 3
    assert lib.b2e_check_model(None) == 1


def test_header_symbols_all_exported():
    lib = _native.load()
    names = declared_symbols()
    assert len(names) >= 16
    for name in names:
        assert hasattr(lib, name), f'{name} declared in b2e.h but not exported by libb2e.so'
    assert set(names) == set(_native.EXPORTS)


def test_version_and_error_string():
    lib = _native.load()
    assert lib.b2e_version() == 2
    assert isinstance(lib.b2e_last_error(), bytes)


def test_model_desc_layout_matches_header():
    # 16 four-byte fields, no padding
    assert C.sizeof(_native.ModelDesc) == 64


def test_num_weights_bert():
    lib = _native.load()
    desc = _native.ModelDesc(arch=_native.ARCH_BERT, num_layers=12)
    assert lib.b2e_num_weights(C.byref(desc)) == 5 + 12 * 12
    desc.arch = _native.ARCH_ESM2
    assert lib.b2e_num_weights(C.byref(desc)) == 3 + 12 * 12
    desc.arch = _native.ARCH_MISTRAL
    assert lib.b2e_num_weights(C.byref(desc)) == 2 + 6 * 12
    desc.arch = 7
    assert lib.b2e_num_weights(C.byref(desc)) == -1


def test_argument_validation_without_touching_the_gpu():
    lib = _native.load()
    # null pointers / bad shapes are rejected before any CUDA call
    assert lib.b2e_gemm_h16(None, None, None, None, None, 128, 128, 64, 0, None) == 1
    assert b'null' in lib.b2e_last_error()
    assert lib.b2e_adjacent_cosine_dist(None, 0, 1, 768, None, None, None) == 0  # <2 rows: no-op
    assert lib.b2e_encode(None, None, None, None, 1, 1, None, 0, None) == 1


@pytest.mark.skipif(torch.cuda.is_available(), reason='placeholder pointers: CPU-only (the GPU suite uses tensors)')
def test_gemm_rejects_a_bias_or_resid_its_epilogue_does_not_read():
    """Checked before the device is touched: a gated epilogue adds no bias, only B2E_EPI_BIAS_RESID adds resid."""
    fake = C.c_void_p(1 << 20)   # never dereferenced: the arguments are rejected first
    for lib in (_native.load('f16'), _native.load('bf16')):
        for epi in (_native.EPI_SWIGLU, _native.EPI_GEGLU):
            assert lib.b2e_gemm_h16(fake, fake, fake, None, fake, 128, 256, 64, epi, None) == 1
            assert b'no bias' in lib.b2e_last_error()
            assert lib.b2e_gemm_nf4(fake, fake, fake, fake, None, fake, 128, 256, 64, epi, None) == 1
            assert b'no bias' in lib.b2e_last_error()
        for epi in (_native.EPI_BIAS, _native.EPI_BIAS_GELU, _native.EPI_SWIGLU, _native.EPI_GEGLU):
            assert lib.b2e_gemm_h16(fake, fake, None, fake, fake, 128, 256, 64, epi, None) == 1
            assert b'reads no resid' in lib.b2e_last_error()
        # accepted combinations get as far as the device check
        assert lib.b2e_gemm_h16(fake, fake, fake, fake, fake, 128, 256, 64, _native.EPI_BIAS_RESID, None) == 4
        assert lib.b2e_gemm_h16(fake, fake, None, None, fake, 128, 256, 64, _native.EPI_SWIGLU, None) == 4


@pytest.mark.skipif(torch.cuda.is_available(), reason='CPU-only behaviour')
def test_no_cpu_fallback():
    x = torch.zeros(4, 256)
    with pytest.raises(_native.NativeError):
        _native.l2_normalize_(x)
    lib = _native.load()
    buf = (C.c_float * 1024)()
    rc = lib.b2e_l2_normalize(buf, 4, 256, None)
    assert rc == 4, 'expected B2E_ERR_NO_DEVICE on a box without a GPU'
    assert b'no CPU fallback' in lib.b2e_last_error()
    from distllm_b200.embed.poolers.mean import average_pool

    with pytest.raises(_native.NativeError):
        average_pool(torch.zeros(2, 4, 256), torch.ones(2, 4, dtype=torch.int64))


def test_two_builds_differ_only_in_storage_dtype():
    f16, bf16 = _native.load('f16'), _native.load('bf16')
    assert f16.b2e_storage_dtype() == _native.DTYPE_F16 and bf16.b2e_storage_dtype() == _native.DTYPE_BF16
    assert f16.b2e_version() == bf16.b2e_version() == 2
    assert _native.storage_of(torch.float16) == 'f16' and _native.storage_of(torch.bfloat16) == 'bf16'
    with pytest.raises(_native.NativeError):
        _native.storage_of(torch.float32)
    # family -> build: the deep Mistral shape needs half, BERT / ESM-2 run the cooler bfloat16 build
    assert _native.storage_for_arch('mistral') == 'f16' and _native.storage_for_arch('bert') == 'bf16'
