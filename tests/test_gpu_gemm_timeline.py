"""The GEMM's timeline instantiation (selected while b2e_debug_set_clock_buffer is set) for the bias and bias + GELU
epilogues at both tile widths: it stamps consumer 0's epilogues (start before end, one pair per tile of CTA 0) and
gives the production kernel's results bit for bit, tail row tile included."""
import ctypes

import pytest
import torch

from distllm_b200 import _native as nv

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('bn', [128, 192])
@pytest.mark.parametrize('epi', ['BIAS', 'BIAS_GELU'])
def test_epilogue_stamps_and_same_bits(epi, bn):
    dev = torch.device('cuda:0')
    lib = nv.load('bf16')
    lib.b2e_debug_set_clock_buffer.argtypes = [ctypes.c_void_p]
    lib.b2e_debug_set_gemm_bn.argtypes = [ctypes.c_int]
    g = torch.Generator(device=dev).manual_seed(5)
    m, n, k = 128 * 132 * 4 + 77, 1536, 768   # four row tiles per CTA, then a tail row tile
    a = (torch.randn(m, k, device=dev, generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(n, k, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(n, device=dev, generator=g)
    code = getattr(nv, f'EPI_{epi}')
    buf = torch.zeros(4, 256, dtype=torch.int64, device=dev)
    try:
        assert lib.b2e_debug_set_gemm_bn(bn) == 0
        want = nv.gemm_h16(a, w, bias, None, code).clone()
        assert lib.b2e_debug_set_clock_buffer(buf.data_ptr()) == 0
        got = nv.gemm_h16(a, w, bias, None, code).clone()
        torch.cuda.synchronize()
    finally:
        lib.b2e_debug_set_clock_buffer(None)
        lib.b2e_debug_set_gemm_bn(0)
    assert torch.equal(got, want)
    start, end = buf[2], buf[3]
    tiles = int((start != 0).sum())
    assert tiles >= 2 and int((end != 0).sum()) == tiles
    assert bool((end[:tiles] > start[:tiles]).all())
