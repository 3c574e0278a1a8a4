"""The GEMM's 192-wide tiles (csrc/gemm.cuh, BN = 192) against its 128-wide ones, and the rule that picks between
them (csrc/b2e_api.cu: gemm_bn).

Each output element sums the same k16 products in the same order at either width, so the two kernels must agree
bit for bit: every epilogue that runs 192 wide, with and without bias, at row counts with tails, one- and
many-tile CTAs, both storage builds, and a whole BERT-base encoder on a full-length and a ragged (packed: device row
count far below the grid's) batch.  b2e_debug_set_gemm_bn forces the width of the W maps built after it."""

from __future__ import annotations

import ctypes as C
from contextlib import contextmanager

import pytest
import torch

from distllm_b200 import _native as nv


@contextmanager
def gemm_bn(lib, bn: int):
    lib.b2e_debug_set_gemm_bn.argtypes = [C.c_int]
    assert lib.b2e_debug_set_gemm_bn(bn) == 0
    try:
        yield
    finally:
        lib.b2e_debug_set_gemm_bn(0)


def width(lib, n: int, epi: int, nf4: bool = False) -> int:
    out = C.c_int(-1)
    assert lib.b2e_debug_gemm_bn(n, epi, int(nf4), C.byref(out)) == 0
    return out.value


def test_width_rule():
    """192 where N % 192 == 0 for 16-bit weights and the non-gated epilogues, else 128; the override forces it only
    where the 192-wide kernel exists."""
    lib = nv.load('bf16')
    with gemm_bn(lib, 0):
        for n in (384, 768, 2304, 3072, 3840, 6144):          # MiniLM / BERT-base / ESM-2 650M QKV / Mistral QKV
            for epi in (nv.EPI_BIAS, nv.EPI_BIAS_GELU, nv.EPI_BIAS_RESID):
                assert width(lib, n, epi) == 192, (n, epi)
        for n in (128, 256, 640, 1024, 1280, 4096, 5120, 14336):   # not multiples of 192
            assert width(lib, n, nv.EPI_BIAS) == 128, n
        for epi in (nv.EPI_SWIGLU, nv.EPI_GEGLU):             # gate / up paired within a 128-row W tile
            assert width(lib, 6144, epi) == 128 and width(lib, 28672, epi) == 128
        assert width(lib, 768, nv.EPI_BIAS, nf4=True) == 128   # the NF4 producer dequantises 128 W rows
    with gemm_bn(lib, 128):
        assert width(lib, 768, nv.EPI_BIAS) == 128 and width(lib, 3072, nv.EPI_BIAS_GELU) == 128
    with gemm_bn(lib, 192):
        assert width(lib, 768, nv.EPI_BIAS) == 192
        assert width(lib, 1280, nv.EPI_BIAS) == 128 and width(lib, 6144, nv.EPI_SWIGLU) == 128
    assert lib.b2e_debug_set_gemm_bn(256) != 0


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


ROWS = (1, 127, 517, 20000)   # one row; a single partial row tile; 5 row tiles with a tail; ~38 tiles per CTA


@pytest.mark.gpu
@pytest.mark.parametrize('k', [128, 768, 3072])
@pytest.mark.parametrize('n', [384, 768, 2304, 3072, 3840, 6144])
@pytest.mark.parametrize('h16', [torch.float16, torch.bfloat16], ids=['f16', 'bf16'])
def test_wide_tiles_equal_narrow_bit_for_bit(dev, h16, n, k):
    lib = nv.load(nv.storage_of(h16))
    g = torch.Generator(device=dev).manual_seed(n * 7 + k)
    w = (torch.randn(n, k, device=dev, generator=g) * 0.05).to(h16)
    bias = torch.randn(n, device=dev, generator=g)
    with gemm_bn(lib, 192):
        assert width(lib, n, nv.EPI_BIAS) == 192
    for m in ROWS:
        a = torch.randn(m, k, device=dev, generator=g).to(h16)
        resid = torch.randn(m, n, device=dev, generator=g).to(h16)
        cases = [(nv.EPI_BIAS, bias, None), (nv.EPI_BIAS, None, None), (nv.EPI_BIAS_GELU, bias, None),
                 (nv.EPI_BIAS_GELU, None, None), (nv.EPI_BIAS_RESID, bias, resid), (nv.EPI_BIAS_RESID, None, resid)]
        for epi, b, r in cases:
            got = {}
            for bn in (128, 192):
                with gemm_bn(lib, bn):
                    got[bn] = nv.gemm_h16(a, w, b, r, epi)
            torch.cuda.synchronize()
            assert torch.isfinite(got[128].float()).all()
            assert torch.equal(got[128], got[192]), (m, epi, b is not None)


@pytest.mark.gpu
def test_bert_base_encoder_equal_at_both_widths(dev):
    """encode_pooled at BERT-base depth: every linear layer of the model (QKV 2304, attention-out 768, FFN-up 3072
    with GELU, FFN-down 768) runs 192 wide by default; the pooled rows must be those of the 128-wide kernels."""
    from transformers import BertConfig

    from distllm_b200.embed.encoders.native import NativeBertEncoder
    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    from tools.workloads import BERT_BASE

    lib = nv.load('bf16')
    cfg = BertConfig(**BERT_BASE)
    sd = random_bert_state_dict(cfg, seed=0, device=dev)
    g = torch.Generator().manual_seed(5)
    b, s = 24, 512
    ids = torch.randint(7, cfg.vocab_size, (b, s), generator=g)
    full = torch.ones(b, s, dtype=torch.int64)
    lens = torch.randint(1, s + 1, (b,), generator=g)
    lens[0] = 3
    ragged = (torch.arange(s)[None] < lens[:, None]).long()
    out = {}
    for bn in (128, 192):
        with gemm_bn(lib, bn):
            enc = NativeBertEncoder(cfg, sd, device=dev)
        try:
            for name, mask in (('full', full), ('ragged', ragged)):
                out[bn, name] = enc.encode_pooled((ids * mask).to(dev), mask.to(dev), None, nv.POOL_MEAN_REF,
                                                  False).clone()
        finally:
            enc.close()
    for name in ('full', 'ragged'):
        assert torch.isfinite(out[128, name]).all()
        assert torch.equal(out[128, name], out[192, name]), name
