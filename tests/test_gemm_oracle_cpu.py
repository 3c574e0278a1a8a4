"""The premises of the exact-arithmetic GEMM tests (tests/test_gpu_gemm_exact.py), on the host: the exact inputs
meet their bounds, the one-hot matrices cover what they claim, the references round as the kernel does, the gated
reference pairs columns as weights.interleave_gate_up lays them out, and the activation epilogues' arithmetic,
emulated in fp32 with the MUFU approximations off by their documented errors, stays within
oracle.gemm.activation_error_bound for every finite 16-bit input and a dense fp32 sweep."""

from __future__ import annotations

import math

import numpy as np
import pytest
import torch
from scipy.special import erf

from distllm_b200.embed.encoders.weights import interleave_gate_up
from oracle import gemm as og

DTYPES = pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16], ids=['f16', 'bf16'])


@pytest.mark.parametrize('k', [64, 128, 192, 320, 576, 768, 3072, 4096, 14336])
def test_ternary_sums_are_small_integers(k):
    g = torch.Generator().manual_seed(k)
    a, w = og.ternary_pair(48, 40, k, g, torch.float32)
    assert set(a.unique().tolist()) <= {-1.0, 0.0, 1.0} and set(w.unique().tolist()) <= {-1.0, 0.0, 1.0}
    assert ((a != 0).sum(dim=1) == min(k, og.TERNARY_NNZ)).all()
    partial = (a.double()[:, None, :] * w.double()[None, :, :]).cumsum(dim=2)   # every prefix of every dot
    assert partial.abs().max() <= og.TERNARY_NNZ < 2 ** 24
    full = og.exact_product(a, w)
    assert torch.equal(full, partial[:, :, -1]) and torch.equal(full, full.round())
    # exact in fp32 in any order, and in both storage types
    assert torch.equal((a @ w.T).double(), full)
    for dt in (torch.float16, torch.bfloat16):
        assert torch.equal(full.to(dt).double(), full)


@pytest.mark.parametrize('count, k', [(384, 64), (768, 320), (517, 576), (1152, 576), (4096, 256), (768, 768),
                                      (3072, 3072), (640, 640)])
def test_one_hot_rows_cover_every_block_edge_and_swizzle_unit(count, k):
    rows, idx = og.one_hot_rows(count, k, torch.float32)
    assert torch.equal(rows.argmax(dim=1), idx) and torch.equal(rows.sum(dim=1), torch.ones(count))
    hit = set(idx.tolist())
    assert hit == set(range(k)) if count >= k else len(hit) == count
    if count >= k:
        for kb in range(k // og.BLOCK_K):
            assert {64 * kb, 64 * kb + 63} <= hit                      # first and last column of every k-block
            assert {64 * kb + 8 * u for u in range(8)} <= hit          # every 16-byte unit of the 128-byte row
    # neighbouring outputs (one accumulator pair, one 8-column group) read different k-blocks when there are several
    if k > 64:
        blocks = idx // og.BLOCK_K
        assert (blocks[1:] != blocks[:-1]).all()


@DTYPES
def test_value_tables(dtype):
    t = og.value_table(dtype)
    f = t.float()
    assert torch.isfinite(f).all() and t.view(torch.int16).unique().numel() == t.numel()
    if dtype == torch.float16:
        assert t.numel() == 2 * 30 * 1024 and (f.abs() >= 2.0 ** -14).all()
        assert f.max() == og.HALF_MAX and f.min() == -og.HALF_MAX
    else:
        assert t.numel() == 2 * 255 * 128 and (f == 0).sum() == 2 and (f.abs() < og.FLT_MIN).sum() == 2 * 128
    g = torch.Generator().manual_seed(0)
    r = og.random_normals((1000,), dtype, g).float()
    assert (r != 0).all() and torch.isfinite(r).all()


def test_storage_rounding_is_nearest_even_and_half_saturates():
    x = torch.tensor([2049.0, 2051.0, 70000.0, -1e9, float('inf'), 65519.0, 65520.0, 1 + 2.0 ** -11])
    assert og.to_storage(x, torch.float16).float().tolist() == [2048.0, 2052.0, og.HALF_MAX, -og.HALF_MAX,
                                                                 og.HALF_MAX, og.HALF_MAX, og.HALF_MAX, 1.0]
    y = torch.tensor([257.0, 259.0, 3e38, 1 + 2.0 ** -8])
    assert og.to_storage(y, torch.bfloat16).float().tolist() == [256.0, 260.0, float(torch.tensor(3e38)
                                                                                     .bfloat16().float()), 1.0]
    # one rounding after both adds: round16(acc + bias) + resid rounded again gives another value
    acc, bias, resid = torch.tensor([[1.0]]), torch.tensor([2.0 ** -11]), torch.tensor([[2.0 ** -11]])
    once = og.epilogue(acc, bias, resid.half(), torch.float16)
    twice = og.epilogue(og.epilogue(acc, bias, None, torch.float16).float(), None, resid.half(), torch.float16)
    assert once.item() == 1 + 2.0 ** -10 and twice.item() == 1.0


@pytest.mark.parametrize('act', ['gelu', 'silu'])
def test_gated_reference_pairs_columns_as_interleave_gate_up(act):
    g = torch.Generator().manual_seed(1)
    gate, up = torch.randn(192, 64, generator=g), torch.randn(192, 64, generator=g)
    a = torch.randn(5, 64, generator=g)
    f = og.gelu64 if act == 'gelu' else og.silu64
    got = og.gated(og.exact_product(a, interleave_gate_up(gate, up)), f)
    want = f(og.exact_product(a, gate)) * og.exact_product(a, up)
    torch.testing.assert_close(got, want, rtol=0, atol=0)


def test_gelu_fit_error():
    """The fitted erf the GELU epilogue uses, over its whole range, plus the clamped tail 1 - erf(4)."""
    x = np.linspace(0, og.GELU_CLAMP, 2_000_001)
    c = og.GELU_Q
    q = ((c[0] * x * x + c[1]) * x * x + c[2]) * x * x + c[3]
    fit = np.abs(np.tanh(x * q) - erf(x / math.sqrt(2))).max() + (1 - erf(4.0))
    assert 1e-5 < fit <= og.GELU_FIT_ERR, fit


def _sweep(dtype) -> np.ndarray:
    """Every finite 16-bit value, a dense fp32 sweep around the fit range and the clamp, and fp32 magnitudes up to
    the largest fp32 (a bias reaches the epilogue as any fp32 value; in bfloat16 up to its largest finite value:
    above it the output is inf, not saturated)."""
    table = og.value_table(dtype).double().numpy()
    dense = np.linspace(-12, 12, 400_001)
    edge = og.GELU_CLAMP + np.linspace(-1e-3, 1e-3, 2001)
    big = np.geomspace(1e-30, 3.4e38 if dtype == torch.float16 else 3.3895e38, 20_001)
    return np.concatenate([table, dense, edge, -edge, big, -big, [0.0]]).astype(np.float32).astype(np.float64)


def _ref(act64, x, dtype, up=None):
    r = act64(x) * (1 if up is None else up)
    return np.clip(r, -og.HALF_MAX, og.HALF_MAX) if dtype == torch.float16 else r


@DTYPES
@pytest.mark.parametrize('err', [-og.TANH_REL_ERR, 0.0, og.TANH_REL_ERR])
def test_gelu_model_within_bound(dtype, err):
    x = _sweep(dtype)
    stored = og.store(og.gelu_kernel_model(x, err), dtype)
    diff = np.abs(stored - _ref(og.gelu64, x, dtype))
    bound = og.activation_error_bound(x, dtype, 'gelu')
    assert np.isfinite(stored).all()
    bad = diff > bound
    assert not bad.any(), (x[bad][:5], diff[bad][:5], bound[bad][:5])
    # the bound is no looser than it has to be: some inputs use more than half of it
    assert (diff > 0.5 * bound).any()


@DTYPES
@pytest.mark.parametrize('ex2_err, rcp_err', [(-og.EX2_REL_ERR, og.RCP_REL_ERR), (0.0, 0.0),
                                              (og.EX2_REL_ERR, -og.RCP_REL_ERR)])
def test_silu_model_within_bound(dtype, ex2_err, rcp_err):
    x = _sweep(dtype)
    stored = og.store(og.silu_kernel_model(x, ex2_err, rcp_err), dtype)
    diff = np.abs(stored - _ref(og.silu64, x, dtype))
    bound = og.activation_error_bound(x, dtype, 'silu')
    assert np.isfinite(stored).all()
    bad = diff > bound
    assert not bad.any(), (x[bad][:5], diff[bad][:5], bound[bad][:5])


@DTYPES
@pytest.mark.parametrize('kind', ['gelu', 'silu'])
def test_gated_model_within_bound(dtype, kind):
    rng = np.random.default_rng(3)
    g = _sweep(dtype)
    up = og.store(rng.standard_normal(g.size) * np.exp2(rng.integers(-8, 9, g.size)), dtype)
    if kind == 'gelu':
        act = og.gelu_kernel_model(g, og.TANH_REL_ERR)
    else:
        act = og.silu_kernel_model(g, og.EX2_REL_ERR, og.RCP_REL_ERR)
    with np.errstate(over='ignore', invalid='ignore'):
        stored = og.store(act * up.astype(np.float32), dtype)
        ref = _ref(og.gelu64 if kind == 'gelu' else og.silu64, g, dtype, up)
    ok = np.isfinite(ref) & np.isfinite(stored)     # bfloat16: act(3e38) * 256 overflows fp32 on both sides
    bound = og.activation_error_bound(g, dtype, kind, up)
    bad = ok & (np.abs(stored - ref) > bound)
    assert not bad.any(), (g[bad][:5], up[bad][:5])
    assert ok.mean() > 0.99
