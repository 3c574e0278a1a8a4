"""The premises of tests/test_gpu_esmc_exact.py and of the bound in test_gpu_esmc.py::test_qk_layernorm_rope, on the
host: ESM C's Walsh rows normalise exactly at 960 and 1152, the q / k gains separate what a wrong gain, partner or head
would compute, every product of the rotation is exact, zero and constant rows normalise to 0 (and to NaN without eps),
the restated table agrees with esm's formula in fp32, and the random-input bound holds for an fp32 restatement of the
kernel's arithmetic while being at least ten times tighter than the tolerance it replaced."""

from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import rows as R
from tools import oracle_esmc as O

WIDTHS = (960, 1152)
EPS = (1e-12, 1e-5)
f32 = np.float32


@pytest.mark.parametrize('h', WIDTHS)
def test_walsh_rows_normalise_exactly(h):
    """Rows 2^6 p: mean 0 and var + eps = 4^6, fused or not; 2^5 is not enough at 960 with eps 1e-5.  Constant rows
    c and offset rows 2^12 + 2^6 p: fl(fl(H c) fl(1/H)) = c, so x - mean is exact (0 for a constant row)."""
    n = R.esmc_order(h)
    rows = R.esmc_walsh_rows(n - 2, h)
    assert (rows.sum(1) == 0).all() and len({r.tobytes() for r in rows}) == n - 2
    inv_h = float(f32(1) / f32(h))
    for a in (5, 6):
        for eps in EPS:
            ss = h * 4.0 ** a
            fused = float(f32(ss * inv_h + float(f32(eps))))
            apart = float(f32(float(f32(ss * inv_h)) + float(f32(eps))))
            ok = fused == apart == 4.0 ** a
            assert ok or (a, h, eps) == (5, 960, 1e-5), (a, eps)
    for c in (0.0, 1.0, -1024.0, 4096.0):
        assert float(f32(float(f32(h * c)) * inv_h)) == c, c
    g = R.qk_gains(h, 0)
    for eps in EPS:
        y = R.layernorm(np.concatenate([rows, 4096.0 + rows, -4096.0 + rows]), g, 0.0, eps)
        assert np.array_equal(y, np.concatenate([rows / 64.0 * g] * 3))


@pytest.mark.parametrize('h', WIDTHS)
def test_gains_tell_the_columns_apart(h):
    """Signed powers of two 2^-3 .. 2^3 and a few zeros; the exponent differs between q and k, between a column and
    its partner (c + 32), a column of the same half 16 away (a partner lane ^ 2) and the next head."""
    q, k = R.qk_gains(h, 0), R.qk_gains(h, 1)
    for g in (q, k):
        nz = g[g != 0]
        e = np.log2(np.abs(nz))
        assert ((e == np.round(e)) & (e >= -3) & (e <= 3)).all()
        assert len(set(e.tolist())) == 7 and (nz > 0).any() and (nz < 0).any()
        zero = np.flatnonzero(g == 0)
        assert 20 <= len(zero) <= 40
        assert (g[zero ^ 32] != 0).all()            # a zero column's partner shows the table entry alone
    both = (q != 0) & (k != 0)
    assert (np.abs(q[both]) != np.abs(k[both])).all()
    c = np.arange(h)
    for g in (q, k):
        for col, other in ((c, c ^ 32), (c, c ^ 16), (c[:-64], c[64:])):
            m = (g[col] != 0) & (g[other] != 0)
            assert (np.abs(g[col])[m] != np.abs(g[other])[m]).all()


def test_rotation_is_exact_on_power_of_two_rows():
    """Every table entry times every gain is exact in fp32, so rope_exact's one rounding is what the kernel computes
    with or without contraction; and it differs from the separately rounded form nowhere here (checked, not assumed)."""
    cos, sin = (u.numpy() for u in O.rotary_tables(2048))
    y = np.array([2.0 ** e * s for e in range(-3, 4) for s in (1, -1)] + [0.0], np.float32)
    for tab in (cos, sin):
        prod = tab[..., None] * y
        assert np.array_equal(prod.astype(np.float64), tab[..., None].astype(np.float64) * y.astype(np.float64))
    g = np.random.default_rng(0)
    h = 960
    rows = (R.esmc_walsh_rows(40, h) / 64.0 * R.qk_gains(h, 1)).astype(np.float32)
    pos = g.integers(0, 2048, 40)
    got = R.rope_exact(rows, cos, sin, pos).reshape(40, -1, 2, 32)
    y = rows.reshape(40, -1, 2, 32)
    c, s = cos[pos][:, None], sin[pos][:, None]
    apart = np.stack([(y[:, :, 0] * c - y[:, :, 1] * s), (y[:, :, 1] * c + y[:, :, 0] * s)], 2).astype(np.float32)
    assert np.array_equal(got, apart)
    zero = y == 0
    assert zero.any()


def test_zero_and_constant_rows_normalise_to_zero():
    """(0 - 0) * rsqrt(eps) * g = 0: the row-path model's zero q / k rows and the exact test's constant rows give 0;
    without eps, rsqrt(0) = inf and 0 * inf = NaN."""
    for h in WIDTHS:
        for c in (0.0, 1.0, -1024.0, 4096.0):
            x = np.full((1, h), c)
            for eps in EPS:
                assert (R.layernorm(x, R.qk_gains(h, 0), 0.0, eps) == 0).all()
    with np.errstate(divide='ignore', invalid='ignore'):
        assert np.isnan(f32(0) * (f32(1) / np.sqrt(f32(0))))
    assert f32(0) * (f32(1) / np.sqrt(f32(1e-5))) == 0


def test_esm_formula_matches_the_oracle_table():
    """oracle.rows.rotary_table (float64 cos / sin of the fp32 angle) and tools/oracle_esmc.py's fp32 torch table
    agree within the allowance at every position of ESM C's table; the allowance is far below a 16-bit ulp of 1."""
    cos, sin = (u.double().numpy() for u in O.rotary_tables(2048))
    c, s, tau = R.rotary_table(np.arange(2048))
    assert (np.abs(c - cos) <= tau).all() and (np.abs(s - sin) <= tau).all()
    assert tau.max() < 2.0 ** -9
    # the table exponent off by one column (2 (k + 1) / 64) scales the angle by 10000^(-1/32): far outside tau
    inv = 1.0 / 10000.0 ** ((2 * np.arange(32) + 2) / 64)
    wrong = np.cos(np.arange(2048)[:, None] * inv)
    assert (np.abs(wrong - c) > tau)[1:].mean() > 0.9


def random_qk(h: int, t: int):
    """test_gpu_esmc.py::test_qk_layernorm_rope's inputs, built the same way."""
    g = torch.Generator().manual_seed(h + t)
    qkv = torch.randn(t, 3 * h, generator=g) * 3 + torch.randn(t, 1, generator=g)
    qg = (1 + 0.3 * torch.randn(h, generator=g))
    kg = (1 + 0.3 * torch.randn(h, generator=g))
    return qkv, qg.numpy(), kg.numpy()


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
@pytest.mark.parametrize('h', WIDTHS)
def test_random_input_bound(h, storage):
    """The fp32 restatement of the kernel (oracle.rows.qk_layernorm_rope_fp32) stays within
    qk_layernorm_rope_bound of the float64 step on test_qk_layernorm_rope's inputs, with and without the 16-bit
    rounding inside the interval check; the bound is at least ten times below the former tolerance (bf16 rtol 1e-2
    atol 2e-2, f16 rtol 2e-3 atol 4e-3) at every element."""
    dtype = {'f16': torch.float16, 'bf16': torch.bfloat16}[storage]
    tol = (1e-2, 2e-2) if dtype == torch.bfloat16 else (2e-3, 4e-3)
    t = 300
    qkv, qg, kg = random_qk(h, t)
    x = qkv.to(dtype).double().numpy()
    cos, sin = (u.numpy() for u in O.rotary_tables(2048))
    pos = (np.arange(t) * 7) % 2048
    worst = 0.0
    for j, g in ((0, qg), (1, kg)):
        xs = x[:, j * h:(j + 1) * h]
        ref, bound = R.qk_layernorm_rope_bound(xs, g, cos, sin, pos, 1e-5)
        got = R.qk_layernorm_rope_fp32(xs, g, cos, sin, pos, 1e-5).astype(np.float64)
        err = np.abs(got - ref)
        assert (err <= bound).all(), float((err / bound).max())
        worst = max(worst, float((err / bound).max()))
        assert R.interval_check(R.round16(got, dtype), ref, bound, dtype) is None
        assert (bound * 10 <= tol[1] + tol[0] * np.abs(ref)).all()
    assert worst > 2.0 ** -10          # the restatement does round: the check is not vacuous


def test_interval_check_rejects_one_ulp_outside():
    ref = np.array([1.0, 1.5, -3.0])
    bound = np.full(3, 1e-6)
    for dtype in (torch.float16, torch.bfloat16):
        got = R.round16(ref, dtype)
        assert R.interval_check(got, ref, bound, dtype) is None
        ulp = float(torch.finfo(dtype).eps)
        assert R.interval_check(got + np.array([ulp, 0, 0]), ref, bound, dtype) is not None


@pytest.mark.parametrize('h', WIDTHS)
def test_row_path_model_esmc(h):
    """ESM C's row-path model: every matrix zero, its reference the bias-free final LayerNorm of the embedding rows,
    the zero embedding row normalising to 0; ids from the model's own vocabulary."""
    cfg, sd, ref = R.row_path_model('esmc', h)
    assert cfg.vocab_size == R.VOCAB and cfg.hidden_size == h
    assert all(not v.any() for k, v in sd.items() if v.dim() == 2 and k != 'embed.weight')
    ids = torch.arange(R.VOCAB)[None]
    y = ref(ids, torch.ones_like(ids), None, torch.bfloat16)
    assert (y[0, -1] == 0).all() and (np.abs(y[0, :-1]) > 0).all()
