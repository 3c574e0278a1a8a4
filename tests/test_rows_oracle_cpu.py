"""The premises of tests/test_gpu_rows_exact.py, on the host: the exactness claims of oracle/rows.py at every built width,
the references against HF's own normalisations, and that the exact inputs separate the kernels' arithmetic from the
faults it guards against (one-pass variance, a dropped epsilon, a 16-bit residual stream, x * (1 / ||x||))."""

from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import rows as R

EPS = (1e-12, 1e-6, 1e-5)


def fma_round(a: float, b: float, c: float) -> float:
    """fl32(a * b + c) with one rounding (a * b + c exact in float64 here)."""
    return float(np.float32(a * b + c))


@pytest.mark.parametrize('h', R.WIDTHS)
def test_walsh_patterns(h):
    n, _ = R.split_width(h)
    rows = R.walsh_rows(n - 2, h)
    assert (rows.sum(1) == 0).all()
    assert len({r.tobytes() for r in rows}) == n - 2
    g = R.walsh_gain(h, 0)
    assert (g.sum() == 0) and ((rows * g).sum(1) == 0).all()      # products stay balanced: never the constant row
    # the half pass of 384 / 640 reads different gains than the previous pass's columns would give
    if h % 256:
        assert (g[h - 128:] != g[h - 384:h - 256]).any()


@pytest.mark.parametrize('h', R.WIDTHS)
def test_variance_and_mean_are_exact(h):
    """fma(H 4^a, fl(1/H), eps) = 4^a for a >= 5 and every eps the families use; fl(fl(H C) fl(1/H)) = C for the
    offsets the tests use."""
    inv_h = float(np.float32(1) / np.float32(h))
    for a in (5, 6, 7, 8, 9):
        for eps in EPS:
            assert fma_round(h * 4.0 ** a, inv_h, float(np.float32(eps))) == 4.0 ** a, (a, eps)
            assert float(np.float32(np.float32(h * 4.0 ** a * inv_h) + np.float32(eps))) == 4.0 ** a, (a, eps)
    for c in (2.0 ** 10, 1088.0, 2.0 ** 15, -2.0 ** 14, 2.0 ** 16):
        assert float(np.float32(float(np.float32(h * c)) * inv_h)) == c, c
    # a = 4 with eps = 1e-5 is not exact everywhere, which is why the rows are 2^5 p
    bad = [h for h in R.WIDTHS if fma_round(h * 256.0, float(np.float32(1) / np.float32(h)), 1e-5) != 256.0]
    assert bad == [] or all(h % 3 == 0 or h % 5 == 0 for h in bad)


def test_layernorm_matches_torch_and_hf():
    """On exact rows the reference equals torch.layer_norm in float64 rounded to fp32, and HF's MistralRMSNorm in fp32,
    bit for bit."""
    from transformers.models.mistral.modeling_mistral import MistralRMSNorm

    for h in R.WIDTHS:
        n, _ = R.split_width(h)
        x = np.concatenate([R.walsh_rows(n - 2, h), 1024.0 + R.walsh_rows(n - 2, h)])
        gamma, beta = R.walsh_gain(h, 3, -1.0), 4.0 * R.pattern(h, 1)
        for eps in EPS:
            ref = R.layernorm(x, gamma, beta, eps)
            t = torch.nn.functional.layer_norm(torch.from_numpy(x), (h,), torch.from_numpy(gamma),
                                               torch.from_numpy(beta), eps)
            assert np.array_equal(ref, t.float().double().numpy()), (h, eps)
            rms = MistralRMSNorm(h, eps=eps)
            rms.weight.data = torch.from_numpy(gamma).float()
            assert np.array_equal(R.rmsnorm(x[:n - 2], gamma, eps),
                                  rms(torch.from_numpy(x[:n - 2]).float()).detach().double().numpy()), (h, eps)


def warp_row_sum(v: np.ndarray) -> np.ndarray:
    """The row kernels' fp32 reduction of [rows, H]: lane l sums its 8 columns of each 256-column pass in order (the
    off lanes of a half pass hold zeros), then the xor butterfly."""
    rows, h = v.shape
    nv = (h + 255) // 256
    full = np.zeros((rows, nv * 256), np.float32)
    full[:, :h] = v
    lanes = full.reshape(rows, nv, 32, 8)
    acc = np.zeros((rows, 32), np.float32)
    for p in range(nv):
        for e in range(8):
            acc = (acc + lanes[:, p, :, e]).astype(np.float32)
    for o in (16, 8, 4, 2, 1):
        acc = (acc + acc[:, np.arange(32) ^ o]).astype(np.float32)
    return acc[:, :1]


def rsqrt_ulps(v: np.ndarray, ulps: int) -> np.ndarray:
    r = (1.0 / np.sqrt(v.astype(np.float64))).astype(np.float32)
    for _ in range(abs(ulps)):
        r = np.nextafter(r, np.float32(np.inf if ulps > 0 else 0))
    return r


def kernel_layernorm(x, gamma, beta, eps, ulps=0, fault=None):
    """warp_layernorm in numpy fp32, in the kernel's reduction order, with rsqrtf pushed ``ulps`` ulps; ``fault``:
    'one_pass' (E[x^2] - mean^2), 'no_eps', 'fused_mean' (mean contracted into x - mean)."""
    x = np.asarray(x, np.float32)
    f = np.float32
    inv_h = f(1) / f(x.shape[-1])
    s = warp_row_sum(x)
    mean = (s * inv_h).astype(f)
    if fault == 'fused_mean':
        d = (x.astype(np.float64) - s.astype(np.float64) * float(inv_h)).astype(f)
    else:
        d = (x - mean).astype(f)
    if fault == 'one_pass':
        var = (warp_row_sum(x * x) * inv_h - mean * mean).astype(f)
    else:
        var = (warp_row_sum(d * d).astype(np.float64) * float(inv_h)).astype(f)
    e = f(0) if fault == 'no_eps' else f(eps)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = rsqrt_ulps((var + e).astype(f), ulps)
        y = ((d * r).astype(np.float64) * np.asarray(gamma, np.float32) + np.asarray(beta, np.float32)).astype(f)
    return y.astype(np.float64)


def kernel_rmsnorm(x, gamma, eps, ulps=0, fault=None):
    x = np.asarray(x, np.float32)
    f = np.float32
    inv_h = f(1) / f(x.shape[-1])
    ss = warp_row_sum(x * x)
    e = f(0) if fault == 'no_eps' else f(eps)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = rsqrt_ulps((ss.astype(np.float64) * float(inv_h) + float(e)).astype(f), ulps)
        return (np.asarray(gamma, np.float32) * (x * r).astype(f)).astype(np.float64)


def rstd_bound(ref: np.ndarray, beta, ulps: int, dtype=np.float32) -> np.ndarray:
    """|y - ref| allowed when rstd is off by ``ulps`` ulps: |ref - beta| ulps 2^-23 plus one fp32 rounding."""
    return np.abs(ref - beta) * ulps * 2.0 ** -23 + np.abs(ref) * 2.0 ** -24


@pytest.mark.parametrize('h', R.WIDTHS)
def test_kernel_models_meet_the_references_and_faults_do_not(h):
    """The kernel-faithful models equal the exact references on the exact rows (Walsh, constant, large offset; zero
    rows for RMSNorm); with rsqrtf pushed to +-1 and +-2 ulp they stay within the 2-ulp rstd bound (and are no longer
    exact: the device premise test is what makes bit-for-bit comparison valid); a one-pass variance (from H = 1024 on,
    where the offset rows' one-pass sums round), a dropped eps and the mean contracted into x - mean (at widths 3 * 2^k
    and 5 * 2^k) fail them."""
    n, _ = R.split_width(h)
    walsh = R.walsh_rows(n - 2, h)
    const = np.array([[c] * h for c in (0.0, 1.0, -3.0, 1024.0)])
    off = 2.0 ** 15 + walsh
    x = np.concatenate([walsh, const, off])
    gamma, beta = R.walsh_gain(h, 3, -1.0), 4.0 * R.pattern(h, 1) + 2.0
    for eps in EPS:
        ref = R.layernorm(x, gamma, beta, eps)
        assert np.array_equal(kernel_layernorm(x, gamma, beta, eps), ref), (h, eps)
        for ulps in (-2, -1, 1, 2):
            got = kernel_layernorm(walsh, gamma, beta, eps, ulps)
            rw = R.layernorm(walsh, gamma, beta, eps)
            assert not np.array_equal(got, rw)
            assert (np.abs(got - rw) <= rstd_bound(rw, beta, abs(ulps))).all(), (h, eps, ulps)
        assert not np.array_equal(kernel_layernorm(x, gamma, beta, eps, fault='no_eps'), ref)
        if eps == 1e-12 and h % 256 != 0 or h in (768, 1280, 2560) and eps == 1e-12:
            assert not np.array_equal(kernel_layernorm(const, gamma, beta, eps, fault='fused_mean'),
                                      R.layernorm(const, gamma, beta, eps)), h
        if h % 256 == 0 and h >= 1024:
            assert not np.array_equal(kernel_layernorm(off, 1.0, 0.0, eps, fault='one_pass'),
                                      R.layernorm(off, 1.0, 0.0, eps)), (h, eps)
        xr = np.concatenate([walsh, np.zeros((1, h))])
        rr = R.rmsnorm(xr, gamma, eps)
        assert np.array_equal(kernel_rmsnorm(xr, gamma, eps), rr), (h, eps)
        for ulps in (-2, 2):
            got = kernel_rmsnorm(walsh, gamma, eps, ulps)
            assert (np.abs(got - rr[:-1]) <= rstd_bound(rr[:-1], 0.0, abs(ulps))).all()
        assert np.isnan(kernel_rmsnorm(xr, gamma, eps, fault='no_eps')[-1]).all()     # zero row: 0 * inf


def test_residual_stream_offsets_do_not_survive_16_bits():
    """The ESM-2 row-path model's residual stream reaches 2^16 +- 32, which neither 16-bit type holds: a residual
    stream stored through 16 bits changes the final norm's input."""
    xres = 2.0 ** 16 + R.walsh_rows(4, 768)
    for dtype in (torch.float16, torch.bfloat16):
        assert not np.array_equal(R.round16(xres, dtype), xres), dtype
    assert sum(R.ESM_BIASES[:3]) == 2.0 ** 16


def test_l2_rows_separate_division_from_reciprocal():
    """The integer rows of test_l2_normalize_divides have exact sums of squares, and x / ||x|| differs from
    x * (1 / ||x||) on them: the parent's reciprocal form fails that test."""
    for h in R.WIDTHS + (4, 132):
        x = R.l2_test_rows(h)
        exp = R.l2_exact(x)
        ss = (x.astype(np.float64) ** 2).sum(-1)
        norm = np.maximum(np.sqrt(ss.astype(np.float32)), R.L2_EPS)[:, None]
        assert np.array_equal(exp, x / norm)
        if h >= 132:
            assert (x * (np.float32(1) / norm) != exp).any(), h


def test_finalize_l2_model_and_fma():
    """fma32 is exactly rounded (checked against exact rationals), and finalize_l2 equals the exact formula on rows
    whose sum of squares fp32 holds."""
    from fractions import Fraction

    g = np.random.default_rng(0)
    a = g.standard_normal(2000).astype(np.float32)
    b = g.standard_normal(2000).astype(np.float32)
    c = (g.standard_normal(2000) * 1e-3).astype(np.float32)
    got = R.fma32(a, b, c)
    for i in range(2000):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.uint32)) & 1))
        assert got[i] == best, i
    x = g.integers(-7, 8, (5, 768)).astype(np.float32)
    assert np.array_equal(R.finalize_l2(x), R.l2_exact(x))


def test_row_path_models_stay_exact():
    """Every family at every width: the reference of the row-path encoder is inside the exact domain (layernorm /
    rmsnorm / mean_pool raise otherwise), for both 16-bit types, at S = 129."""
    for fam, widths in R.FAMILY_WIDTHS.items():
        for h in widths:
            for live in (('word', 'pos', 'type') if fam == 'bert' else ('word',)):
                _, _, ref = R.row_path_model(fam, h, live)
                s = 129
                mask = (torch.arange(s)[None] < torch.tensor([s, 64, 2, 1])[:, None]).long()
                ids = torch.randint(0, R.VOCAB, (4, s), generator=torch.Generator().manual_seed(h))
                types = (torch.arange(s)[None] % 2).expand(4, s).contiguous()
                for dtype in (torch.float16, torch.bfloat16):
                    y = ref(ids, mask, types, dtype)
                    for kind in ('ref', 'per_row'):
                        R.finalize_l2(R.mean_pool(y, R.pool_weights(mask, kind)))
                    R.l2_exact(R.last_token(y, mask))
