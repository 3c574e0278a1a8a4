"""Inputs whose row-kernel outputs are known bit for bit, and the references they are judged by.  TEST
INFRASTRUCTURE ONLY.

The row kernels (csrc/rowops.cuh, csrc/mistral_ops.cuh) normalise, gather and pool rows in fp32.  Their outputs are
known exactly when every intermediate value is exact:

* Walsh sign patterns.  ``pattern(H, k)`` is row k of the Sylvester-Hadamard matrix of the power-of-two factor n of H
  (H = n * {1, 3, 5}), Kronecker-multiplied by a fixed +-1 row of length 3 or 5 (``ODD_SIGNS``).  A pattern with
  k != 0 has mean exactly 0; the elementwise product of patterns k and k' is pattern k ^ k' (up to the odd factor,
  whose square is all ones).  Rows are 2^a * pattern(H, r) with 0 < r < n/2, gains 2^j * pattern(H, n/2): an output
  pattern never collapses to the constant row along a chain of norms.
* Sum of squares.  A row 2^a * p has sum of squares H * 4^a, exact in fp32, and the kernels' ``ss * fl(1/H) + eps``
  (one fused multiply-add) rounds to exactly 4^a for a >= 5 at every built H and eps <= 1e-5
  (tests/test_rows_oracle_cpu.py checks this).  The mean of ``C + 2^a p`` is ``fl(fl(H C) fl(1/H)) = C`` for a power
  of two C, so the two-pass variance is exact on large offsets, where a one-pass E[x^2] - mean^2 is not.
* rstd.  Outputs are then exact PROVIDED ``rsqrtf(4^a)`` returns 2^-a.  The CUDA math library documents rsqrtf only
  to 2 ulp; every bit-for-bit family of tests/test_gpu_rows_exact.py rests on this premise, and that file's first
  test establishes it on the device (+-2^a rows, gamma 1, beta 0 normalise to exactly +-1).
* Pooling.  Outputs of the form +-2^j +- 2^k sum exactly over any number of rows in any order, so a pooled numerator
  is an exact fp32 value and the mean is one IEEE division; the l2 reference divides as F.normalize does.

``layernorm`` / ``rmsnorm`` follow the kernels' fp32 steps and raise ``ValueError`` on a row outside this exact
domain rather than return a value the device need not match.  ``finalize_l2`` replays pool_finalize_kernel's
sum-of-squares order (256 threads, fused multiply-adds, warp butterflies, eight warp partials) with an exact fp32
FMA, so an l2-normalised mean is known bit for bit too.

Known deviation, not reached by these tests: with token dropout, esm_embed_kernel computes w * (0.88 / (1 - r)) where
HF (and oracle/esm.py) compute (w * 0.88) / (1 - r); the two differ by an fp32 ulp in about 30 % of values.  The
row-path models here run ESM-2 with token dropout off.
"""

from __future__ import annotations

import numpy as np
import torch

from oracle import pooling as opool

WIDTHS = (256, 384, 512, 640, 768, 1024, 1280, 2048, 2560, 4096)
ODD_SIGNS = {1: (1.0,), 3: (1.0, 1.0, -1.0), 5: (1.0, -1.0, 1.0, 1.0, -1.0)}
ROW_SCALE = 5            # rows 2^5 * pattern: eps <= 1e-5 vanishes in var + eps at every built width
POOL_EPS = np.float32(1e-9)
L2_EPS = np.float32(1e-12)

f32 = np.float32


def split_width(h: int) -> tuple[int, int]:
    """H = n * odd with n a power of two and odd in {1, 3, 5}."""
    for odd in (1, 3, 5):
        n = h // odd
        if h % odd == 0 and n & (n - 1) == 0:
            return n, odd
    raise ValueError(f'width {h} is not 2^k * {{1, 3, 5}}')


def walsh(n: int, k: int) -> np.ndarray:
    """Row k of the Sylvester-Hadamard matrix of order n: (-1)^popcount(k & c)."""
    c = np.arange(n)
    bits = np.zeros(n, dtype=np.int64)
    x = c & k
    while x.any():
        bits += x & 1
        x >>= 1
    return np.where(bits % 2 == 0, 1.0, -1.0)


def pattern(h: int, k: int) -> np.ndarray:
    """+-1 float64 row of width h: ODD_SIGNS[odd] (x) walsh(n, k), column i * n + c = sign_i * walsh_c."""
    n, odd = split_width(h)
    return np.kron(np.asarray(ODD_SIGNS[odd]), walsh(n, k))


def row_index(i: int, h: int) -> tuple[int, float]:
    """(Walsh index in [1, n/2), sign) of the i-th distinct row: indices first, then their negatives."""
    n, _ = split_width(h)
    m = n // 2 - 1
    return 1 + i % m, (1.0 if (i // m) % 2 == 0 else -1.0)


def walsh_rows(count: int, h: int, a: int = ROW_SCALE) -> np.ndarray:
    """[count, h] float64: row i = 2^a * sign_i * pattern(h, index_i) (distinct for i < n - 2)."""
    out = np.empty((count, h))
    for i in range(count):
        k, s = row_index(i, h)
        out[i] = s * 2.0 ** a * pattern(h, k)
    return out


def walsh_gain(h: int, j: int, sign: float = 1.0) -> np.ndarray:
    """A gain 2^j * sign * pattern(h, n/2): it maps row index r to r ^ n/2, never to the constant row."""
    n, _ = split_width(h)
    return sign * 2.0 ** j * pattern(h, n // 2)


# ------------------------------------------------------------------------------------------- exactness guards
def _r32(x) -> np.ndarray:
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def dyadic_exact(x: np.ndarray, axis: int = -1) -> bool:
    """Whether every partial sum of x along ``axis``, in any order, is exact in fp32: all values are integer
    multiples of one power of two 2^k, and the sum of their magnitudes is below 2^24 such units."""
    x = np.abs(np.asarray(x, np.float64))
    m, e = np.frexp(x)
    mant = (m * 2.0 ** 53).astype(np.int64)
    low = np.log2(np.where(mant == 0, 1, mant & -mant)).astype(np.int64)
    unit = np.where(x != 0, e - 53 + low, 1000).min(axis, keepdims=True)     # lowest set bit along the axis
    return bool(np.all(np.sum(x / 2.0 ** unit, axis=axis) < 2.0 ** 24))


def _power_of_four_root(v: np.ndarray) -> np.ndarray:
    """2^-a where v = 4^a; NaN elsewhere."""
    m, e = np.frexp(v)                       # v = m 2^e, m in [0.5, 1)
    ok = (m == 0.5) & ((e - 1) % 2 == 0)
    return np.where(ok, np.ldexp(1.0, -((e - 1) // 2)), np.nan)


def _rstd(v: np.ndarray, zero_rows: np.ndarray) -> np.ndarray:
    r = _power_of_four_root(v)
    bad = np.isnan(r) & ~zero_rows
    if bad.any():
        raise ValueError(f'var + eps = {v[bad][:4]}: not a power of four, rsqrt is not exact there')
    return np.where(np.isnan(r), 1.0, r)


# ------------------------------------------------------------------------------------------- norms
def layernorm(x, gamma, beta, eps: float) -> np.ndarray:
    """warp_layernorm on exact rows: mean = fl(sum * fl(1/H)), d = x - mean, rstd = rsqrt(fma(sum d^2, fl(1/H),
    eps)), y = fma(d * rstd, gamma, beta).  float64 holding fp32 values; raises outside the exact domain."""
    x = np.asarray(x, np.float64)
    h = x.shape[-1]
    inv_h = float(f32(1) / f32(h))
    if not dyadic_exact(x):
        raise ValueError('row sums are not exact in fp32')
    mean = _r32(x.sum(-1, keepdims=True) * inv_h)
    d = _r32(x - mean)
    if not dyadic_exact(d * d):
        raise ValueError('sums of squares are not exact in fp32')
    v = _r32((d * d).sum(-1, keepdims=True) * inv_h + float(f32(eps)))
    rstd = _rstd(v, (d == 0).all(-1, keepdims=True))
    return _r32(d * rstd * np.asarray(gamma, np.float64) + np.asarray(beta, np.float64))


def rmsnorm(x, gamma, eps: float) -> np.ndarray:
    """warp_rmsnorm on exact rows: y = gamma * (x * rsqrt(fma(sum x^2, fl(1/H), eps)))."""
    x = np.asarray(x, np.float64)
    h = x.shape[-1]
    inv_h = float(f32(1) / f32(h))
    if not dyadic_exact(x * x):
        raise ValueError('sums of squares are not exact in fp32')
    v = _r32((x * x).sum(-1, keepdims=True) * inv_h + float(f32(eps)))
    r = _rstd(v, (x == 0).all(-1, keepdims=True))
    return _r32(np.asarray(gamma, np.float64) * _r32(x * r))


def round16(x, dtype: torch.dtype) -> np.ndarray:
    """Round to the 16-bit type (nearest-even) and back to float64."""
    return torch.from_numpy(np.asarray(x, np.float64)).to(dtype).double().numpy()


# ------------------------------------------------------------------------------------------- pooling
def pool_weights(mask: torch.Tensor, kind: str) -> np.ndarray:
    """Weights [B, S] of the mean poolers.  'ref': what oracle.pooling.average_pool leaves in the mask (column 0 and
    every sequence's last column cleared in every row); 'per_row': column 0 and the row's own last token cleared."""
    m = mask.clone()
    if kind == 'ref':
        opool.average_pool(torch.zeros(*m.shape, 1, dtype=torch.float64), m)
        return m.double().numpy()
    w = m.double()
    s = w.shape[1]
    w[:, 0] = 0
    for i, n in enumerate(mask.sum(1).tolist()):
        w[i, n - 1 if n > 0 else s - 1] = 0
    return w.numpy()


def mean_pool(y: np.ndarray, w: np.ndarray) -> np.ndarray:
    """fp32 [B, H]: (sum_s w y) / max(count, 1e-9), the numerator exact, one IEEE division."""
    num = np.einsum('bs,bsh->bh', w, y)
    if not dyadic_exact(w[:, :, None] * y, axis=1):
        raise ValueError('pooled numerator is not exact in fp32')
    count = np.maximum(w.sum(1, dtype=np.float64).astype(np.float32), POOL_EPS)
    return num.astype(np.float32) / count[:, None]


def last_token(y: np.ndarray, mask: torch.Tensor) -> np.ndarray:
    """oracle.pooling.last_token_pool: column S-1 when every row's last mask entry is set, else len - 1."""
    return opool.last_token_pool(torch.from_numpy(y), mask.clone()).numpy().astype(np.float32)


def fma32(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
    """fmaf(a, b, c) on float32 arrays, exactly: a*b is exact in float64, the error of the float64 sum is recovered
    (two-sum) and breaks the ties where the float64 sum sits on an fp32 rounding midpoint."""
    a, b, c = (np.asarray(t, np.float32) for t in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)
    r = s.astype(np.float32)
    up, dn = np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(-np.inf))
    r64 = r.astype(np.float64)
    r = np.where((s == (r64 + up.astype(np.float64)) / 2) & (e > 0), up, r)
    r = np.where((s == (r64 + dn.astype(np.float64)) / 2) & (e < 0), dn, r)
    return r


def finalize_l2(v: np.ndarray, threads: int = 256) -> np.ndarray:
    """pool_finalize_kernel's l2 step on fp32 rows v [B, H]: thread t accumulates fmaf(v, v, ss) over columns
    t, t + 256, ...; warp butterflies (xor 16 .. 1); lane 0 of each warp; the eight partials summed in order; then
    v / max(sqrtf(total), 1e-12)."""
    v = np.asarray(v, np.float32)
    b, h = v.shape
    ss = np.zeros((b, threads), np.float32)
    for c0 in range(0, h, threads):
        cols = v[:, c0:c0 + threads]
        ss[:, :cols.shape[1]] = fma32(cols, cols, ss[:, :cols.shape[1]])
    x = ss.reshape(b, threads // 32, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        x = (x + x[..., lane ^ o]).astype(np.float32)
    tot = np.zeros(b, np.float32)
    for i in range(threads // 32):
        tot = (tot + x[:, i, 0]).astype(np.float32)
    return v / np.maximum(np.sqrt(tot), L2_EPS)[:, None]


def l2_test_rows(h: int) -> np.ndarray:
    """37 integer rows of width h (|x| <= 7: exact sums of squares), one all zero (0 / 1e-12 = 0) and one with a
    single non-zero element."""
    g = np.random.default_rng(h)
    x = g.integers(-7, 8, (37, h)).astype(np.float32)
    x[3] = 0.0
    x[4] = 0.0
    x[4, h - 1] = 3.0
    return x


def l2_exact(x: np.ndarray) -> np.ndarray:
    """x / max(||x||, 1e-12) for rows whose sum of squares is exact in fp32 (any summation order gives it)."""
    x = np.asarray(x, np.float32)
    sq = x.astype(np.float64) ** 2
    if not dyadic_exact(sq):
        raise ValueError('sum of squares is not exact in fp32')
    ss = sq.sum(-1).astype(np.float32)
    return x / np.maximum(np.sqrt(ss), L2_EPS)[:, None]


# ------------------------------------------------------------------------------------------- ESM C
# ESM C's widths are not 2^k * {1, 3, 5}: 960 = 15 x 64 and 1152 = 9 x 128, the odd factor's signs the Kronecker
# product of two of ODD_SIGNS' rows.  Rows are 2^6 * pattern: var + eps rounds to 4^6 at both widths for eps 1e-12 and
# 1e-5, fused or not (2^5 is not enough at 960 with eps 1e-5; tests/test_esmc_exact_cpu.py).
ODD = {960: (3, 5), 1152: (3, 3)}
ESMC_SCALE = 6
ESMC_HEAD = 64


def esmc_pattern(h: int, k: int) -> np.ndarray:
    a, b = ODD[h]
    n = h // (a * b)
    return np.kron(np.kron(ODD_SIGNS[a], ODD_SIGNS[b]), walsh(n, k))


def esmc_order(h: int) -> int:
    """n, the Walsh order of an ESM C width."""
    return h // (ODD[h][0] * ODD[h][1])


def esmc_walsh_rows(count: int, h: int, a: int = ESMC_SCALE) -> np.ndarray:
    """[count, h]: row i = 2^a * sign_i * esmc_pattern(h, index_i), distinct for i < n - 2 (as walsh_rows)."""
    m = esmc_order(h) // 2 - 1
    return np.stack([(1.0 if (i // m) % 2 == 0 else -1.0) * 2.0 ** a * esmc_pattern(h, 1 + i % m)
                     for i in range(count)])


def esmc_gain(h: int, j: int, sign: float = 1.0) -> np.ndarray:
    return sign * 2.0 ** j * esmc_pattern(h, esmc_order(h) // 2)


def qk_gains(h: int, which: int) -> np.ndarray:
    """q_ln (which 0) or k_ln (1) gains of ESM C's fused q / k step: signed powers of two 2^-3 .. 2^3 whose exponent
    changes between q and k, between the two halves of a head (c, c + 32) and between heads (c, c + 64) -- a swapped
    gain, a wrong partner or a wrong head changes the bits -- and a few zeros, whose partners' outputs are then the
    table entries alone."""
    c = np.arange(h)
    e = (5 * c + 3 * (c // ESMC_HEAD) + 2 * (c % ESMC_HEAD >= 32) + 4 * which) % 7 - 3
    sign = np.where(((3 * c + c // ESMC_HEAD + which) // 2) % 2 == 0, 1.0, -1.0)
    g = sign * 2.0 ** e
    g[(c + 13 * which) % 37 == 5] = 0.0
    return g


def rope_exact(y, cos, sin, pos) -> np.ndarray:
    """The halves rotation of fp32 rows y [T, W] (64-wide heads) at positions pos with the fp32 tables cos / sin
    [S, 32], for rows whose every product with the table is exact in fp32 (powers of two, 0): round32(y1 c - y2 s),
    round32(y2 c + y1 s) -- one rounding, whether or not the products are contracted into fmas.  float32 [T, W]."""
    y = np.asarray(y, np.float32)
    t, w = y.shape
    y = y.reshape(t, w // ESMC_HEAD, 2, ESMC_HEAD // 2)
    c = np.asarray(cos, np.float32)[pos][:, None, :]
    s = np.asarray(sin, np.float32)[pos][:, None, :]
    y1, y2 = y[:, :, 0], y[:, :, 1]
    p2s, p1s = y2 * s, y1 * s
    for a, b, p in ((y2, s, p2s), (y1, s, p1s)):
        if not np.array_equal(p.astype(np.float64), a.astype(np.float64) * b.astype(np.float64)):
            raise ValueError('a product of the rotation is not exact in fp32')
    return np.stack([fma32(y1, c, -p2s), fma32(y2, c, p1s)], 2).reshape(t, w)


def rotary_table(pos, base: float = 10000.0, d: int = ESMC_HEAD):
    """The fp32 rotary table of HF's rotary embeddings and of esm's (esm/layers/rotary.py of the esm package),
    restated from their documented behaviour: inv_freq = 1 / base^(arange(0, d, 2) / d) in fp32, the angle the fp32
    product position * inv_freq, then cos and sin.  Returns float64 (cos, sin, tau) [len(pos), d/2]: tau allows the
    device's table 8 fp32 ulps of the angle plus 8 of the result (tests/test_gpu_rows_exact.py's rotary_reference
    uses it too)."""
    inv = 1.0 / (torch.tensor(base, dtype=torch.float32) ** (torch.arange(0, d, 2).float() / d))
    ang = (torch.from_numpy(np.asarray(pos, np.float32))[:, None] * inv[None]).double().numpy()
    return np.cos(ang), np.sin(ang), np.abs(ang) * 2.0 ** -20 + 2.0 ** -21


def warp_butterfly(v: np.ndarray) -> np.ndarray:
    """warp_sum over the last axis (32 lanes) in fp32: v += shfl_xor(v, o) for o = 16 .. 1."""
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lane ^ o]).astype(np.float32)
    return v[..., 0]


def qk_layernorm_rope_fp32(x, gamma, cos, sin, pos, eps: float) -> np.ndarray:
    """qk_layernorm_rope_kernel's fp32 arithmetic on one side (the q or the k rows x [T, H]) restated on the host:
    each lane's sum over its columns in pass order, the warp butterfly, mean = fl(sum * fl(1/H)); fmaf sums of
    squares of x - mean over the on lanes, var = fma(ss, fl(1/H), eps), rstd correctly rounded (rsqrtf is within 2
    ulp), y = fl(fl((x - mean) rstd) g); the rotation with contracted products.  float32 [T, H]."""
    x = np.asarray(x, np.float32)
    t, h = x.shape
    nv = (h + 255) // 256
    pad = np.zeros((t, nv * 256), np.float32)
    pad[:, :h] = x
    lanes = pad.reshape(t, nv, 32, 8).transpose(0, 2, 1, 3).reshape(t, 32, nv * 8)
    on = np.zeros(nv * 256, bool)
    on[:h] = True
    on = on.reshape(nv, 32, 8).transpose(1, 0, 2).reshape(32, nv * 8)
    inv_h = np.float32(1) / np.float32(h)
    s = np.zeros((t, 32), np.float32)
    for k in range(nv * 8):
        s = (s + lanes[:, :, k]).astype(np.float32)
    mean = (warp_butterfly(s) * inv_h).astype(np.float32)[:, None, None]
    d = (lanes - mean).astype(np.float32)
    ss = np.zeros((t, 32), np.float32)
    for k in range(nv * 8):
        ss = np.where(on[:, k], fma32(d[:, :, k], d[:, :, k], ss), ss)
    var = fma32(warp_butterfly(ss), inv_h, np.float32(eps))
    rstd = (1.0 / np.sqrt(var.astype(np.float64))).astype(np.float32)[:, None, None]
    y = (d * rstd).astype(np.float32)
    y = y.reshape(t, 32, nv, 8).transpose(0, 2, 1, 3).reshape(t, nv * 256)[:, :h]
    y = (y * np.asarray(gamma, np.float32)).astype(np.float32).reshape(t, h // ESMC_HEAD, 2, ESMC_HEAD // 2)
    c = np.asarray(cos, np.float32)[pos][:, None, :]
    sn = np.asarray(sin, np.float32)[pos][:, None, :]
    y1, y2 = y[:, :, 0], y[:, :, 1]
    return np.stack([fma32(y1, c, -(y2 * sn)), fma32(y2, c, y1 * sn)], 2).reshape(t, h)


def qk_layernorm_rope_bound(x, gamma, cos, sin, pos, eps: float):
    """(reference, bound) of ESM C's q / k step on one side, rows x [T, H] of 16-bit values: the float64 LayerNorm
    without bias, gain, and the rotation with the fp32 table values handed to the kernel.  Any fp32 evaluation of the
    kernel's steps is within bound of the reference before its one 16-bit rounding, u = 2^-24:
      the mean      |dmu| <= (H + 2) u mean|x|   (a sum of H terms, the product with fl(1/H))
      the scale     relative (H + 16) u / 2 + (dmu / sigma)^2   (var: a sum of H positive squares, fl(1/H) and the
                    product with it, + eps: (H + 2) u, halved by the square root; rsqrtf's 2 ulps: 4u; x - mean and
                    the two products of y: 3u; the mean's error adds (dmu / sigma)^2 to var)
      so            |dy| <= |g| rstd (dmu + |x - mu| scale)
      the rotation  |c| |dy1| + |s| |dy2| plus one rounding per product and one per sum: 2u (|y1 c| + |y2 s|)."""
    x = np.asarray(x, np.float64)
    t, h = x.shape
    u = 2.0 ** -24
    mu = x.mean(-1, keepdims=True)
    d = x - mu
    var = (d * d).mean(-1, keepdims=True) + np.float32(eps)
    r = 1.0 / np.sqrt(var)
    dmu = (h + 2) * u * np.abs(x).mean(-1, keepdims=True)
    scale = (h + 16) * u / 2 + dmu * dmu / var
    g = np.asarray(gamma, np.float64)
    y = (d * r * g).reshape(t, h // ESMC_HEAD, 2, ESMC_HEAD // 2)
    dy = (np.abs(g) * r * (dmu + np.abs(d) * scale)).reshape(y.shape)
    c = np.asarray(cos, np.float32)[pos][:, None, :].astype(np.float64)
    s = np.asarray(sin, np.float32)[pos][:, None, :].astype(np.float64)
    y1, y2, d1, d2 = y[:, :, 0], y[:, :, 1], dy[:, :, 0], dy[:, :, 1]
    ref = np.stack([y1 * c - y2 * s, y2 * c + y1 * s], 2).reshape(t, h)
    b1 = np.abs(c) * d1 + np.abs(s) * d2 + 2 * u * (np.abs(y1 * c) + np.abs(y2 * s))
    b2 = np.abs(c) * d2 + np.abs(s) * d1 + 2 * u * (np.abs(y2 * c) + np.abs(y1 * s))
    return ref, np.stack([b1, b2], 2).reshape(t, h) * (1 + 2.0 ** -10)


def interval_check(got, ref, bound, dtype) -> str | None:
    """got = round16(v) for some v within bound of ref: got in [round16(ref - bound), round16(ref + bound)] (rounding
    is monotonic).  None, or a description of the first element outside."""
    got = np.asarray(got, np.float64)
    lo, hi = round16(ref - bound, dtype), round16(ref + bound, dtype)
    bad = ~((got >= lo) & (got <= hi))
    if not bad.any():
        return None
    i = tuple(int(k) for k in np.argwhere(bad)[0])
    return (f'{bad.sum()} of {bad.size} outside; first at {i}: got {got[i]!r}, reference {ref[i]!r} '
            f'+- {bound[i]:.3g}')


# ------------------------------------------------------------------------------------------- row-path encoders
# Every weight matrix zero: by the GEMM's bias provenance every linear layer outputs exactly round16(bias), and
# attention is multiplied by a zero matrix.  What remains of each family's forward pass is its row kernels:
#   BERT        LN_emb((word + type) + pos) -> per layer LN_a(round16(bo) + h), LN_o(round16(b2) + h) (post-LN)
#   ESM-2       xres = word * mask, += round16(bo_l), += round16(b2_l) in that order; final LN(xres)
#   ModernBERT  xres = LN_emb(tok) (no biases anywhere); final LN(xres)
#   Mistral / Qwen3   xres = embed; final RMSNorm(xres)
#   ESM C       xres = embed; final LN(xres) without bias (the pre-norm LayerNorms carry biases, but feed zero
#               matrices only, and no Linear layer has a bias).  Its q / k rows are exactly 0, and the
#               fused q / k LayerNorm maps them to (0 - 0) * rsqrt(eps) * gain = 0 (NaN without eps)
# The inner pre-norm LayerNorms of ESM-2, ModernBERT, ESM C and the decoders feed zero matrices only.
VOCAB = 48
LAYERS = 2
ESM_BIASES = (2.0 ** 15, 2.0 ** 14, 2.0 ** 14, -2.0 ** 15)   # bo0, b20, bo1, b21: xres reaches 2^16 +- 32


def _zero_matrices(sd: dict) -> dict:
    return {k: (torch.zeros_like(v) if v.dim() == 2 and 'embed' not in k else v) for k, v in sd.items()}


def _t(x) -> torch.Tensor:
    return torch.from_numpy(np.asarray(x, np.float64)).float()


def row_path_model(fam: str, h: int, live: str = 'word', max_pos: int = 1100):
    """(HF config, state dict, reference) of a 2-layer ``fam`` model of width h whose output is a composition of row
    kernels.  ``reference(ids, mask, types)`` -> float64 [B, S, H] final hidden state, exact fp32 values.
    BERT: ``live`` names the one embedding table ('word', 'pos', 'type') that holds Walsh rows; the others are 0."""
    from distllm_b200.embed.encoders import weights as W

    if fam == 'esmc':
        sd = _zero_matrices(W.random_esmc_state_dict(h, LAYERS, 256, seed=h, vocab=VOCAB))
        emb = esmc_walsh_rows(VOCAB, h)
        emb[VOCAB - 1] = 0.0          # the final LayerNorm of a zero row: 0, and NaN without eps
        sd['embed.weight'] = _t(emb)
        g_f = esmc_gain(h, 3, -1.0)
        sd['transformer.norm.weight'] = _t(g_f)
        cfg = W.esmc_config(sd)

        def reference(ids, mask, types, dtype):
            return layernorm(emb[ids.numpy()], g_f, 0.0, W.ESMC_EPS)
        return cfg, sd, reference

    n, _ = split_width(h)
    beta_f = 2.0 ** 3 * pattern(h, 1 + (n // 2 - 2) % (n // 2 - 1))     # the final norm's bias: a pattern
    if fam == 'bert':
        from transformers import BertConfig
        cfg = BertConfig(vocab_size=VOCAB, hidden_size=h, num_hidden_layers=LAYERS, num_attention_heads=h // 64,
                         intermediate_size=256, max_position_embeddings=max_pos, type_vocab_size=2,
                         layer_norm_eps=1e-12)
        sd = _zero_matrices(W.random_bert_state_dict(cfg, seed=h))
        tables = {'word': VOCAB, 'pos': max_pos, 'type': 2}
        keys = {'word': 'word_embeddings', 'pos': 'position_embeddings', 'type': 'token_type_embeddings'}
        for name, rows in tables.items():
            sd[f'embeddings.{keys[name]}.weight'] = _t(walsh_rows(rows, h) if name == live else np.zeros((rows, h)))
        gains = [walsh_gain(h, 5, (-1.0) ** i) for i in range(1 + 2 * LAYERS)]
        betas = [np.full(h, 2.0 ** (7 + i)) for i in range(2 * LAYERS - 1)] + [beta_f]   # only the last: a pattern
        sd['embeddings.LayerNorm.weight'], sd['embeddings.LayerNorm.bias'] = _t(gains[0]), _t(np.full(h, 64.0))
        for l in range(LAYERS):
            p = f'encoder.layer.{l}.'
            for name in ('attention.self.query', 'attention.self.key', 'attention.self.value', 'intermediate.dense'):
                sd[p + name + '.bias'].zero_()
            sd[p + 'attention.output.dense.bias'] = _t(np.full(h, 2.0 ** 10))
            sd[p + 'output.dense.bias'] = _t(np.full(h, -2.0 ** 9))
            for i, name in enumerate(('attention.output.LayerNorm', 'output.LayerNorm')):
                sd[p + name + '.weight'] = _t(gains[1 + 2 * l + i])
                sd[p + name + '.bias'] = _t(betas[2 * l + i])

        def reference(ids, mask, types, dtype):
            word = sd['embeddings.word_embeddings.weight'].double().numpy()
            pos = sd['embeddings.position_embeddings.weight'].double().numpy()
            typ = sd['embeddings.token_type_embeddings.weight'].double().numpy()
            s = ids.shape[1]
            tt = types.numpy() if types is not None else np.zeros_like(ids.numpy())
            x = (word[ids.numpy()] + typ[tt]) + pos[np.arange(s)][None]
            hdn = round16(layernorm(x, gains[0], 64.0, cfg.layer_norm_eps), dtype)
            for l in range(LAYERS):
                p = f'encoder.layer.{l}.'
                for name, b in (('attention.output', 'attention.output.dense.bias'), ('output', 'output.dense.bias')):
                    tmp = round16(sd[p + b].double().numpy(), dtype)
                    y = layernorm(tmp + hdn, sd[p + name + '.LayerNorm.weight'].double().numpy(),
                                  sd[p + name + '.LayerNorm.bias'].double().numpy(), cfg.layer_norm_eps)
                    hdn = y if (l == LAYERS - 1 and name == 'output') else round16(y, dtype)
            return hdn
        return cfg, sd, reference

    if fam == 'esm':
        from transformers import EsmConfig
        cfg = EsmConfig(vocab_size=VOCAB, hidden_size=h, num_hidden_layers=LAYERS, num_attention_heads=h // 64,
                        intermediate_size=256, max_position_embeddings=max_pos, position_embedding_type='rotary',
                        token_dropout=False, mask_token_id=VOCAB - 1, pad_token_id=1, layer_norm_eps=1e-5,
                        emb_layer_norm_before=False)
        sd = _zero_matrices(W.random_esm_state_dict(cfg, seed=h))
        sd['embeddings.word_embeddings.weight'] = _t(walsh_rows(VOCAB, h))
        biases = iter(ESM_BIASES)
        for l in range(LAYERS):
            p = f'encoder.layer.{l}.'
            for name in ('attention.self.query', 'attention.self.key', 'attention.self.value', 'intermediate.dense'):
                sd[p + name + '.bias'].zero_()
            sd[p + 'attention.output.dense.bias'] = _t(np.full(h, next(biases)))
            sd[p + 'output.dense.bias'] = _t(np.full(h, next(biases)))
        sd['encoder.emb_layer_norm_after.weight'] = _t(walsh_gain(h, 4, -1.0))
        sd['encoder.emb_layer_norm_after.bias'] = _t(beta_f)

        def reference(ids, mask, types, dtype):
            word = sd['embeddings.word_embeddings.weight'].double().numpy()
            xres = _r32(word[ids.numpy()] * mask.numpy()[..., None])
            for b in ESM_BIASES:
                xres = _r32(xres + round16(np.float64(b), dtype))
            return layernorm(xres, sd['encoder.emb_layer_norm_after.weight'].double().numpy(),
                             beta_f, cfg.layer_norm_eps)
        return cfg, sd, reference

    if fam == 'modernbert':
        from transformers import ModernBertConfig
        cfg = ModernBertConfig(vocab_size=VOCAB, hidden_size=h, num_hidden_layers=LAYERS,
                               num_attention_heads=h // 64, intermediate_size=256, max_position_embeddings=max_pos,
                               local_attention=128, norm_eps=1e-5, pad_token_id=0, bos_token_id=1, eos_token_id=2,
                               cls_token_id=1, sep_token_id=2)
        sd = _zero_matrices(W.random_modernbert_state_dict(cfg, seed=h))
        sd['embeddings.tok_embeddings.weight'] = _t(walsh_rows(VOCAB, h))
        g_e, g_f = walsh_gain(h, 5), walsh_gain(h, 2, -1.0)
        sd['embeddings.norm.weight'], sd['embeddings.norm.bias'] = _t(g_e), _t(np.full(h, 2.0 ** 10))
        sd['final_norm.weight'], sd['final_norm.bias'] = _t(g_f), _t(beta_f)

        def reference(ids, mask, types, dtype):
            tok = sd['embeddings.tok_embeddings.weight'].double().numpy()
            xres = layernorm(tok[ids.numpy()], g_e, 2.0 ** 10, cfg.norm_eps)
            return layernorm(xres, g_f, beta_f, cfg.norm_eps)
        return cfg, sd, reference

    if fam in ('mistral', 'qwen3'):
        heads = max(2, h // 128)
        common = dict(vocab_size=VOCAB, hidden_size=h, num_hidden_layers=LAYERS, num_attention_heads=heads,
                      num_key_value_heads=max(1, heads // 4), head_dim=128, intermediate_size=256,
                      max_position_embeddings=max_pos)
        if fam == 'mistral':
            from transformers import MistralConfig
            cfg = MistralConfig(rms_norm_eps=1e-5, sliding_window=None, **common)
            sd = _zero_matrices(W.random_mistral_state_dict(cfg, seed=h))
        else:
            from transformers import Qwen3Config
            cfg = Qwen3Config(rms_norm_eps=1e-6, rope_parameters={'rope_type': 'default', 'rope_theta': 1e6},
                              tie_word_embeddings=False, **common)
            sd = _zero_matrices(W.random_qwen3_state_dict(cfg, seed=h))
        emb = walsh_rows(VOCAB, h)
        emb[VOCAB - 1] = 0.0          # RMSNorm of a zero row: 0, and NaN without eps
        sd['embed_tokens.weight'] = _t(emb)
        g_f = walsh_gain(h, 3, -1.0)
        sd['norm.weight'] = _t(g_f)

        def reference(ids, mask, types, dtype):
            emb = sd['embed_tokens.weight'].double().numpy()
            return rmsnorm(emb[ids.numpy()], g_f, cfg.rms_norm_eps)
        return cfg, sd, reference
    raise ValueError(fam)


# Widths each family is built for (b2e_check_model, tests/test_widths_cpu.py): the 128-column half pass widths
# 384 / 640 only in the families with biases on their row kernels' inputs.
FAMILY_WIDTHS = {'bert': WIDTHS, 'esm': WIDTHS,
                 'modernbert': tuple(h for h in WIDTHS if h % 256 == 0),
                 'mistral': tuple(h for h in WIDTHS if h % 256 == 0),
                 'qwen3': tuple(h for h in WIDTHS if h % 256 == 0),
                 'esmc': tuple(ODD)}
