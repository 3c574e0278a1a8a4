"""GEMM inputs whose output is known bit for bit, references rounded as the kernel rounds, and the error bound of
the activation epilogues (csrc/gemm.cuh).  TEST INFRASTRUCTURE ONLY.

* :func:`ternary_pair` -- sparse matrices over {-1, 0, 1}: every A row has at most 256 nonzeros, so every partial
  sum is an integer of magnitude <= 256 < 2^24 and every output is an integer |out| <= 256.  Such sums are exact in
  fp32 in any order (tensor cores, float64), and integers up to 256 are exact in bfloat16 (2048 in half): a wrong,
  missing or repeated operand changes the output bits.
* :func:`one_hot_rows` -- W rows e_pi(n) give out[m, n] = A[m, pi(n)]; A rows e_sigma(m) give out[m, n] =
  W[n, sigma(m)].  Exact for any finite 16-bit values: every other product is 0 * x.
* :func:`value_table` -- every finite, nonzero, normal half value, or every finite bfloat16 value.
* :func:`epilogue` -- the kernel's epilogue on an exact accumulator: round16(fp32(fp32(acc + bias) + resid)),
  round to nearest even, half saturating to +-65504 (``cvt.rn.satfinite``).
* :func:`gated` -- gate / up pairing of ``weights.interleave_gate_up``'s row order.
* :func:`activation_error_bound` -- the stored output's distance from the float64 activation, derived from the
  epilogue's fp32 arithmetic and the PTX ISA's stated errors of the MUFU approximations.
* :func:`gelu_kernel_model` / :func:`silu_kernel_model` -- that arithmetic in numpy, with the approximations
  perturbed by their documented errors (tests/test_gemm_oracle_cpu.py shows the bound holds for them).
"""

from __future__ import annotations

import math

import numpy as np
import torch

HALF_MAX = 65504.0
BLOCK_K = 64                # one k-block of the kernel
GATE_UP_BLOCK = 64          # weights.interleave_gate_up
TERNARY_NNZ = 256           # nonzeros per A row of ternary_pair: |out| <= 256

# GELU epilogue (gelu_erf_fast): erf(x / sqrt2) ~= tanh(xc * Q(xc^2)), xc = clamp(x, +-CLAMP)
GELU_CLAMP = float(np.float32(5.65685))
GELU_Q = tuple(float(np.float32(c)) for c in (-1.35688221e-05, -1.95764464e-04, 3.65498251e-02, 7.97818838e-01))
# max |tanh(x Q(x^2)) - erf(x / sqrt2)| over |x| <= GELU_CLAMP, plus 1 - erf(4) for the clamped tail (the code
# comment says 1.4e-5; tests/test_gemm_oracle_cpu.py measures it)
GELU_FIT_ERR = 1.5e-5
# PTX ISA, "Floating Point Instructions": tanh.approx.f32 "maximum relative error of 2^-10.987" (2^-11 in older
# editions); ex2.approx.ftz.f32 "maximum relative error ... 2^-22" over the range the epilogue uses; rcp.approx.ftz.f32
# "maximum ulp error is 1", i.e. relative 2^-23.  All three flush subnormal results (ftz) or return them (tanh).
TANH_REL_ERR = 2.0 ** -10.987
EX2_REL_ERR = 2.0 ** -22
RCP_REL_ERR = 2.0 ** -23
LOG2E_F32 = float(np.float32(1.4426950408889634))
FLT_MIN = 2.0 ** -126


# ------------------------------------------------------------------------------------------------ storage rounding
def to_storage(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """fp32 (or exact float64 that fp32 holds) -> the 16-bit storage type, round to nearest even; half saturates
    to +-65504 like ``cvt.rn.satfinite.f16.f32`` (NaN stays NaN)."""
    x = x.to(torch.float32)
    if dtype == torch.float16:
        x = torch.where(torch.isnan(x), x, x.clamp(-HALF_MAX, HALF_MAX))
    return x.to(dtype)


def epilogue(acc: torch.Tensor, bias: torch.Tensor | None, resid: torch.Tensor | None, dtype: torch.dtype
             ) -> torch.Tensor:
    """EPI_BIAS / EPI_BIAS_RESID on an accumulator that fp32 holds exactly: round16(fp32(fp32(acc + bias) + resid)).
    One rounding to 16 bits; the fp32 adds are IEEE round-to-nearest on any device."""
    v = acc.to(torch.float32)
    if bias is not None:
        v = v + bias.to(v.device, torch.float32)[None, :]
    if resid is not None:
        v = v + resid.to(v.device).to(torch.float32)
    return to_storage(v, dtype)


def exact_product(a: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """a @ w.T in float64 (exact for the inputs of this module), in row chunks."""
    out = torch.empty((a.shape[0], w.shape[0]), dtype=torch.float64, device=a.device)
    w64 = w.to(torch.float64)
    step = max(1, (1 << 26) // max(1, w.shape[0]))
    for lo in range(0, a.shape[0], step):
        out[lo:lo + step] = a[lo:lo + step].to(torch.float64) @ w64.T
    return out


# ------------------------------------------------------------------------------------------------ exact inputs
def ternary_pair(m: int, n: int, k: int, gen: torch.Generator, dtype: torch.dtype, device=None
                 ) -> tuple[torch.Tensor, torch.Tensor]:
    """A [m, k] with min(k, 256) entries +-1 per row at random columns (the rest 0), W [n, k] uniform over
    {-1, 0, 1}.  |every partial sum| <= 256, so the product is exact in any order and in both storage types."""
    device = device or gen.device
    nnz = min(k, TERNARY_NNZ)
    cols = torch.rand((m, k), generator=gen, device=device).argsort(dim=1)[:, :nnz]
    a = torch.zeros((m, k), dtype=torch.float32, device=device)
    sign = torch.randint(0, 2, (m, nnz), generator=gen, device=device).to(torch.float32) * 2 - 1
    a.scatter_(1, cols, sign)
    w = torch.randint(-1, 2, (n, k), generator=gen, device=device).to(torch.float32)
    return a.to(dtype), w.to(dtype)


def covering_index(count: int, k: int) -> torch.Tensor:
    """[count] column indices in [0, k): every column (so every k-block, its first and last column and each 8-column
    16-byte swizzle unit) once count >= k, in an order that puts neighbouring outputs in different k-blocks and
    scatters them over the swizzle units: output i reads k-block i % (k/64), column 9 j mod 64 of it (j = i // (k/64),
    a permutation of the 64 columns)."""
    kb = k // BLOCK_K
    i = torch.arange(count, dtype=torch.int64) % k
    return BLOCK_K * (i % kb) + (9 * (i // kb)) % BLOCK_K


def one_hot_rows(count: int, k: int, dtype: torch.dtype, device=None) -> tuple[torch.Tensor, torch.Tensor]:
    """(rows [count, k] with row i = e_idx[i], idx) for idx = covering_index(count, k)."""
    idx = covering_index(count, k)
    rows = torch.zeros((count, k), dtype=dtype)
    rows[torch.arange(count), idx] = 1
    return rows.to(device), idx.to(device)


def value_table(dtype: torch.dtype) -> torch.Tensor:
    """Every finite nonzero normal half value (61 440), or every finite bfloat16 value including the subnormals and
    both zeros (65 280), ascending by bit pattern, as ``dtype``."""
    bits = torch.arange(1 << 16, dtype=torch.int32)
    exp = (bits >> (10 if dtype == torch.float16 else 7)) & (0x1f if dtype == torch.float16 else 0xff)
    top = 0x1f if dtype == torch.float16 else 0xff
    keep = exp != top
    if dtype == torch.float16:
        keep &= exp != 0
    return bits[keep].to(torch.int16).view(dtype)


def random_normals(shape, dtype: torch.dtype, gen: torch.Generator) -> torch.Tensor:
    """Values drawn from :func:`value_table` without zeros and subnormals (any finite normal 16-bit value)."""
    t = value_table(dtype)
    t = t[t.float().abs() >= (2.0 ** -14 if dtype == torch.float16 else FLT_MIN)]
    pick = torch.randint(0, t.numel(), shape, generator=gen, device=gen.device)
    return t.to(gen.device)[pick]


# ------------------------------------------------------------------------------------------------ gated epilogues
def gated(product: torch.Tensor, act) -> torch.Tensor:
    """[M, N] product of A with interleave_gate_up(gate, up) -> act(gate) * up [M, N/2]: columns
    [128t, 128t + 64) are gate and [128t + 64, 128t + 128) up of outputs [64t, 64t + 64)."""
    m, n = product.shape
    blocks = product.reshape(m, n // (2 * GATE_UP_BLOCK), 2, GATE_UP_BLOCK)
    return (act(blocks[:, :, 0]) * blocks[:, :, 1]).reshape(m, n // 2)


def gelu64(x):
    """Exact erf-GELU in float64 (numpy or torch)."""
    if isinstance(x, torch.Tensor):
        x = x.to(torch.float64)
        return 0.5 * x * (1 + torch.special.erf(x / math.sqrt(2)))
    from scipy.special import erf
    x = np.asarray(x, np.float64)
    return 0.5 * x * (1 + erf(x / math.sqrt(2)))


def silu64(x):
    """Exact SiLU in float64 (numpy or torch), without overflow warnings for large |x|."""
    if isinstance(x, torch.Tensor):
        x = x.to(torch.float64)
        return x * torch.sigmoid(x)
    from scipy.special import expit
    x = np.asarray(x, np.float64)
    return x * expit(x)


def half_ulp(v, dtype: torch.dtype):
    """Half a unit in the last place of the storage type at magnitude |v| (numpy float64): the largest error of
    round-to-nearest there, including the subnormal range (bfloat16 shares fp32's, with 7 stored bits)."""
    v = np.abs(np.asarray(v, np.float64))
    mant, emin = (10, -14) if dtype == torch.float16 else (7, -126)
    with np.errstate(divide='ignore'):
        e = np.floor(np.log2(np.maximum(v, 2.0 ** emin)))
    return np.ldexp(1.0, (np.maximum(e, emin) - mant - 1).astype(np.int64))


def activation_error_bound(x, dtype: torch.dtype, kind: str = 'gelu', up=None):
    """Largest |stored - ref| of an activation epilogue at pre-activation x (numpy float64 array), where
    ref = act(x) (EPI_BIAS_GELU) or act(x) * up (EPI_GEGLU / EPI_SWIGLU with up value ``up``) in float64, and for
    half both stored and ref are clamped to +-65504 (the saturation is exact, and clamping only shrinks distances).

    GELU: 0.5 |x| (GELU_FIT_ERR + TANH_REL_ERR |tanh| + 2^-18).  The fit error includes the clamp's tail; tanh's
    relative error at |tanh| <= 1; 2^-18 covers the fp32 roundings of xc^2, the fma chain and xc q (|xc q| < 8,
    four roundings move tanh by < 2^-19) and of the final fma (2^-24 |x|).
    SiLU: |silu| (RCP_REL_ERR + 3 2^-24 + (EX2_REL_ERR + |x| 2^-23) sigmoid(-x)) + (|x| + 1) 2^-126.  ex2's error
    and the rounding of -x log2e (relative 2^-23 with the fp32 constant's own error, which 2^z turns into an
    absolute |x| 2^-23 relative to e) reach sigmoid damped by e / (1 + e) = sigmoid(-x); rcp, 1 + e and x r round
    once each; the ftz flush of a reciprocal below 2^-126 loses at most |x| 2^-126.
    Gated: |up| times the above, plus the rounding of the fp32 product.  Finally half an ulp of the output."""
    x = np.asarray(x, np.float64)
    ax = np.abs(x)
    if kind == 'gelu':
        val = np.abs(gelu64(x))
        pre = 0.5 * ax * (GELU_FIT_ERR + TANH_REL_ERR + 2.0 ** -18)
    elif kind == 'silu':
        from scipy.special import expit
        val = np.abs(silu64(x))
        pre = val * (RCP_REL_ERR + 3 * 2.0 ** -24 + (EX2_REL_ERR + ax * 2.0 ** -23) * expit(-x)) + (ax + 1) * FLT_MIN
    else:
        raise ValueError(kind)
    pre = pre + FLT_MIN      # fp32 subnormal results of 0.5 x and the fmas round at 2^-149
    if up is not None:
        au = np.abs(np.asarray(up, np.float64))
        val = val * au
        pre = pre * au + val * 2.0 ** -24
    if dtype == torch.float16:
        val = np.minimum(val, HALF_MAX)
    return pre + half_ulp(val + pre, dtype)


# ------------------------------------------------------------------------------------------------ kernel models
def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _fma(a, b, c):
    """fp32 fma: the exact product of two fp32 values is a float64, one rounding of the sum (to float64, then fp32:
    off by one fp32 ulp at worst, far inside the bound's 2^-18)."""
    return _f32(np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64))


def _ftz(x):
    x = np.asarray(x, np.float32)
    return np.where(np.abs(x) < np.float32(FLT_MIN), np.float32(0), x)


def gelu_kernel_model(x, tanh_err: float = 0.0) -> np.ndarray:
    """gelu_erf_fast in fp32, operation by operation, with tanh.approx = tanh * (1 + tanh_err)."""
    x = _f32(x)
    with np.errstate(over='ignore', invalid='ignore'):
        xc = np.minimum(np.maximum(x, np.float32(-GELU_CLAMP)), np.float32(GELU_CLAMP))
        v = xc * xc
        q = _fma(v, GELU_Q[0], GELU_Q[1])
        q = _fma(v, q, GELU_Q[2])
        q = _fma(v, q, GELU_Q[3])
        t = _f32(np.tanh((xc * q).astype(np.float64)) * (1 + tanh_err))
        h = np.float32(0.5) * x
        return _fma(h, t, h)


def silu_kernel_model(x, ex2_err: float = 0.0, rcp_err: float = 0.0) -> np.ndarray:
    """silu in fp32: x * rcp.approx.ftz(1 + ex2.approx.ftz(-log2e * x)), each approximation times (1 + err)."""
    x = _f32(x)
    with np.errstate(over='ignore', invalid='ignore'):
        z = _ftz(np.float32(-LOG2E_F32) * x)
        e = _ftz(_f32(np.exp2(z.astype(np.float64)) * (1 + ex2_err)))
        d = np.float32(1) + e
        r = _ftz(_f32((1.0 / d.astype(np.float64)) * (1 + rcp_err)))
        return x * r


def store(x: np.ndarray, dtype: torch.dtype) -> np.ndarray:
    """fp32 results as the kernel stores them, back in float64."""
    return to_storage(torch.from_numpy(np.ascontiguousarray(_f32(x))), dtype).to(torch.float64).numpy()
