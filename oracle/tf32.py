"""The TF32 arithmetic of the tensor-core retrieval scans (distllm_b200/csrc/topk_tc.cuh) restated on the host, and
inputs on which the TF32 scan ranks rows differently from the exact fp32 decision.  TEST INFRASTRUCTURE ONLY.

The tensor-core search is exact only if its margin holds: a row the TF32 scan scores below the threshold
`edge - 2 eps - bin` must not be able to reach the k-th best exact score.  This module states every number that
argument uses, the way the kernels compute it, so that a test can hold the device's intermediate state (the hook
b2e_debug_topk_tc_state) to the formulas:

  conversion   a wgmma reads fp32 operands as TF32 (10 explicit mantissa bits).  Two models: truncation (the low 13
               bits dropped, relative error < 2^-10 per operand) and round-to-nearest-even (< 2^-11).  A product of
               two converted operands has 22 significant bits, so it is exact in fp32.
  accumulation the products are summed in fp32 in an order the hardware does not document.  In any order, with a
               rounding or a truncating adder, the sum of H terms is off by at most (H - 1) 2^-23 sum |p_i| to first
               order: SCAN_ACC_ULPS_PER_TERM below.  That is the allowance `accumulation_allowance` grants a device
               score against the float64 sum of the converted products.
  margin       eps = 1.5 2^-9 r (inner product), r = |q| M; L2 adds the terms of `eps_l2`.
  rescore      the exact decision's fp32 dot product: per lane a chain of H / 32 fmaf, then a xor tree of 5 adds,
               so |error| <= (H / 32 + 5) 2^-24 sum |q_i x_i| (`rescore_error`).

`adversarial` builds corpora whose planted rows the TF32 scan, under a given conversion model, ranks in the wrong
order, so that only the fp32 rescore of a large enough candidate set returns the right answer.
"""

from __future__ import annotations

from fractions import Fraction
from typing import NamedTuple

import numpy as np
import torch

BINS = 2048            # TC_BINS
MAX_CAND = 4096        # TC_MAX_CAND
EPS_SCALE = np.float32(1.5 / 512.0)
SCAN_ACC_ULPS_PER_TERM = 2.0 ** -23
TRUNC, RNE = 'trunc', 'rne'
MODELS = (TRUNC, RNE)
F32 = np.float32


# ------------------------------------------------------------------------------------------- conversion
def _tf32_bits(u, model: str):
    """fp32 bit patterns (uint32 numpy / int32 torch) -> their TF32 conversion's bit patterns"""
    if model == TRUNC:
        return u & (0xFFFFE000 if isinstance(u, np.ndarray) else -0x2000)
    if model != RNE:
        raise ValueError(f'unknown TF32 model {model!r}')
    finite = ((u >> 23) & 0xFF) != 0xFF
    up = (u + 0xFFF + ((u >> 13) & 1)) & (0xFFFFE000 if isinstance(u, np.ndarray) else -0x2000)
    return np.where(finite, up, u) if isinstance(u, np.ndarray) else torch.where(finite, up, u)


def tf32(x, model: str):
    """The TF32 value of every element of a float32 numpy array or torch tensor, as float32 of the same kind:
    truncation (low 13 mantissa bits dropped) or round-to-nearest-even on those bits (infinities and NaNs kept)."""
    if isinstance(x, np.ndarray):
        if x.dtype != np.float32:
            raise TypeError('tf32 expects float32')
        return _tf32_bits(x.view(np.uint32), model).astype(np.uint32).view(np.float32)
    if x.dtype != torch.float32:
        raise TypeError('tf32 expects float32')
    return _tf32_bits(x.contiguous().view(torch.int32), model).view(torch.float32)


def tf32_scores(queries: torch.Tensor, corpus: torch.Tensor, model: str, chunk: int = 1 << 14):
    """(S, A): float64 [Q, N] sums of the converted products, and of their magnitudes, computed in row chunks on the
    corpus' device (the device scan's value up to its accumulation error)."""
    qt = tf32(queries, model).to(corpus.device, torch.float64)
    s = torch.empty((queries.shape[0], corpus.shape[0]), dtype=torch.float64, device=corpus.device)
    a = torch.empty_like(s)
    for lo in range(0, corpus.shape[0], chunk):
        x = tf32(corpus[lo:lo + chunk], model).to(torch.float64)
        s[:, lo:lo + chunk] = qt @ x.T
        a[:, lo:lo + chunk] = qt.abs() @ x.abs().T
    return s, a


def abs_score_matrix(queries: torch.Tensor, corpus: torch.Tensor, chunk: int = 1 << 14) -> torch.Tensor:
    """[Q, N] float64 sum |q_i x_i|, in row chunks on the corpus' device"""
    q = queries.to(corpus.device, torch.float64).abs()
    out = torch.empty((queries.shape[0], corpus.shape[0]), dtype=torch.float64, device=corpus.device)
    for lo in range(0, corpus.shape[0], chunk):
        out[:, lo:lo + chunk] = q @ corpus[lo:lo + chunk].to(torch.float64).abs().T
    return out


def accumulation_allowance(h: int, abs_products):
    """What fp32 accumulation of h exact products may add, in any order, rounding or truncating"""
    return h * SCAN_ACC_ULPS_PER_TERM * abs_products


def rescore_error(h: int, abs_dot):
    """Bound of the fp32 rescore's error: H / 32 fmaf per lane, then 5 adds across the warp.  For L2 pass D
    (a sum of non-negative terms) and add two roundings per term for the differences: rescore_error(h + 64, D)."""
    return (h / 32 + 5) * 2.0 ** -24 * abs_dot


# ------------------------------------------------------------------------------------------ the margin
def eps_ip(r) -> np.float32:
    """tc_prepare_queries_kernel: eps = r * 1.5 / 512 in fp32 (1.5 / 512 is exact)"""
    return F32(r) * EPS_SCALE


def eps_l2(r, qnorm, max_norm, h: int) -> np.float32:
    """tc_prepare_queries_kernel<true>: d = eps_S + H 2^-24 M^2 + 2^-23 (r + M^2) bounds |v - v_exact|, and
    eps = (d + H 2^-24 qm^2) 1.0001 with qm = |q| 1.0001 + M (the half of e_D the threshold's 2 eps carries).
    Evaluated in fp32 without contraction; qnorm is the fp32 |q| (sqrt of the device's sum of squares)."""
    r, m = F32(r), F32(max_norm)
    m2 = m * m
    qm = F32(qnorm) * F32(1.0001) + m
    d = r * EPS_SCALE + F32(h) * F32(2.0 ** -24) * m2 + F32(2.0 ** -23) * (r + m2)
    return (d + F32(h) * F32(2.0 ** -24) * qm * qm) * F32(1.0001)


def shift_of(max_norm) -> np.float32:
    """the L2 histogram's extension below -r: M^2 / 2"""
    return F32(0.5) * F32(max_norm) * F32(max_norm)


def bin_width(r, shift=0.0) -> np.float32:
    """score_threshold_kernel: 2 r / BINS (inner product), (2 r + shift) / BINS (L2)"""
    return (F32(2.0) * F32(r) + F32(shift)) / F32(BINS)


def thresholds(found: int, r, eps, shift=0.0) -> tuple[np.float32, np.float32]:
    """thr = edge - 2 eps - bin with edge = lo + found * bin, lo = -r - shift: the value without contraction and
    with found * bin + lo fused into one FMA (nvcc contracts by default; the two may differ in the last bit)."""
    r, eps, shift = F32(r), F32(eps), F32(shift)
    w = bin_width(r, shift)
    lo = -r - shift
    plain = lo + F32(found) * w
    fused = F32(np.float64(found) * np.float64(w) + np.float64(lo))
    return tuple((e - F32(2.0) * eps) - w for e in (plain, fused))


# -------------------------------------------------------------------------------- histogram and walk
def l2_values(scores: np.ndarray, norm2: np.ndarray) -> np.ndarray:
    """v = fl(S - fl(n / 2)) per row (l2_value): scores [N] or [N, Q], norm2 [N], fp32"""
    n2 = norm2.astype(F32) * F32(0.5)
    return (scores.astype(F32) - (n2[:, None] if scores.ndim == 2 else n2)).astype(F32)


def bins_ip(s: np.ndarray, r) -> np.ndarray:
    """tc_bin: u = (s + r) * 1024 / r in fp32, truncated, NaN / negative -> 0, clamped to BINS - 1"""
    r = F32(r)
    with np.errstate(invalid='ignore', over='ignore'):
        u = ((s.astype(F32) + r) * F32(BINS * 0.5)) / r
    b = np.where(u > 0, np.minimum(np.floor(np.where(u > 0, u, 0)), BINS - 1), 0)
    return b.astype(np.int64)


def bins_l2(v: np.ndarray, r, shift) -> np.ndarray:
    """tc_bin_l2 over [lo, r]: u = (v - lo) * scale, lo = -r - shift, scale = BINS / (2 r + shift)"""
    r, shift = F32(r), F32(shift)
    lo = -r - shift
    scale = F32(BINS) / (F32(2.0) * r + shift)
    with np.errstate(invalid='ignore', over='ignore'):
        u = (v.astype(F32) - lo) * scale
    b = np.where(u > 0, np.minimum(np.floor(np.where(u > 0, u, 0)), BINS - 1), 0)
    return b.astype(np.int64)


def histogram(bins: np.ndarray) -> np.ndarray:
    return np.bincount(bins, minlength=BINS).astype(np.int64)


def found_bin(hist: np.ndarray, need: int) -> int:
    """score_threshold_kernel's walk: the highest bin b with sum(hist[b:]) >= need (0 if none)"""
    from_top = np.cumsum(hist[::-1])
    hit = np.nonzero(from_top >= need)[0]
    return int(BINS - 1 - hit[0]) if hit.size else 0


# ------------------------------------------------------------------------------------ adversarial inputs
N_DELTA, N_EXTRA, N_PAD = 8, 16, 8
ROUNDED_LOW_BITS = {TRUNC: 0x1FFF, RNE: 0x0FFF}   # the largest conversion error each model makes near 1.0


def rounded_one(model: str) -> float:
    """1.0 with the low 13 bits ROUNDED_LOW_BITS[model]: converts to exactly 1.0 under `model`, with error
    ~2^-10 (truncation) or just under 2^-11 (round-to-nearest, below the midpoint)"""
    return 1.0 + ROUNDED_LOW_BITS[model] * 2.0 ** -23


class Layout(NamedTuple):
    nb: int
    a: slice        # the exact half: query +-1, outrankers +-1
    d: slice        # N_DELTA columns of the exact half that carry each outranker's fine offset
    b: slice        # the rounded half: query and winner +-rounded_one
    e: slice        # per-query columns no planted row uses (they move r, and with it the bin grid)
    p: slice        # columns no query uses: pad the planted rows to one norm


def layout(h: int) -> Layout:
    nb = (h - N_DELTA - N_EXTRA - N_PAD) // 2
    if nb < 16 or 2 * nb + N_DELTA + N_EXTRA + N_PAD != h:
        raise ValueError(f'adversarial inputs need an even H >= 64, got {h}')
    o = [0, nb, nb + N_DELTA, 2 * nb + N_DELTA, 2 * nb + N_DELTA + N_EXTRA, h]
    return Layout(nb, *(slice(o[i], o[i + 1]) for i in range(5)))


class Planted(NamedTuple):
    queries: torch.Tensor      # [Q, H] f32
    corpus: torch.Tensor       # [N, H] f32
    winners: torch.Tensor      # [Q] row ids: the exact best row of each query
    outrankers: torch.Tensor   # [Q, k] row ids, in exact order: the exact places 2 .. k + 1, the TF32 places 1 .. k


def offsets(h: int, model: str) -> int:
    """m0: the first outranker scores nb + m0 2^-10, below the winner's exact nb v^2 by at least twice the fp32
    rescore's error bound (so that the rescored order is the exact one), and at most that plus 2^-10"""
    nb = layout(h).nb
    v = Fraction(ROUNDED_LOW_BITS[model], 1 << 23) + 1
    s_w = nb * v * v
    guard = Fraction(2 * rescore_error(h + 64, 4 * nb)).limit_denominator(1 << 40)
    return int((s_w - nb - guard) * 1024) - 1


def adversarial(n: int, h: int, q: int, k: int, model: str, seed: int, device=None,
                far_background: bool = False) -> Planted:
    """A corpus of n rows and q queries for both metrics, inverted by the TF32 scan under `model`.

    For every query: the winner lives on the rounded half B, where query and winner entries are +-rounded_one:
    exact score nb v^2, TF32 score nb (each operand converts to 1.0).  k outrankers live on the exact half: +-1
    where the query is +-1, plus offsets m 2^-10 (m <= 1023 per column, TF32-exact) on the D columns, so every one
    of their products and partial sums is exact in TF32 and fp32.  Their scores nb + (m0 - j) 2^-10, j < k, lie
    between the winner's TF32 score and its exact one: the TF32 scan puts all k above the winner, the exact order
    puts the winner first.  A pad column gives every planted row the same squared norm (to fp32 rounding), so the
    L2 order (v = q.x - |x|^2 / 2) is the inner-product order.  The query's E columns take a random share of |q|^2
    in [0, nb), which moves r and the bin grid from query to query.  Background rows: random directions of norm
    sqrt(nb) / 2, scoring far below nb; with `far_background` (L2 only) norms of 300 to 1000 |q|, so that
    max_norm ~ 10^3 |q| and the L2 histogram's shift M^2 / 2 dominates its range.
    """
    lay = layout(h)
    nb = lay.nb
    m0 = offsets(h, model)
    if m0 - k + 1 < 4:
        raise ValueError(f'H={h} leaves room for {m0 - 3} outrankers under {model}, asked for {k}')
    device = torch.device(device or 'cpu')
    g = torch.Generator().manual_seed(seed)
    gd = torch.Generator(device=device).manual_seed(seed + 1)
    v = rounded_one(model)
    queries = torch.zeros((q, h), dtype=torch.float64)
    sign = torch.randint(0, 2, (q, lay.e.start), generator=g).to(torch.float64) * 2 - 1
    queries[:, :lay.e.start] = sign
    queries[:, lay.b] *= v
    share = torch.rand(q, generator=g, dtype=torch.float64) * nb
    extra = torch.randn((q, N_EXTRA), generator=g, dtype=torch.float64)
    queries[:, lay.e] = extra * (share / (extra * extra).sum(dim=1)).sqrt()[:, None]

    rows = torch.zeros((q, k + 1, h), dtype=torch.float64)
    rows[:, 0, lay.b] = sign[:, lay.b] * v
    rows[:, 1:, lay.a] = sign[:, None, lay.a]
    m = m0 - torch.arange(k, dtype=torch.int64)
    piece = (m[:, None] + torch.arange(N_DELTA)[None, :]) // N_DELTA      # m spread over the D columns, each <= 1023
    rows[:, 1:, lay.d] = sign[:, None, lay.d] * (piece.to(torch.float64) * 2.0 ** -10)[None]
    norm2 = (rows * rows).sum(dim=2)
    rows[:, :, lay.p.start] = (norm2.max() - norm2).sqrt()

    ids = torch.randperm(n, generator=g)[:q * (k + 1)].view(q, k + 1)
    if far_background:
        qn = float(queries.norm(dim=1).max())
        scale = (300.0 + 700.0 * torch.rand((n, 1), generator=gd, device=device)) * qn
    else:
        scale = torch.full((n, 1), 0.5 * nb ** 0.5, device=device)
    corpus = torch.randn((n, h), generator=gd, device=device)
    corpus *= scale / corpus.norm(dim=1, keepdim=True)
    corpus[ids.reshape(-1).to(device)] = rows.reshape(-1, h).to(device, torch.float32)
    return Planted(queries.to(device, torch.float32), corpus, ids[:, 0], ids[:, 1:])
