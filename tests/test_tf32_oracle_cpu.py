"""oracle/tf32.py without a device: the two TF32 conversion models on chosen bit patterns, the adversarial
builders' inversion under the model each was built for, and the restated histogram walk and threshold on
hand-made histograms."""

from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import tf32 as ot


def bits(*u):
    return np.array(u, dtype=np.uint32).view(np.float32)


# (input bits, truncated, rounded to nearest even)
PATTERNS = [
    (0x3F800000, 0x3F800000, 0x3F800000),   # 1.0: already TF32
    (0x3F801FFF, 0x3F800000, 0x3F802000),   # low bits all ones: the largest truncation error, RNE rounds up
    (0x3F800FFF, 0x3F800000, 0x3F800000),   # just below the midpoint: down under both
    (0x3F801000, 0x3F800000, 0x3F800000),   # the midpoint, even result bit: down
    (0x3F803000, 0x3F802000, 0x3F804000),   # the midpoint, odd result bit: up to even
    (0xBF801FFF, 0xBF800000, 0xBF802000),   # negative: truncation goes toward zero, RNE away
    (0x3FFFFFFF, 0x3FFFE000, 0x40000000),   # RNE carries into the exponent: 2.0
    (0x7F7FFFFF, 0x7F7FE000, 0x7F800000),   # the largest float rounds to infinity
    (0x00001FFF, 0x00000000, 0x00002000),   # subnormal
    (0x7F800000, 0x7F800000, 0x7F800000),   # infinity stays
]


@pytest.mark.parametrize('kind', ['numpy', 'torch'])
def test_tf32_conversion_models_on_chosen_bit_patterns(kind):
    x = bits(*(p[0] for p in PATTERNS))
    for col, model in ((1, ot.TRUNC), (2, ot.RNE)):
        want = [p[col] for p in PATTERNS]
        if kind == 'numpy':
            got = ot.tf32(x, model).view(np.uint32).tolist()
        else:
            got = ot.tf32(torch.from_numpy(x), model).view(torch.int32).numpy().view(np.uint32).tolist()
        assert got == want, (model, [hex(g) for g in got])
    nan = ot.tf32(bits(0x7FC01FFF), ot.RNE)
    assert np.isnan(nan[0])


def test_tf32_keeps_10_mantissa_bits_and_bounds_the_relative_error():
    x = np.random.default_rng(0).standard_normal(100_000).astype(np.float32)
    for model, bound in ((ot.TRUNC, 2.0 ** -10), (ot.RNE, 2.0 ** -11)):
        t = ot.tf32(x, model)
        assert (t.view(np.uint32) & 0x1FFF == 0).all()
        rel = np.abs(t.astype(np.float64) - x) / np.abs(x)
        assert rel.max() <= bound
        if model == ot.TRUNC:
            assert (np.abs(t) <= np.abs(x)).all()
    assert ot.tf32(bits(0x3F800000 | ot.ROUNDED_LOW_BITS[ot.TRUNC]), ot.TRUNC)[0] == 1.0
    assert ot.tf32(bits(0x3F800000 | ot.ROUNDED_LOW_BITS[ot.RNE]), ot.RNE)[0] == 1.0


# ------------------------------------------------------------------------------------------ the builders
def emulated(planted, model):
    """float64 scores of the TF32-converted operands (exact for every planted row: see oracle/tf32.py)"""
    s, _ = ot.tf32_scores(planted.queries, planted.corpus, model)
    return s


def order_ip(s, k):
    return torch.sort(s, dim=1, descending=True, stable=True).indices[:, :k]


def order_l2(s, norm2, k):
    return torch.sort(s - norm2[None] / 2, dim=1, descending=True, stable=True).indices[:, :k]


@pytest.mark.parametrize('model', ot.MODELS)
@pytest.mark.parametrize('h,k', [(256, 1), (768, 10), (768, 256), (1024, 100)])
def test_builders_invert_the_order_under_their_model(model, h, k):
    q, n = 5, 3001
    p = ot.adversarial(n, h, q, k, model, seed=h + k)
    exact = p.queries.double() @ p.corpus.double().T
    norm2 = (p.corpus.double() ** 2).sum(dim=1)
    want = torch.cat([p.winners[:, None], p.outrankers[:, :k - 1]], dim=1)
    tf = emulated(p, model)
    norm2_f32 = norm2.float().double()   # the stored norms are fp32
    for name, ex, em in (('ip', order_ip(exact, k), order_ip(tf, k)),
                         ('l2', order_l2(exact, norm2, k), order_l2(tf, norm2_f32, k))):
        assert torch.equal(ex, want), name                        # exact: the winner first, then the outrankers
        assert torch.equal(em, p.outrankers), name                 # TF32: the k outrankers, the winner below them
    # the inversion is a real gap on the TF32 side, not a tie
    w = tf.gather(1, p.winners[:, None])[:, 0]
    kth = tf.gather(1, p.outrankers[:, -1:])[:, 0]
    assert bool((kth - w >= 4 * 2.0 ** -10).all())
    # and the exact margin of the winner over the outrankers covers the fp32 rescore
    gap = exact.gather(1, p.winners[:, None])[:, 0] - exact.gather(1, p.outrankers[:, :1])[:, 0]
    assert bool((gap > 2 * ot.rescore_error(h + 64, 4 * ot.layout(h).nb)).all())


def test_trunc_builder_does_not_invert_under_round_to_nearest():
    """The two models give different answers on these inputs: what lets a GPU test tell them apart."""
    p = ot.adversarial(2000, 768, 3, 10, ot.TRUNC, seed=3)
    tf = emulated(p, ot.RNE)
    assert bool((order_ip(tf, 1)[:, 0] == p.winners).all())


@pytest.mark.parametrize('far', [False, True])
def test_background_stays_below_the_planted_rows(far):
    h, q, k, n = 768, 16, 100, 20_000
    p = ot.adversarial(n, h, q, k, ot.TRUNC, seed=11, far_background=far)
    exact = p.queries.double() @ p.corpus.double().T
    norm2 = (p.corpus.double() ** 2).sum(dim=1)
    mine = torch.zeros_like(exact, dtype=torch.bool)
    mine.scatter_(1, torch.cat([p.winners[:, None], p.outrankers], dim=1), True)
    planted = set(torch.cat([p.winners[:, None], p.outrankers], dim=1).flatten().tolist())
    assert len(planted) == q * (k + 1)
    v = exact - norm2[None] / 2
    lowest = v.masked_fill(~mine, float('inf')).min(dim=1).values
    others = v.masked_fill(mine, float('-inf')).max(dim=1).values
    assert bool((others < lowest - 0.05 * ot.layout(h).nb).all())
    if far:
        m = float(norm2.max().sqrt())
        assert 500 < m / float(p.queries.double().norm(dim=1).max()) < 1001
    else:
        s_low = exact.masked_fill(~mine, float('inf')).min(dim=1).values
        s_oth = exact.masked_fill(mine, float('-inf')).max(dim=1).values
        assert bool((s_oth < s_low - 0.5 * ot.layout(h).nb).all())


def test_queries_move_the_bin_grid():
    """The E columns spread r over the queries: the k-th TF32 score sits at different offsets within its bin."""
    p = ot.adversarial(2000, 768, 16, 1, ot.TRUNC, seed=5)
    m = float(p.corpus.double().norm(dim=1).max())
    r = p.queries.double().norm(dim=1) * m
    kth = ot.layout(768).nb + ot.offsets(768, ot.TRUNC) * 2.0 ** -10
    frac = ((kth + r) / (2 * r / ot.BINS)) % 1.0
    assert float(frac.max() - frac.min()) > 0.5


# ----------------------------------------------------------------------------- histogram and threshold
def test_bins_cover_the_range_and_clamp():
    r = np.float32(3.0)
    s = np.array([-3.0, -3.5, 0.0, 2.9999, 3.0, 7.0, np.nan], dtype=np.float32)
    assert ot.bins_ip(s, r).tolist() == [0, 0, 1024, 2047, 2047, 2047, 0]
    shift = np.float32(8.0)
    v = np.array([-11.0, -12.0, 3.0, 0.0], dtype=np.float32)
    b = ot.bins_l2(v, r, shift)
    assert b.tolist()[:3] == [0, 0, 2047]
    assert b[3] == int(np.float32(11.0) * (np.float32(2048) / np.float32(14.0)))


def test_walk_finds_the_bin_of_the_need_th_row():
    h = np.zeros(ot.BINS, dtype=np.int64)
    h[2047], h[2000], h[5] = 3, 2, 10
    assert ot.found_bin(h, 1) == 2047
    assert ot.found_bin(h, 3) == 2047          # need reached exactly at the top bin's boundary
    assert ot.found_bin(h, 4) == 2000
    assert ot.found_bin(h, 5) == 2000          # ... and exactly at the second bin's
    assert ot.found_bin(h, 6) == 5
    assert ot.found_bin(h, 15) == 5
    low = np.zeros(ot.BINS, dtype=np.int64)
    low[0] = 40_000                              # every row in the lowest bin
    assert ot.found_bin(low, 256) == 0


def test_threshold_restatement():
    r, eps = np.float32(1.25), ot.eps_ip(1.25)
    assert eps == np.float32(1.25 * 1.5 / 512)
    w = ot.bin_width(r)
    assert w == np.float32(2.5 / 2048)
    for found in (0, 1, 1023, 1024, 2047):
        for thr in ot.thresholds(found, r, eps):
            edge = -1.25 + found * 2.5 / 2048
            assert abs(float(thr) - (edge - 2 * float(eps) - float(w))) <= 2e-7
    # the lowest bin: the threshold lies below -r, so every row is a candidate
    assert max(ot.thresholds(0, r, eps)) < -r
    # L2: the grid starts at -r - shift and the bins are (2 r + shift) / 2048 wide
    shift = ot.shift_of(2.0)
    assert shift == 2.0 and ot.bin_width(r, shift) == np.float32(4.5 / 2048)
    thr = ot.thresholds(2047, r, np.float32(0.0), shift)[0]
    assert thr == np.float32(np.float32(-3.25 + 2047 * np.float32(4.5 / 2048)) - np.float32(4.5 / 2048))


def test_eps_l2_is_the_header_formula():
    r, qn, m, h = 1.0, 1.0, 1.0, 768
    d = r * 1.5 / 512 + h * 2.0 ** -24 * m * m + 2.0 ** -23 * (r + m * m)
    want = (d + h * 2.0 ** -24 * (qn * 1.0001 + m) ** 2) * 1.0001
    assert abs(float(ot.eps_l2(r, qn, m, h)) - want) <= 4 * np.spacing(np.float32(want))
