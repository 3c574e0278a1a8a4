"""The premises of tests/test_gpu_attention_exact.py, checked on the host: the float64 oracle (oracle/attention.py)
equals HF's eager attention with its masks; the key-count and needle inputs are exact in both 16-bit types and
their expectations follow from fp32 arithmetic; the needles win by >= 40 in the log2 domain and every trap would
win by as much if it leaked; the error bound holds for a faithful model of the kernel and fails for perturbed ones."""

from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import attention as oa

DTYPES = [pytest.param(torch.float16, id='f16'), pytest.param(torch.bfloat16, id='bf16')]


def prefix_mask(lens: list[int], S: int) -> torch.Tensor:
    return (torch.arange(S)[None] < torch.tensor(lens)[:, None]).long()


def hf_eager(qkv, mask, heads, kv_heads, d, mode, window):
    """transformers' eager_attention_forward in float64 with the masks masking_utils builds for each mode."""
    import transformers.masking_utils as mu
    from transformers.models.bert.modeling_bert import eager_attention_forward

    B, S = mask.shape
    q, k, v = oa.split_qkv(qkv.double(), heads, kv_heads, d)
    q, k, v = (t.view(B, S, -1, d).transpose(1, 2) for t in (q, k, v))
    k, v = (t.repeat_interleave(heads // kv_heads, dim=1) for t in (k, v))
    pad = mu.padding_mask_function(mask.bool())
    fn = {0: mu.bidirectional_mask_function,
          1: mu.sliding_window_bidirectional_mask_function(window) if mode == 1 else None,
          2: mu.sliding_window_causal_mask_function(window) if window else mu.causal_mask_function}[mode]
    add = mu.eager_mask(batch_size=B, q_length=S, kv_length=S, mask_function=mu.and_masks(fn, pad),
                        attention_mask=None, dtype=torch.float64)
    out, _ = eager_attention_forward(SimpleNamespace(training=False), q, k, v, add, scaling=d ** -0.5)
    return out.reshape(B * S, heads, d)


@pytest.mark.parametrize('mode,window,d,heads,kv_heads', [(0, 0, 64, 2, 2), (0, 0, 32, 3, 3), (1, 5, 64, 2, 2),
                                                           (2, 0, 128, 4, 2), (2, 7, 128, 4, 1)])
def test_oracle_equals_hf_eager_attention(mode, window, d, heads, kv_heads):
    g = torch.Generator().manual_seed(d + window)
    B, S = 4, 40
    mask = torch.ones(B, S, dtype=torch.int64)
    mask[1, 30:] = 0                  # right padding
    mask[2, :9] = 0                   # left padding
    mask[3, 12:20] = 0                # a hole
    if mode == 0:
        mask[3] = 0                   # nothing attended: HF's uniform average
    qkv = torch.randn(B * S, (heads + 2 * kv_heads) * d, generator=g)
    lay = oa.layout_of(mask, packed=False)
    ref = oa.reference(qkv, mask, heads, kv_heads, d, mode, window, lay)
    hf = hf_eager(qkv, mask, heads, kv_heads, d, mode, window)
    assert ref.spec.sum() > 0.8 * B * S
    torch.testing.assert_close(ref.out[ref.spec], hf[ref.spec], rtol=1e-12, atol=1e-12)
    # rows without a visible key: only the left-padded queries of the causal / windowed modes
    if mode == 0:
        assert bool(ref.spec.all())


def test_packed_oracle_equals_padded_oracle():
    g = torch.Generator().manual_seed(3)
    B, S, heads, d = 3, 70, 2, 64
    mask = prefix_mask([70, 1, 33], S)
    qkv = torch.randn(B, S, 3 * heads * d, generator=g)
    for mode, window in ((0, 0), (1, 4), (2, 9)):
        pad = oa.reference(qkv.view(B * S, -1), mask, heads, heads, d, mode, window, oa.layout_of(mask, False))
        lay = oa.layout_of(mask, True)
        assert lay.packed and lay.row0 == (0, 70, 71)
        pk = oa.reference(oa.to_layout(qkv, lay, 1e4), mask, heads, heads, d, mode, window, lay)
        valid = mask.bool().view(-1)
        torch.testing.assert_close(oa.to_layout(pad.out.view(B, S, heads, d), lay)[:sum(lay.len)],
                                   pk.out[:sum(lay.len)], rtol=1e-12, atol=1e-13)
        assert bool(pk.spec[:sum(lay.len)].all()) and not bool(pk.spec[sum(lay.len):].any())
        assert bool(pad.spec[valid].all())
    # a mask that is not a prefix everywhere keeps the identity layout
    mask[1, 0] = 0
    mask[1, 5] = 1
    assert not oa.layout_of(mask, True).packed


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('mode,window,d,heads,kv_heads,packed', [(0, 0, 64, 2, 2, False), (0, 0, 32, 2, 2, True),
                                                                  (1, 16, 64, 2, 2, True), (2, 65, 128, 4, 1, False)])
def test_count_inputs_are_exact_and_match_the_float64_oracle(dtype, mode, window, d, heads, kv_heads, packed):
    S = 200
    mask = prefix_mask([200, 131, 64, 1], S)
    if not packed:
        mask[1, :70] = 0     # left padding
        mask[2] = 0          # empty row
    lay = oa.layout_of(mask, packed)
    assert lay.packed == packed
    qkv, expected, spec, _ = oa.count_inputs(mask, heads, kv_heads, d, mode, window, lay, dtype)
    assert torch.equal(qkv.float().to(dtype), qkv)
    q, _, v = oa.split_qkv(qkv.float(), heads, kv_heads, d)
    assert not bool(q[:sum(lay.len) if packed else None].any())
    assert bool((v[:sum(lay.len) if packed else None] == v[:sum(lay.len) if packed else None].round()).all())
    ref = oa.reference(qkv, mask, heads, kv_heads, d, mode, window, lay)
    assert torch.equal(ref.spec, spec)
    # the float64 oracle rounded once to the storage type is the fp32 expectation (both round w count / n)
    assert torch.equal(ref.out[spec].to(dtype), expected[spec])
    # and the faithful model of the kernel reproduces it bit for bit
    got = oa.kernel_model(qkv, mask, heads, kv_heads, d, mode, window, lay, dtype)
    assert torch.equal(got[spec], expected[spec])


@pytest.mark.parametrize('d', [32, 64, 128])
def test_count_expectation_moves_for_one_key_more_or_less_and_for_a_row_sum_off_by_2_to_the_minus_7(d):
    """Keys 0 .. n-1 visible: the next key leaking in, the last one dropped, or a normalisation 1 + 2^-7 off
    changes the expected row at every n up to 1500 (both storage types)."""
    for dtype in (torch.float16, torch.bfloat16):
        for n in range(1, 1501):
            w = 7.0
            cnt = torch.bincount(torch.arange(n) % d, minlength=d).float()
            want = oa.finish(w * cnt, torch.tensor(float(n)), dtype)
            more = cnt.clone()
            more[n % d] += 1
            assert not torch.equal(oa.finish(w * more, torch.tensor(float(n + 1)), dtype), want)
            if n > 1:
                less = cnt.clone()
                less[(n - 1) % d] -= 1
                assert not torch.equal(oa.finish(w * less, torch.tensor(float(n - 1)), dtype), want)
            assert not torch.equal(oa.finish(w * cnt, torch.tensor(n * (1 + 2.0 ** -7)), dtype), want)


NEEDLE_CASES = [
    # mode, window, d, heads, kv_heads, S, lens, packed
    (0, 0, 64, 2, 2, 200, [200, 130, 64], False),
    (0, 0, 64, 2, 2, 200, [200, 130, 64], True),
    (0, 0, 32, 2, 2, 256, [256, 255, 1], True),
    (0, 0, 64, 2, 2, 1100, [1100, 1030], False),
    (1, 16, 64, 2, 2, 300, [300, 129, 65], True),
    (1, 65, 64, 2, 2, 300, [300, 280], False),
    (2, 0, 128, 4, 1, 260, [260, 128, 100], True),
    (2, 63, 128, 4, 2, 300, [300, 190], False),
]


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('mode,window,d,heads,kv_heads,S,lens,packed', NEEDLE_CASES)
def test_needles_win_by_40_and_traps_would_win_by_40(dtype, mode, window, d, heads, kv_heads, S, lens, packed):
    mask = prefix_mask(lens, S)
    if not packed and len(lens) > 1:
        mask[1, :3] = 0      # left padding
    lay = oa.layout_of(mask, packed)
    nd = oa.needle_inputs(mask, heads, kv_heads, d, mode, window, lay, dtype, seed=S)
    assert torch.equal(nd.qkv.float().to(dtype), nd.qkv)
    worst, worst_trap = oa.needle_margins(nd, heads, kv_heads, d, mask, mode, window, lay)
    assert worst >= 40 and worst_trap >= 40, (worst, worst_trap)
    assert len(nd.traps) > 0 and nd.decoys > 0
    assert nd.check.sum() > 0.9 * sum(lay.len) * heads - heads * 3
    # the oracle agrees: the output is v of the target to far below a 16-bit ulp
    ref = oa.reference(nd.qkv, mask, heads, kv_heads, d, mode, window, lay)
    sel = nd.check
    assert torch.equal(ref.out[sel].to(dtype), nd.expected[sel])
    # and so does the faithful kernel model, bit for bit
    got = oa.kernel_model(nd.qkv, mask, heads, kv_heads, d, mode, window, lay, dtype)
    assert torch.equal(got[sel], nd.expected[sel])
    if packed and len(lens) > 1:   # some trap sits in the next sequence's first keys
        nxt = [r for _, _, r in nd.traps if any(lay.row0[b] <= r < lay.row0[b] + 4 for b in range(1, lay.B))]
        assert nxt


@pytest.mark.parametrize('d', [32, 64, 128])
def test_needle_alpha_gives_a_40_margin(d):
    a = oa.needle_alpha(d)
    assert a == {32: 256, 64: 256, 128: 512}[d]
    assert a / math.sqrt(d) * oa.LOG2E >= 40


# ------------------------------------------------------------------------- the bound is met, and it is not vacuous
def sharp_case(dtype, S=512, heads=12, sharp=1.0):
    g = torch.Generator().manual_seed(S)
    B = 2
    qkv = torch.randn(B * S, 3 * heads * 64, generator=g)
    qkv[:, :heads * 64] *= sharp
    mask = torch.ones(B, S, dtype=torch.int64)
    lay = oa.layout_of(mask, False)
    qkv = qkv.to(dtype)
    return qkv, mask, lay, oa.reference(qkv, mask, heads, heads, 64, 0, 0, lay)


PERTURBATIONS = {
    'scale x1.01': dict(scale=1.01),
    'row sum x(1+2^-5)': dict(tot_factor=1 + 2.0 ** -5),
    'row sum x(1+2^-7)': dict(tot_factor=1 + 2.0 ** -7),
    'P in fp8 e4m3': dict(p_dtype=torch.float8_e4m3fn),
    '1% exp error': dict(exp_err=0.01),
}
# which perturbation the bound catches at the (2, 512, 12) case, by storage type.  The bound is ~8x looser in
# bfloat16 (u = 2^-8): there a row sum 0.8 % too large stays inside it, and the key-count and needle families must
# catch that one instead -- they do, bit for bit (test_count_expectation_moves_...).
CAUGHT = {
    torch.float16: set(PERTURBATIONS),
    torch.bfloat16: set(PERTURBATIONS) - {'row sum x(1+2^-7)'},
}


@pytest.mark.parametrize('dtype', DTYPES)
def test_faithful_kernel_model_meets_the_bound_and_perturbed_ones_do_not(dtype):
    qkv, mask, lay, ref = sharp_case(dtype)
    faithful = oa.kernel_model(qkv, mask, 12, 12, 64, 0, 0, lay, dtype)
    assert oa.excess(faithful, ref, dtype, oa.E_EX2) <= 1.0
    # the polynomial variants' looser exponentials are inside the bound too
    poly = oa.kernel_model(qkv, mask, 12, 12, 64, 0, 0, lay, dtype, exp_err=oa.E_POLY)
    assert oa.excess(poly, ref, dtype, oa.E_POLY) <= 1.0
    caught = set()
    for name, kw in PERTURBATIONS.items():
        if oa.excess(oa.kernel_model(qkv, mask, 12, 12, 64, 0, 0, lay, dtype, **kw), ref, dtype, oa.E_EX2) > 1.0:
            caught.add(name)
    assert caught == CAUGHT[dtype]


def test_bound_catches_p_through_bfloat16_in_the_half_build_on_sharp_attention():
    """P rounded to bfloat16 instead of half (8x the P rounding) hides in the bound on diffuse attention; with
    sharper scores a few keys dominate each row and it shows."""
    qkv, mask, lay, ref = sharp_case(torch.float16, S=256, heads=4, sharp=3.0)
    faithful = oa.kernel_model(qkv, mask, 4, 4, 64, 0, 0, lay, torch.float16)
    assert oa.excess(faithful, ref, torch.float16, oa.E_EX2) <= 1.0
    bf = oa.kernel_model(qkv, mask, 4, 4, 64, 0, 0, lay, torch.float16, p_dtype=torch.bfloat16)
    assert oa.excess(bf, ref, torch.float16, oa.E_EX2) > 1.0


def test_finish_is_ieee_division_then_round_to_nearest():
    o = torch.tensor([1.0, 2.0, 3.0, 1000.0, 7.0])
    tot = torch.tensor([3.0, 3.0, 7.0, 3.0, 1.0])
    for dtype in (torch.float16, torch.bfloat16):
        got = oa.finish(o, tot, dtype)
        inv = np.float32(1.0) / tot.numpy().astype(np.float32)
        want = torch.from_numpy((o.numpy().astype(np.float32) * inv).astype(np.float32)).to(dtype)
        assert torch.equal(got, want)
        assert got[-1].item() == 7.0
