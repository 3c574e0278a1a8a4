"""-m gpu: every attention instantiation (csrc/attention.cuh) in both builds and both token layouts, judged by
inputs whose output is known bit for bit and by a float64 reference with an error bound derived from the kernel's
arithmetic (oracle/attention.py; its premises are checked on the host by tests/test_attention_oracle_cpu.py).

(a) key counts: q = 0 and v_j[c] = w [j = c mod D], so O[i, c] = w count_c(i) / n(i), exact in fp32: one key too
    many or too few, a neighbouring sequence's or kv head's rows, or a normalisation one 16-bit ulp off changes it.
(b) needles: each query aims at one key at an edge (first / last visible, 63/64, 127/128, window edges, diagonal,
    last key) and wins by >= 40 in the log2 domain; keys it must not see carry patterns that would win if they
    leaked.  The output must be v of the target exactly.
(c) random inputs (ragged, left padding, holes, empty rows, rescale ramps, sharp scores) against the float64
    reference, within oracle.attention.error_bound.

The padded layout goes through the standalone entry points (b2e_attention_*), the packed one through
b2e_debug_attention_packed, which runs the encoder's own layout preparation and launch."""

from __future__ import annotations

import ctypes
import functools

import pytest
import torch

from distllm_b200 import _native as nv
from oracle import attention as oa

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(params=[torch.float16, torch.bfloat16], ids=['f16', 'bf16'])
def h16(request):
    return request.param


# instantiation: (head_dim, mode, head_dim-64 variant or None, heads, kv_heads)
INSTANTIATIONS = {
    'd32': (32, 0, None, 2, 2),
    **{f'd64-v{v}': (64, 0, v, 2, 2) for v in (0, 1, 5, 64, 65, 69, 193)},
    **{f'win-v{v}': (64, 1, v, 2, 2) for v in (0, 64, 128, 192)},
    **{f'gqa{r}': (128, 2, None, 4, 4 // r) for r in (1, 2, 4)},
    # ESM C's head counts (esmc-300m, esmc-600m): qkv rows of 2880 and 3456 columns
    'esmc15': (64, 0, None, 15, 15),
    'esmc18': (64, 0, None, 18, 18),
}
RAGGED = (513, 512, 511, 257, 256, 255, 129, 128, 127, 65, 64, 63, 1)
# shape: (S, lengths of the right-padded rows or a named mask, rows of K scaled up along the sequence, q scale)
SHAPES = {
    'S513-ragged': (513, RAGGED, False, 1.0),
    'S300-ragged': (300, (300, 257, 129, 65, 1), False, 1.0),
    'S1026-ramp': (1026, (1026, 1000), True, 1.0),
    'S1500-sharp': (1500, (1500, 700), False, 3.0),
    'S1': (1, (1,) * 5, False, 1.0),
    'S300-holes': (300, 'holes', False, 1.0),      # left padding, a hole, an empty row: padded layout only
    'waves': (300, 'waves', False, 1.0),           # 40 sequences x 12 heads: far more CTAs than twice the SMs
}
WINDOWS = (1, 16, 63, 64, 65, 127, 128, 300)


def cases(family: str):
    out = []
    for inst, (d, mode, _, _, _) in INSTANTIATIONS.items():
        if mode == 0:
            shapes = [(s, 0) for s in ('S513-ragged', 'S1026-ramp', 'S1500-sharp', 'S1', 'S300-holes')]
        else:
            shapes = [('S300-ragged', w) for w in WINDOWS] + [('S513-ragged', 64), ('S1026-ramp', 65),
                                                              ('S1500-sharp', 300), ('S1', 16), ('S300-holes', 63)]
            if mode == 2:
                shapes.append(('S513-ragged', 0))
        if family != 'needle' and inst in ('d32', 'd64-v1', 'd64-v193', 'win-v192', 'gqa4'):
            shapes.append(('waves', 0 if mode == 0 else 128))
        for shape, w in shapes:
            for layout in ('padded', 'packed'):
                if layout == 'packed' and shape == 'S300-holes':
                    continue
                out.append(pytest.param(inst, shape, w, layout, id=f'{inst}-{shape}-w{w}-{layout}'))
    return out


def make_mask(shape: str, mode: int) -> torch.Tensor:
    S, lens, _, _ = SHAPES[shape]
    if lens == 'holes':
        m = torch.ones(4, S, dtype=torch.int64)
        m[1, :70] = 0            # left padding
        m[2, 100:140] = 0        # a hole
        m[3, 250:] = 0
        if mode == 0:
            m[3] = 0             # nothing attended: the uniform average over S keys
        return m
    if lens == 'waves':
        lens = torch.randint(1, S + 1, (40,), generator=torch.Generator().manual_seed(5)).tolist()
    return (torch.arange(S)[None] < torch.tensor(lens)[:, None]).long()


def heads_of(inst: str, shape: str) -> tuple[int, int]:
    _, _, _, heads, kv_heads = INSTANTIATIONS[inst]
    if shape == 'waves':
        return heads * 6, kv_heads * 6
    return heads, kv_heads


@pytest.fixture
def variant(h16):
    """Selects the head_dim-64 variant of a case for the library of the storage type; back to the default after."""
    lib = nv.load(nv.storage_of(h16))
    lib.b2e_debug_set_att3_variant.argtypes = [ctypes.c_int]

    def select(v):
        if v is not None:
            assert lib.b2e_debug_set_att3_variant(v) == 0
    yield select
    lib.b2e_debug_set_att3_variant(-1)


def run(inst: str, qkv: torch.Tensor, mask: torch.Tensor, heads: int, kv_heads: int, window: int,
        lay: oa.Layout) -> torch.Tensor:
    d, mode, _, _, _ = INSTANTIATIONS[inst]
    B, S = mask.shape
    if lay.packed:
        ctx = nv.attention_packed(qkv, mask, B, S, heads, kv_heads, d, window, causal=mode == 2)
    elif mode == 2:
        ctx = nv.attention_causal_d128(qkv, mask, B, S, heads, kv_heads, window)
    elif mode == 1:
        ctx = nv.attention_d64_window(qkv, mask, B, S, heads, window)
    elif d == 32:
        ctx = nv.attention_d32(qkv, mask, B, S, heads)
    else:
        ctx = nv.attention_d64(qkv, mask, B, S, heads)
    torch.cuda.synchronize()
    return ctx.view(B * S, heads, d)


def bits(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().view(torch.int16)


def check_untouched_tail(got: torch.Tensor, lay: oa.Layout) -> None:
    """Rows past the last packed token belong to no sequence: the kernel must leave them alone."""
    if lay.packed:
        assert not bool(got[sum(lay.len):].any())


# ------------------------------------------------------------------------------------------------ (a) key counts
@pytest.mark.parametrize('inst,shape,window,layout', cases('count'))
def test_key_counts_bit_exact(dev, h16, variant, inst, shape, window, layout):
    d, mode, v, _, _ = INSTANTIATIONS[inst]
    heads, kv_heads = heads_of(inst, shape)
    mask = make_mask(shape, mode)
    lay = oa.layout_of(mask, layout == 'packed')
    assert lay.packed == (layout == 'packed')
    trap = 4096.0
    qkv, expected, spec, zero = oa.count_inputs(mask, heads, kv_heads, d, mode, window, lay, h16, trap=trap)
    variant(v)
    got = run(inst, qkv.to(dev), mask.to(dev), heads, kv_heads, window, lay).cpu()
    assert bool(torch.isfinite(got.float()).all())
    check_untouched_tail(got, lay)
    same = bits(got) == bits(expected)
    if v is not None and (v >> 2) & 3 and h16 == torch.bfloat16:
        # poly_exp2 clamps at -126: a masked key weighs 2^-126 instead of 0, which bfloat16 P keeps.  A column no
        # visible key contributes to can then read sum(2^-126 v) / n -- far below any value a 16-bit activation
        # resolves next to the row's other entries; every column with a count stays bit-exact
        leak = oa.POLY_FLOOR * oa.KC * ((mask.shape[1] + oa.KC - 1) // oa.KC) * trap
        g = got.float()
        tiny = zero[:, None, :].expand_as(g) & (g >= 0) & (g <= leak)
        same |= tiny
    bad = spec[:, None, None].expand_as(same) & ~same
    assert not bool(bad.any()), f'{int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}'


# -------------------------------------------------------------------------------------------------- (b) needles
@functools.lru_cache(maxsize=None)
def needles(inst: str, shape: str, window: int, packed: bool):
    """One set of needle inputs for both builds: v rounded to bfloat16 is exact in half too."""
    d, mode, _, _, _ = INSTANTIATIONS[inst]
    heads, kv_heads = heads_of(inst, shape)
    mask = make_mask(shape, mode)
    lay = oa.layout_of(mask, packed)
    nd = oa.needle_inputs(mask, heads, kv_heads, d, mode, window, lay, torch.bfloat16, seed=mask.shape[1] + window)
    worst, worst_trap = oa.needle_margins(nd, heads, kv_heads, d, mask, mode, window, lay)
    assert worst >= 40 and worst_trap >= 40, (worst, worst_trap)
    return mask, lay, nd


@pytest.mark.parametrize('inst,shape,window,layout', cases('needle'))
def test_needles_bit_exact(dev, h16, variant, inst, shape, window, layout):
    _, _, v, _, _ = INSTANTIATIONS[inst]
    heads, kv_heads = heads_of(inst, shape)
    mask, lay, nd = needles(inst, shape, window, layout == 'packed')
    qkv, expected = nd.qkv.to(h16), nd.expected.to(h16)
    assert torch.equal(qkv.to(torch.bfloat16), nd.qkv)
    variant(v)
    got = run(inst, qkv.to(dev), mask.to(dev), heads, kv_heads, window, lay).cpu()
    assert bool(torch.isfinite(got.float()).all())
    check_untouched_tail(got, lay)
    sel = nd.check
    ok = (bits(got) == bits(expected)).all(-1) | ~sel
    assert bool(ok.all()), f'{int((~ok).sum())} rows miss their target key, first (row, head) {(~ok).nonzero()[0]}'


# ------------------------------------------------------------------------------------------- (c) random, bound
@pytest.mark.parametrize('inst,shape,window,layout', cases('random'))
def test_random_inputs_within_the_error_bound(dev, h16, variant, inst, shape, window, layout):
    d, mode, v, _, _ = INSTANTIATIONS[inst]
    heads, kv_heads = heads_of(inst, shape)
    mask = make_mask(shape, mode)
    B, S = mask.shape
    lay = oa.layout_of(mask, layout == 'packed')
    _, _, ramp, sharp = SHAPES[shape]
    g = torch.Generator(device=dev).manual_seed(S * 7 + window + d)
    x = torch.randn(B, S, heads + 2 * kv_heads, d, device=dev, generator=g)
    x[:, :, :heads] *= sharp
    if ramp:   # key norms grow along the sequence: the running maximum jumps and the rescale fires
        x[:, :, heads:heads + kv_heads] *= torch.linspace(0.2, 6.0, S, device=dev)[None, :, None, None]
    qkv = oa.to_layout(x.reshape(B, S, -1).to(h16), lay, fill=1e4)
    variant(v)
    got = run(inst, qkv, mask.to(dev), heads, kv_heads, window, lay)
    assert bool(torch.isfinite(got.float()).all())
    check_untouched_tail(got, lay)
    ref = oa.reference(qkv, mask, heads, kv_heads, d, mode, window, lay)
    e = oa.e_exp(v) if v is not None else oa.E_EX2
    assert oa.excess(got, ref, h16, e) <= 1.0


# ------------------------------------------------------------------------------------------- packed debug entry
@pytest.mark.parametrize('inst,window', [('d32', 0), ('d64-v193', 0), ('d64-v5', 0), ('win-v0', 63), ('gqa2', 100)])
def test_packed_entry_falls_back_to_the_padded_layout_bit_for_bit(dev, h16, variant, inst, window):
    """A mask that is not a non-empty prefix in every row (left padding, a hole, an empty row) keeps the identity
    layout: the debug entry must give exactly what the standalone padded entry gives."""
    d, mode, v, heads, kv_heads = INSTANTIATIONS[inst]
    mask = make_mask('S300-holes', mode)
    B, S = mask.shape
    lay = oa.layout_of(mask, True)
    assert not lay.packed
    g = torch.Generator(device=dev).manual_seed(17)
    qkv = torch.randn(B * S, (heads + 2 * kv_heads) * d, device=dev, generator=g).to(h16)
    variant(v)
    md = mask.to(dev)
    want = run(inst, qkv, md, heads, kv_heads, window, lay)
    got = nv.attention_packed(qkv, md, B, S, heads, kv_heads, d, window, causal=mode == 2).view_as(want)
    assert torch.equal(bits(got), bits(want))


def test_packed_entry_rejects_shapes_without_a_kernel(dev):
    qkv = torch.zeros(64, 3 * 2 * 32, device=dev, dtype=torch.float16)
    mask = torch.ones(1, 64, dtype=torch.int64, device=dev)
    with pytest.raises(nv.NativeError, match='no kernel'):
        nv.attention_packed(qkv, mask, 1, 64, 2, 2, 32, window=8)
    with pytest.raises(nv.NativeError, match='no kernel'):
        nv.attention_packed(qkv, mask, 1, 64, 2, 2, 32, causal=True)
