"""-m gpu: the persistent ping-pong GEMM (csrc/gemm.cuh) against absolute references, in both builds and at both tile
widths wherever the 192-wide kernel exists (oracle/gemm.py; its premises are checked on the host by
tests/test_gemm_oracle_cpu.py).

(a) provenance: one-hot W rows (out[m, n] = A[m, pi(n)]) and one-hot A rows (out[m, n] = W[n, sigma(m)]) with any
    finite normal 16-bit values, fp32 bias and 16-bit residuals: every element lands where it belongs, bit for bit.
(b) integer sums: ternary operands whose every partial sum is a small integer, K/64 from 1 to 224 (the 3-, 4- and
    5-stage rings at, below and past a wrap), M across the register-path tails, N from 128 to 28 672: bit for bit.
(c) schedule shapes derived from the SM count: CTAs with one, two, three and about forty turns, either consumer last.
(d) guard rows: every call writes into the middle of a sentinel-filled buffer; nothing outside [M, N] may change and
    nothing inside may keep the sentinel.
(e) the device row count (b2e_debug_gemm_rows): rows below it are the plain call's, rows at or beyond it untouched.
(f) activation epilogues within oracle.gemm.activation_error_bound: every finite 16-bit value and a dense fp32 range
    as bias (W = 0) and as A (W one-hot), the gated pairs with up values no wrong pairing fits, half's saturation.
(g) NF4 against the host's dequantisation, not against the 16-bit kernel.
(h) a bias or residual the epilogue would not read is rejected.

A failure names the first mismatching (m, n), its tile, CTA, consumer and turn, and the expected and actual bits."""

from __future__ import annotations

import ctypes as C
from contextlib import contextmanager

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from distllm_b200.embed.encoders import nf4
from distllm_b200.embed.encoders.weights import interleave_gate_up
from oracle import gemm as og

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FFF            # a NaN in both storage types that no epilogue produces from finite inputs
GUARD = 2                    # whole sentinel rows before and after the output (keeps its 16-byte alignment)
GLU = (nv.EPI_SWIGLU, nv.EPI_GEGLU)


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


@pytest.fixture(params=[torch.float16, torch.bfloat16], ids=['f16', 'bf16'])
def h16(request):
    return request.param


@contextmanager
def gemm_bn(lib, bn: int):
    lib.b2e_debug_set_gemm_bn.argtypes = [C.c_int]
    assert lib.b2e_debug_set_gemm_bn(bn) == 0
    try:
        yield
    finally:
        lib.b2e_debug_set_gemm_bn(0)


def width(lib, n: int, epi: int, nf4_w: bool) -> int:
    out = C.c_int(-1)
    assert lib.b2e_debug_gemm_bn(n, epi, int(nf4_w), C.byref(out)) == 0
    return out.value


def widths(n: int) -> list[int]:
    """The tile widths a 16-bit W of n rows can run at with a non-gated epilogue."""
    return [128, 192] if n % 192 == 0 else [128]


class Run:
    """One GEMM call into a guarded buffer: ``out`` is the [M, N_out] window, ``bn`` the width it ran at."""

    def __init__(self, dev, h16, a, w, bias, resid, m, n, k, epi, *, bn=128, absmax=None, m_dev=None):
        lib = nv.load(nv.storage_of(h16))
        n_out = n // 2 if epi in GLU else n
        self.buf = torch.full((m + 2 * GUARD, n_out), SENTINEL, dtype=torch.int16, device=dev).view(h16)
        self.out = self.buf[GUARD:GUARD + m]
        self.m, self.n, self.epi = m, n, epi
        stream = nv.stream_ptr(dev)
        ptr = nv._ptr
        with gemm_bn(lib, bn):
            self.bn = width(lib, n, epi, absmax is not None)
            if m_dev is not None:
                md = torch.tensor([m_dev], dtype=torch.int32, device=dev)
                lib.b2e_debug_gemm_rows.restype = C.c_int
                lib.b2e_debug_gemm_rows.argtypes = [C.c_void_p] * 6 + [C.c_int] * 4 + [C.c_void_p] * 2
                rc = lib.b2e_debug_gemm_rows(a.data_ptr(), w.data_ptr(), ptr(absmax), ptr(bias), ptr(resid),
                                             self.out.data_ptr(), m, n, k, epi, md.data_ptr(), stream)
            elif absmax is not None:
                rc = lib.b2e_gemm_nf4(a.data_ptr(), w.data_ptr(), absmax.data_ptr(), ptr(bias), ptr(resid),
                                      self.out.data_ptr(), m, n, k, epi, stream)
            else:
                rc = lib.b2e_gemm_h16(a.data_ptr(), w.data_ptr(), ptr(bias), ptr(resid), self.out.data_ptr(),
                                      m, n, k, epi, stream)
        nv.check(rc, lib)
        torch.cuda.synchronize(dev)
        self.sms = torch.cuda.get_device_properties(dev).multi_processor_count
        guard = torch.cat([self.buf[:GUARD], self.buf[GUARD + m:]]).view(torch.int16)
        assert (guard == SENTINEL).all(), f'{self.what()}: the GEMM wrote outside its [M, N] output'

    def what(self) -> str:
        return f'M={self.m} N={self.n} epi={self.epi} BN={self.bn}'

    def locate(self, m: int, col: int) -> str:
        """Tile, CTA, consumer and turn of output (m, col), as gemm_tiles and the launch assign them."""
        glu = self.epi in GLU
        n_tiles = self.n // (128 if glu else self.bn)
        tile = (m // 128) * n_tiles + col // (64 if glu else self.bn)
        tiles = n_tiles * -(-self.m // 128)
        grid = min(tiles, self.sms)
        turn = tile // grid
        return f'tile {tile} (row block {m // 128}, column block {tile % n_tiles}), CTA {tile % grid} of {grid}, ' \
               f'consumer {turn % 2}, turn {turn}'

    def mismatch(self, rows: torch.Tensor, cols: torch.Tensor, want: torch.Tensor, got: torch.Tensor, n_bad: int,
                 label: str) -> str:
        m, col = int(rows[0]), int(cols[0])
        w, g = int(want[0]) & 0xFFFF, int(got[0]) & 0xFFFF
        return (f'{self.what()} {label}: {n_bad} elements wrong; first (m={m}, n={col}) in {self.locate(m, col)}: '
                f'expected 0x{w:04x}, got 0x{g:04x}')

    def assert_bits(self, want: torch.Tensor, rows: slice = slice(None), label: str = '') -> None:
        got = self.out[rows].contiguous().view(torch.int16)
        ref = want.to(self.out.dtype).contiguous().view(torch.int16)
        assert got.shape == ref.shape
        bad = got != ref
        if bad.any():
            idx = bad.nonzero()
            r0 = rows.start or 0
            pytest.fail(self.mismatch(idx[:, 0] + r0, idx[:, 1], ref[bad], got[bad], idx.shape[0], label))

    def assert_within(self, want64: torch.Tensor, bound: torch.Tensor, label: str = '') -> None:
        got = self.out.double()
        ref = want64.clamp(-og.HALF_MAX, og.HALF_MAX) if self.out.dtype == torch.float16 else want64
        bad = ~((got - ref).abs() <= bound)
        if bad.any():
            idx = bad.nonzero()
            r, c = int(idx[0, 0]), int(idx[0, 1])
            pytest.fail(f'{self.what()} {label}: {idx.shape[0]} elements outside the bound; first (m={r}, n={c}) in '
                        f'{self.locate(r, c)}: ref {float(ref[r, c])!r}, got {float(got[r, c])!r}, '
                        f'bound {float(bound[r, c])!r}')


def scaled_bias(n: int, gen: torch.Generator) -> torch.Tensor:
    """Arbitrary fp32 values over many binades (small ones too: a bias read from the wrong group must show)."""
    return torch.randn(n, generator=gen, device=gen.device) * torch.exp2(
        torch.randint(-12, 13, (n,), generator=gen, device=gen.device).float())


# ------------------------------------------------------------------------------------------------ (a) provenance
PROVENANCE = [(517, 768, 320), (129, 384, 576), (300, 1152, 64)]
EPI_CASES = [(nv.EPI_BIAS, False, False), (nv.EPI_BIAS, True, False), (nv.EPI_BIAS_RESID, True, True),
             (nv.EPI_BIAS_RESID, False, True)]


@pytest.mark.parametrize('bn', [128, 192])
@pytest.mark.parametrize('m, n, k', PROVENANCE)
@pytest.mark.parametrize('side', ['w-one-hot', 'a-one-hot'])
def test_provenance_bit_for_bit(dev, h16, side, m, n, k, bn):
    g = torch.Generator(device=dev).manual_seed(m + n + k)
    if side == 'w-one-hot':       # out[m, n] = A[m, pi(n)]
        w, idx = og.one_hot_rows(n, k, h16, dev)
        a = og.random_normals((m, k), h16, g)
        acc = a.float()[:, idx]
    else:                         # out[m, n] = W[n, sigma(m)]
        a, idx = og.one_hot_rows(m, k, h16, dev)
        w = og.random_normals((n, k), h16, g)
        acc = w.float()[:, idx].T.contiguous()
    for epi, with_bias, with_resid in EPI_CASES:
        bias = scaled_bias(n, g) if with_bias else None
        resid = og.random_normals((m, n), h16, g) if with_resid else None
        run = Run(dev, h16, a, w, bias, resid, m, n, k, epi, bn=bn)
        run.assert_bits(og.epilogue(acc, bias, resid, h16), label=f'{side} bias={with_bias}')


# ------------------------------------------------------------------------------------------------ (b) integer sums
SUMS = ([(517, 768, 64 * kb) for kb in (1, 2, 3, 4, 5, 6, 9, 12, 48)]
        + [(257, 4096, 14336), (129, 3072, 14336)]
        + [(m, 384, 320) for m in (1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 517, 4099, 20000)]
        + [(129, 128, 128), (129, 256, 128), (129, 640, 128), (129, 1152, 192), (129, 28672, 128),
           (4099, 3072, 768), (20000, 768, 768)])


@pytest.mark.parametrize('m, n, k', SUMS)
def test_integer_sums_bit_for_bit(dev, h16, m, n, k):
    g = torch.Generator(device=dev).manual_seed(m * 31 + n * 7 + k)
    a, w = og.ternary_pair(m, n, k, g, h16)
    acc = og.exact_product(a, w)
    bias = torch.randint(-8, 9, (n,), generator=g, device=dev).float()
    resid = torch.randint(-64, 65, (m, n), generator=g, device=dev).to(h16)
    for bn in widths(n):
        Run(dev, h16, a, w, None, None, m, n, k, nv.EPI_BIAS, bn=bn).assert_bits(og.epilogue(acc, None, None, h16))
        Run(dev, h16, a, w, bias, resid, m, n, k, nv.EPI_BIAS_RESID, bn=bn).assert_bits(
            og.epilogue(acc, bias, resid, h16), label='resid')


# ------------------------------------------------------------------------------------------------ (c) schedules
def schedule_shapes(sms: int, bn: int) -> dict[str, tuple[int, int]]:
    """name -> (row tiles, column tiles): the tile count against the SM count (grid = min(tiles, SMs)).  At BN = 192
    N is a multiple of 384, so the column tiles come in pairs and an odd count becomes the next even one."""
    cols = 1 if bn == 128 else 2
    counts = {'tiles<SMs': sms - cols, 'tiles=SMs': sms, 'SMs+1': sms + 1, '2SMs-1': 2 * sms - 1, '2SMs+1': 2 * sms + 1,
              '3 per CTA': 3 * sms}
    shapes = {name: (-(-t // cols), cols) for name, t in counts.items()}
    shapes['40 per CTA'] = (5 * sms, 8)
    return shapes


@pytest.mark.parametrize('shape', ['tiles<SMs', 'tiles=SMs', 'SMs+1', '2SMs-1', '2SMs+1', '3 per CTA', '40 per CTA'])
@pytest.mark.parametrize('bn', [128, 192])
def test_schedule_shapes_bit_for_bit(dev, h16, sms, shape, bn):
    rows_t, cols_t = schedule_shapes(sms, bn)[shape]
    m, n, k = 128 * rows_t - 3, bn * cols_t, 128      # the last row tile has a tail: register-path stores
    tiles = rows_t * cols_t
    turns = [len(range(c, tiles, min(tiles, sms))) for c in range(min(tiles, sms))]
    g = torch.Generator(device=dev).manual_seed(tiles * bn)
    a, w = og.ternary_pair(m, n, k, g, h16)
    bias = torch.randint(-8, 9, (n,), generator=g, device=dev).float()
    run = Run(dev, h16, a, w, bias, None, m, n, k, nv.EPI_BIAS, bn=bn)
    assert run.bn == bn
    run.assert_bits(og.epilogue(og.exact_product(a, w), bias, None, h16), label=f'{shape}, turns {set(turns)}')


# ------------------------------------------------------------------------------------------------ (e) device rows
@pytest.mark.parametrize('kind', ['bn128', 'bn192', 'swiglu', 'nf4'])
def test_device_row_count(dev, h16, kind):
    m, k = 517, 192
    n = 256 if kind == 'swiglu' else 768
    epi = nv.EPI_SWIGLU if kind == 'swiglu' else nv.EPI_BIAS
    bn = 192 if kind == 'bn192' else 128
    g = torch.Generator(device=dev).manual_seed(n + len(kind))
    a, w = og.ternary_pair(m, n, k, g, h16)
    absmax = None
    if kind == 'nf4':
        w = torch.randint(0, 256, (n, k // 2), generator=g, device=dev, dtype=torch.uint8)
        absmax = (torch.rand((k // 64, n), generator=g, device=dev) - 0.3).contiguous()
    bias = None if epi in GLU else scaled_bias(n, g)
    full = Run(dev, h16, a, w, bias, None, m, n, k, epi, bn=bn, absmax=absmax)
    assert full.bn == bn
    if kind in ('bn128', 'bn192'):
        full.assert_bits(og.epilogue(og.exact_product(a, w), bias, None, h16))
    for m_dev in (0, 1, 127, 128, 129, m - 1, m):
        run = Run(dev, h16, a, w, bias, None, m, n, k, epi, bn=bn, absmax=absmax, m_dev=m_dev)
        run.assert_bits(full.out[:m_dev], rows=slice(0, m_dev), label=f'm_dev={m_dev}, rows below it')
        untouched = torch.full((m - m_dev, run.out.shape[1]), SENTINEL, dtype=torch.int16, device=dev).view(h16)
        run.assert_bits(untouched, rows=slice(m_dev, m), label=f'm_dev={m_dev}, rows at or beyond it untouched')


# ------------------------------------------------------------------------------------------------ (f) activations
def sweep(h16) -> torch.Tensor:
    """Every finite 16-bit value of the build (normal half / all bfloat16), a dense fp32 range across the GELU fit
    and its clamp at |x| = 5.657, and fp32 magnitudes up to fp32's (half) or bfloat16's (bfloat16) largest."""
    table = og.value_table(h16).double()
    dense = torch.linspace(-12, 12, 60_001, dtype=torch.float64)
    edge = og.GELU_CLAMP + torch.linspace(-1e-3, 1e-3, 201, dtype=torch.float64)
    big = torch.logspace(-30, float(np.log10(3.4e38 if h16 == torch.float16 else 3.3895e38)), 4001,
                         dtype=torch.float64)
    return torch.cat([table, dense, edge, -edge, big, -big]).float()


def as_columns(x: torch.Tensor, n_mult: int) -> torch.Tensor:
    """x padded with zeros to a multiple of n_mult."""
    return torch.cat([x, x.new_zeros((-x.numel()) % n_mult)])


@pytest.mark.parametrize('bn', [128, 192])
def test_gelu_every_value_as_bias(dev, h16, bn):
    """W = 0, so the pre-activation is exactly the fp32 bias."""
    x = as_columns(sweep(h16), 384).to(dev)
    n, m, k = x.numel(), 3, 64
    a = torch.ones((m, k), dtype=h16, device=dev)
    w = torch.zeros((n, k), dtype=h16, device=dev)
    run = Run(dev, h16, a, w, x, None, m, n, k, nv.EPI_BIAS_GELU, bn=bn)
    assert run.bn == bn
    xs = x.double().cpu().numpy()
    bound = torch.from_numpy(og.activation_error_bound(xs, h16, 'gelu')).to(dev).expand(m, n)
    run.assert_within(og.gelu64(x).expand(m, n), bound, 'gelu(bias)')
    if h16 == torch.float16:      # saturation, not inf
        big = x > 70000
        assert big.any() and (run.out[:, big].float() == og.HALF_MAX).all()


@pytest.mark.parametrize('bn', [128, 192])
def test_gelu_every_value_through_a(dev, h16, bn):
    """W one-hot: out[m, n] = gelu(A[m, pi(n)]) with the 16-bit values of the build as A."""
    table = og.value_table(h16)
    n = k = 384
    w, idx = og.one_hot_rows(n, k, h16, dev)
    a = as_columns(table, k).reshape(-1, k).to(dev)
    m = a.shape[0]
    run = Run(dev, h16, a, w, None, None, m, n, k, nv.EPI_BIAS_GELU, bn=bn)
    assert run.bn == bn
    x = a.double()[:, idx]
    bound = torch.from_numpy(og.activation_error_bound(x.cpu().numpy(), h16, 'gelu')).to(dev)
    run.assert_within(og.gelu64(x), bound, 'gelu(A)')


def up_values(n_out: int, dev) -> torch.Tensor:
    """Up value of output column j: (1 + (j % 8) / 8) 2^((j % 64) // 8), 64 distinct values in each 64-column output
    block (exact in both types), at least 6 % apart: pairing a gate with any other up column of its W tile moves
    the product by more than 4x the bound (asserted on the reference)."""
    j = torch.arange(n_out, device=dev)
    return (1 + (j % 8).double() / 8) * torch.exp2(((j % 64) // 8).double())


@pytest.mark.parametrize('epi', [nv.EPI_SWIGLU, nv.EPI_GEGLU], ids=['swiglu', 'geglu'])
def test_gated_epilogues(dev, h16, epi):
    kind = 'silu' if epi == nv.EPI_SWIGLU else 'gelu'
    act = og.silu64 if kind == 'silu' else og.gelu64
    n_out = 256
    n, k = 2 * n_out, 2 * n_out
    eye = torch.eye(k, dtype=h16, device=dev)
    w = interleave_gate_up(eye[:n_out], eye[n_out:]).contiguous()     # gate j = e_j, up j = e_(n_out + j)
    u = up_values(n_out, dev)
    g = torch.Generator(device=dev).manual_seed(epi)
    # margin rows: gates where the activation is well conditioned
    shape = (300, n_out)
    mag = 0.5 + 7.5 * torch.rand(shape, generator=g, device=dev, dtype=torch.float64)
    small = 0.5 + 0.5 * torch.rand(shape, generator=g, device=dev, dtype=torch.float64)
    neg = torch.rand(shape, generator=g, device=dev) < 0.3
    gates = torch.where(neg, -(small if kind == 'gelu' else mag), mag).to(h16)   # GELU is flat below -1
    ref = act(gates.double()) * u
    bound = torch.from_numpy(og.activation_error_bound(gates.double().cpu().numpy(), h16, kind,
                                                       u.expand_as(ref).cpu().numpy())).to(dev)
    blocks = u.reshape(-1, 64)
    gap = (blocks[:, :, None] - blocks[:, None, :]).abs() + torch.eye(64, device=dev) * 1e9
    nearest = gap.min(dim=2).values.reshape(-1)                        # closest wrong up value in the W tile
    assert (act(gates.double()).abs() * nearest >= 4 * bound).all(), 'the up values do not separate the pairings'
    # sweep rows: every finite value of the build as a gate
    table = as_columns(og.value_table(h16), n_out).reshape(-1, n_out).to(dev)
    rows = [gates, table]
    if h16 == torch.float16:       # gate values whose product saturates
        rows.append(torch.full((2, n_out), 60000.0, device=dev).to(h16))
    gate_rows = torch.cat(rows)
    m = gate_rows.shape[0]
    a = torch.cat([gate_rows, u.to(h16).expand(m, n_out)], dim=1).contiguous()
    run = Run(dev, h16, a, w, None, None, m, n, k, epi)
    ref = act(gate_rows.double()) * u
    bound = torch.from_numpy(og.activation_error_bound(gate_rows.double().cpu().numpy(), h16, kind,
                                                       u.expand_as(ref).cpu().numpy())).to(dev)
    ok = ref.abs() < 3.3e38        # bfloat16: act(3e38) * up leaves fp32 (inf on both sides, not compared)
    run.assert_within(torch.where(ok, ref, 0.0), torch.where(ok, bound, float('inf')), kind)
    if h16 == torch.float16:
        sat = ref > 65520
        assert sat.any() and (run.out.float()[sat] == og.HALF_MAX).all()


# ------------------------------------------------------------------------------------------------ (g) NF4
@pytest.mark.parametrize('kb', [1, 4, 5, 9])
def test_nf4_against_host_dequantisation(dev, h16, kb):
    k, n, m = 64 * kb, 5120, 1100        # 40 x 9 tiles: two or three turns per CTA
    g = torch.Generator(device=dev).manual_seed(kb)
    codes = torch.randint(0, 256, (n, k // 2), generator=g, device=dev, dtype=torch.uint8)
    absmax = torch.rand((kb, n), generator=g, device=dev) * 2 - 0.5      # negative scales too
    absmax[torch.rand((kb, n), generator=g, device=dev) < 0.05] = 0.0
    absmax[0, :7] = torch.tensor([0.0, -1.0, 1.0, 3e4, -1e-3, 0.5, 1e5])  # f16 saturates 1e5 * code
    absmax = absmax.contiguous()
    assert set(codes.flatten().unique().tolist()) == set(range(256))       # every code in both nibbles
    w16 = og.to_storage(nf4.nf4_dequantize(codes, absmax), h16)
    a, idx = og.one_hot_rows(m, k, h16, dev)                               # out[m, n] = w16[n, sigma(m)]
    # ... as a sum: a -0 weight (code 0.0 times a negative scale, or a negative code times scale 0) plus the +0
    # products of the row's other weights is +0
    acc = w16.float()[:, idx].T + 0.0
    bias = scaled_bias(n, g)
    for b in (None, bias):
        run = Run(dev, h16, a, codes, b, None, m, n, k, nv.EPI_BIAS, absmax=absmax)
        run.assert_bits(og.epilogue(acc, b, None, h16), label=f'bias={b is not None}')


# ------------------------------------------------------------------------------------------------ (h) contract
def test_arguments_the_epilogue_does_not_read_are_rejected(dev, h16):
    m, n, k = 128, 256, 64
    a = torch.zeros((m, k), dtype=h16, device=dev)
    w = torch.zeros((n, k), dtype=h16, device=dev)
    codes = torch.zeros((n, k // 2), dtype=torch.uint8, device=dev)
    absmax = torch.zeros((1, n), device=dev)
    bias = torch.zeros(n, device=dev)
    resid = torch.zeros((m, n), dtype=h16, device=dev)
    for epi in GLU:
        with pytest.raises(nv.NativeError, match='no bias'):
            nv.gemm_h16(a, w, bias, None, epi)
        with pytest.raises(nv.NativeError, match='no bias'):
            nv.gemm_nf4(a, codes, absmax, bias, None, epi)
    for epi in (nv.EPI_BIAS, nv.EPI_BIAS_GELU, *GLU):
        with pytest.raises(nv.NativeError, match='reads no resid'):
            nv.gemm_h16(a, w, None, resid, epi)
        with pytest.raises(nv.NativeError, match='reads no resid'):
            nv.gemm_nf4(a, codes, absmax, None, resid, epi)
    torch.cuda.synchronize(dev)
