"""-m gpu: ESM C's fused q / k LayerNorm + rotary step (qk_layernorm_rope_kernel<960 | 1152>, csrc/mistral_ops.cuh) bit
for bit, and ESM C's rotary table against esm's formula through the encoder's own step.  The premises are checked on
the host by tests/test_esmc_exact_cpu.py.

(a) q and k rows +-2^6 times a Walsh pattern (oracle.rows.esmc_walsh_rows: mean 0, var + eps = 4^6) normalise to
    exactly +-1 times the gain.  The gains (oracle.rows.qk_gains) are signed powers of two 2^-3 .. 2^3 that differ
    between q and k, between the halves of a head and between heads, with a few zeros; every product with the table
    is exact in fp32, so each output is round16(fl32(y1 c - y2 s)) of the very table handed to the kernel, contracted
    or not.  Constant rows give exactly 0 (NaN without eps) and large-offset rows 2^12 + 2^6 p the same as Walsh
    rows; position-0 rows give round16(LN(x) g).  Padded positions t % S, packed positions tok_src % S with tok_src
    past S, rows from t_real on and every V column untouched byte for byte; T = 1, 1000 and 16 897, both widths, both
    builds.
(b) A 2-layer ESM C encoder with those gains as q_ln / k_ln runs its own rotary step (b2e_debug_rotary) on Walsh rows
    at S up to 2048, ragged, left-padded and holed masks, packed and padded layouts: within rotary_reference's
    allowance (8 fp32 ulps of the angle plus 8 of the result) of esm's fp32 table formula, which the zero-gain columns
    expose as round16(g c) and round16(g s) alone; position-0 rows bit for bit."""

from __future__ import annotations

import ctypes as C
import functools
import os

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from oracle import rows as R
from tools import oracle_esmc as O

pytestmark = pytest.mark.gpu

WIDTHS = (960, 1152)
EPS = (1e-12, 1e-5)
TABLE = 2048                           # ESM C's table length (max_pos)
CONSTS = (0.0, 1.0, -1024.0, 4096.0)   # fl(fl(H c) fl(1/H)) = c at both widths: x - mean = 0
OFFSET = 4096.0                        # 2^12 +- 2^6 is exact in both 16-bit types


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


def mismatch(got: np.ndarray, exp: np.ndarray, h: int, what) -> str | None:
    """None when got == exp element for element (+0 == -0, NaN never equal), else the first wrong element's row,
    side, head and element within the head."""
    bad = ~(got == exp)
    if not bad.any():
        return None
    r, c = (int(i) for i in np.argwhere(bad)[0])
    side = ('q', 'k', 'v')[c // h]
    return (f'{what}: {bad.sum()} of {bad.size} differ; first at row {r}, {side} head {(c % h) // 64}, element '
            f'{c % 64}: expected {exp[r, c]!r}, got {got[r, c]!r}')


# ---------------------------------------------------------------------------------- (a) qk_layernorm_rope_ exactly
def const_rows(t: int) -> tuple[np.ndarray, np.ndarray]:
    """The tokens whose q row (every 11th) or k row (every 13th, not also an 11th) is constant."""
    tt = np.arange(t)
    return tt % 11 == 3, (tt % 13 == 5) & (tt % 11 != 3)


@functools.lru_cache(maxsize=2)
def exact_rows(h: int, t: int) -> np.ndarray:
    """[t, 3h] float32 (every value exact): each token's q and k rows 2^6 * +-pattern (drawn independently); every
    11th token's q row a constant and its k row an offset row +-2^12 + 2^6 p, every 13th token the other way round;
    V small integers."""
    rows = R.esmc_walsh_rows(R.esmc_order(h) - 2, h)
    g = np.random.default_rng(h + t)
    qk = rows[g.integers(0, len(rows), (t, 2))]
    tt = np.arange(t)
    for j, sel in enumerate(const_rows(t)):
        qk[sel, j] = np.asarray(CONSTS)[tt[sel] % len(CONSTS)][:, None]
        qk[sel, 1 - j] += OFFSET * np.where(tt[sel] % 2 == 0, 1.0, -1.0)[:, None]
    return np.concatenate([qk[:, 0], qk[:, 1], g.integers(-128, 128, (t, h))], 1).astype(np.float32)


@functools.lru_cache(maxsize=4)
def normalised(h: int, t: int, eps: float) -> tuple[np.ndarray, np.ndarray]:
    """LN(x) * gain of the q and k rows, exactly, as float32 (oracle.rows.layernorm raises outside the exact
    domain)."""
    x = exact_rows(h, t)
    return tuple(R.layernorm(x[:, j * h:(j + 1) * h], R.qk_gains(h, j), 0.0, eps).astype(np.float32)
                 for j in (0, 1))


@pytest.mark.parametrize('t', [1, 1000, 16897])
@pytest.mark.parametrize('h', WIDTHS)
def test_qk_layernorm_rope_bit_exact(dev, h, t):
    x = exact_rows(h, t)
    qg, kg = (torch.from_numpy(R.qk_gains(h, j)).float().to(dev) for j in (0, 1))
    cos, sin = O.rotary_tables(TABLE)
    cn, sn = cos.numpy(), sin.numpy()
    cos_d, sin_d = cos.to(dev).contiguous(), sin.to(dev).contiguous()
    src = np.random.default_rng(t).integers(0, 4 * TABLE, t)
    src[:4] = (0, TABLE, TABLE - 1, 4 * TABLE - 1)[:t]            # tok_src past S: % S decides the position
    used = (2 * t) // 3                                            # 0 at T = 1: nothing may change
    t_real = torch.tensor([used, t], dtype=torch.int32, device=dev)
    tok_src = torch.from_numpy(src).to(dev, torch.int32)
    padded = np.arange(t) % TABLE                                  # 0, 1, 2047 and all between at T = 16 897
    layouts = {'padded': (None, None, padded, t), 'packed': (t_real, tok_src, src % TABLE, used),
               't_real': (t_real, None, padded, used)}
    const = const_rows(t)
    for eps in EPS:
        ys = normalised(h, t, eps)
        for name, (n_dev, src_dev, pos, live) in layouts.items():
            if eps != 1e-5 and name != 'padded':
                continue
            rot = [R.rope_exact(y[:live], cn, sn, pos[:live]) for y in ys]      # fp32, before the 16-bit rounding
            p0 = pos[:live] == 0
            for dtype in (torch.float16, torch.bfloat16):
                case = (h, t, str(dtype), eps, name)
                qkv = torch.from_numpy(x).to(dtype)
                assert torch.equal(qkv.float(), torch.from_numpy(x))
                got = nv.qk_layernorm_rope_(qkv.to(dev), qg, kg, cos_d, sin_d, eps, n_dev, src_dev).cpu()
                assert torch.equal(got[live:].view(torch.int16), qkv[live:].view(torch.int16)), (*case, 'rows past T')
                assert torch.equal(got[:, 2 * h:].view(torch.int16), qkv[:, 2 * h:].view(torch.int16)), (*case, 'V')
                g = got[:live, :2 * h].double().numpy()
                exp = np.concatenate([R.round16(r, dtype) for r in rot], 1)
                msg = mismatch(g, exp, h, case)
                assert msg is None, msg
                y0 = np.concatenate([y[:live][p0] for y in ys], 1)
                assert np.array_equal(g[p0], R.round16(y0, dtype)), (*case, 'position 0')
                for j in (0, 1):
                    assert (g[const[j][:live], j * h:(j + 1) * h] == 0).all(), (*case, 'constant rows')


# ---------------------------------------------------------------------------------- (b) the encoder's rotary step
ROT_S = 2048


def default_packing() -> bool:
    """The packing state of a process that never called b2e_debug_set_packing (B2E_PACKED=0 turns it off)."""
    return os.environ.get('B2E_PACKED', '1')[:1] != '0'


def set_packing(lib, on: bool) -> None:
    lib.b2e_debug_set_packing.argtypes = [C.c_int]
    nv.check(lib.b2e_debug_set_packing(int(on)), lib)


def rotary_masks() -> dict[str, torch.Tensor]:
    ragged = (torch.arange(ROT_S)[None] < torch.tensor([ROT_S, ROT_S - 1, 1025, 2, 1])[:, None]).long()
    short = (torch.arange(300)[None] < torch.tensor([300, 257, 1])[:, None]).long()
    left = torch.ones(3, ROT_S, dtype=torch.int64)
    left[1, :700] = 0
    left[2, :ROT_S - 1] = 0
    holes = torch.ones(3, ROT_S, dtype=torch.int64)
    holes[1, 100:300] = 0
    holes[2] = 0
    return {'ragged': ragged, 'ragged-300': short, 'left': left, 'holes': holes}


def layout_positions(mask: torch.Tensor, packed: bool) -> np.ndarray:
    """Position of each of the B*S qkv rows in the encoder's token layout, -1 past the last packed token: the layout
    packs only when every row is a non-empty prefix."""
    b, s = mask.shape
    lens = mask.sum(1).tolist()
    if packed and all(n > 0 and bool(mask[i, :n].all()) for i, n in enumerate(lens)):
        pos = np.full(b * s, -1)
        pos[:sum(lens)] = np.concatenate([np.arange(n) for n in lens])
        return pos
    return np.tile(np.arange(s), b)


def rotary_intervals(x: np.ndarray, pos: np.ndarray, gains: dict, h: int, dtype):
    """For one token layout (positions pos, -1 past the last packed token): per (layer, q or k) the interval
    [round16(ref - bound), round16(ref + bound)] of every live element, ref the rotation of LN(x) * gain (exactly
    +-gain, 0 on zero-gain columns) by esm's table and bound rotary_reference's allowance, and the exact position-0
    rows round16(LN(x) * gain)."""
    from distllm_b200.embed.encoders import weights as W

    live = pos >= 0
    c, sn, tau = (a[:, None] for a in R.rotary_table(pos[live]))
    p0 = pos[live] == 0
    out = {}
    for layer, pair in gains.items():
        for j, gain in enumerate(pair):
            y = R.layernorm(x[live, j * h:(j + 1) * h], gain, 0.0, W.ESMC_EPS)
            y4 = y.reshape(len(y), h // 64, 2, 32)
            y1, y2 = y4[:, :, 0], y4[:, :, 1]
            ref = np.stack([y1 * c - y2 * sn, y2 * c + y1 * sn], 2).reshape(len(y), h)
            bnd = (np.abs(y1) + np.abs(y2)) * (tau + 2.0 ** -23)
            bound = np.stack([bnd, bnd], 2).reshape(len(y), h)
            out[layer, j] = (R.round16(ref - bound, dtype), R.round16(ref + bound, dtype), R.round16(y[p0], dtype))
    return live, p0, out


@pytest.mark.parametrize('storage', ['bf16', 'f16'])
@pytest.mark.parametrize('h', WIDTHS)
def test_esmc_rotary_table_against_esm_formula(dev, h, storage):
    from distllm_b200.embed.encoders import weights as W
    from distllm_b200.embed.encoders.native import NativeEsmcEncoder

    sd = W.random_esmc_state_dict(h, 2, 256, seed=h)
    gains = {0: (R.qk_gains(h, 0), R.qk_gains(h, 1)), 1: (R.qk_gains(h, 1), R.qk_gains(h, 0))}   # swapped per layer
    for layer, (gq, gk) in gains.items():
        sd[f'transformer.blocks.{layer}.attn.q_ln.weight'] = torch.from_numpy(gq).float()
        sd[f'transformer.blocks.{layer}.attn.k_ln.weight'] = torch.from_numpy(gk).float()
    enc = NativeEsmcEncoder(W.esmc_config(sd), sd, device=dev, storage=storage)
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    rows = R.esmc_walsh_rows(R.esmc_order(h) - 2, h)
    try:
        for mname, mask in rotary_masks().items():
            b, s = mask.shape
            t = b * s
            g = np.random.default_rng(s + b)
            x = np.concatenate([rows[g.integers(0, len(rows), t)], rows[g.integers(0, len(rows), t)],
                                g.integers(-128, 128, (t, h)).astype(np.float64)], 1)
            before = torch.from_numpy(x).to(dtype)
            expected = {}       # left-padded and holed masks keep the padded layout: one expectation for both
            for packed in (True, False):
                pos = layout_positions(mask, packed)
                if pos.tobytes() not in expected:
                    expected[pos.tobytes()] = rotary_intervals(x, pos, gains, h, dtype)
                live, p0, want = expected[pos.tobytes()]
                for layer in (0, 1):
                    case = (h, storage, mname, f'packed={packed}', f'layer={layer}')
                    set_packing(enc._lib, packed)
                    got = nv.debug_rotary_(enc, layer, before.to(dev).contiguous(), mask.to(dev)).cpu()
                    assert torch.equal(got[:, 2 * h:].view(torch.int16), before[:, 2 * h:].view(torch.int16)), \
                        (*case, 'V changed')
                    assert torch.equal(got[~torch.from_numpy(live)].view(torch.int16),
                                       before[~torch.from_numpy(live)].view(torch.int16)), (*case, 'rows past T')
                    for j in (0, 1):
                        lo, hi, exact0 = want[layer, j]
                        gj = got[live, j * h:(j + 1) * h].double().numpy()
                        bad = ~((gj >= lo) & (gj <= hi))
                        if bad.any():
                            r, col = (int(k) for k in np.argwhere(bad)[0])
                            pytest.fail(f'{case} {"qk"[j]}: {bad.sum()} of {bad.size} outside; first at live row {r}, '
                                        f'head {col // 64}, element {col % 64}: got {gj[r, col]!r}, allowed '
                                        f'[{lo[r, col]!r}, {hi[r, col]!r}]')
                        assert np.array_equal(gj[p0], exact0), (*case, ('q', 'k')[j], 'position 0')
    finally:
        set_packing(enc._lib, default_packing())
        enc.close()
