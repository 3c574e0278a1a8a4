"""-m gpu: the row kernels (csrc/rowops.cuh, csrc/mistral_ops.cuh) and the pooled output tail, bit for bit, on inputs
whose every intermediate value is exact (oracle/rows.py; its premises are checked on the host by
tests/test_rows_oracle_cpu.py).

(a) The rsqrt premise: +-2^a Walsh rows with gamma 1, beta 0 normalise to exactly +-1.  Every other test here rests
    on it.
(b) b2e_layernorm on Walsh, constant and large-offset rows; b2e_pool_mean with exact sums and with sums a 16-bit input
    type cannot hold; b2e_l2_normalize on rows that separate x / ||x|| from x * (1 / ||x||); b2e_adjacent_cosine_dist
    on integer rows against oracle/semantic.py.
(c) Row-path encoders: every family at every width it is built for, in both builds, with every weight matrix zero, so
    that the forward pass is a composition of row kernels (oracle.rows.row_path_model).  b2e_encode (fp32 and
    storage-type outputs) and b2e_encode_pooled (three pool kinds, l2 off and on, packed and padded token layouts)
    over ragged, full, left-padded and holed masks, an empty row and S = 1, at S = 64, 65, 129 and 1100 (1, 2, 3 and
    16 pool splits).
(d) Rotary: b2e_debug_rotary runs an encoder's own rotary step on one-hot and random q / k heads, against HF's fp32
    table formula of each family within a stated bound (rotary_reference)."""

from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from oracle import rows as R
from oracle import semantic as osem

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(params=[torch.float16, torch.bfloat16], ids=['f16', 'bf16'])
def h16(request):
    return request.param


def first_mismatch(got: np.ndarray, exp: np.ndarray, where) -> str | None:
    """None when got == exp element for element (+0 == -0), else a description of the first wrong element: its
    index as named by ``where(index)``, its column's pass and lane in the row kernels, and both values' bits."""
    got, exp = np.asarray(got, np.float32), np.asarray(exp, np.float32)
    bad = ~(got == exp)
    if not bad.any():
        return None
    idx = tuple(int(i) for i in np.argwhere(bad)[0])
    c = idx[-1]
    g, e = got[idx], exp[idx]
    return (f'{bad.sum()} of {bad.size} differ; first at {where(idx)}, column {c} (pass {c // 256}, lane '
            f'{(c % 256) // 8}): expected {e!r} (0x{np.float32(e).view(np.uint32):08x}), '
            f'got {g!r} (0x{np.float32(g).view(np.uint32):08x})')


# ---------------------------------------------------------------------------------- (a) the rsqrt premise
@pytest.mark.parametrize('h', R.WIDTHS)
def test_rsqrt_premise_walsh_rows_normalise_to_signs(dev, h, h16):
    """rsqrtf(4^a) = 2^-a on the device: +-2^a rows (a = 4 .. 9) with gamma 1 and beta 0 give exactly +-1."""
    n, _ = R.split_width(h)
    for a in range(4, 10):
        x = R.walsh_rows(n - 2, h, a)
        for eps in (1e-12, 1e-5):
            if a == 4 and eps == 1e-5:
                continue      # 256 + 1e-5 does not round to 256 at every width (host test)
            got = nv.layernorm(torch.from_numpy(x).to(dev, h16), torch.ones(h, device=dev),
                               torch.zeros(h, device=dev), eps, torch.float32).cpu().numpy()
            msg = first_mismatch(got, x / 2.0 ** a, lambda i: f'row {i[0]}')
            assert msg is None, (a, eps, msg)


# ---------------------------------------------------------------------------------- (b) standalone entry points
def layernorm_rows(h: int, dtype: torch.dtype) -> np.ndarray:
    """Walsh rows, constant rows and large-offset rows m + 32 p, m as large as the 16-bit type holds m +- 32 (in half,
    a one-pass variance loses them from H = 1024 on; tests/test_rows_oracle_cpu.py)."""
    n, _ = R.split_width(h)
    walsh = R.walsh_rows(n - 2, h)
    const = np.array([[c] * h for c in (0.0, 1.0, -3.0, 1024.0, -2.0 ** 14)])
    offset = (2.0 ** 15 if dtype == torch.float16 else 2.0 ** 12) + R.walsh_rows(n - 2, h)
    return np.concatenate([walsh, const, offset, -offset])


@pytest.mark.parametrize('h', R.WIDTHS)
def test_layernorm_exact(dev, h, h16):
    """Walsh rows, constant rows (beta exactly: a dropped eps gives NaN) and large-offset rows, with a Walsh gain and
    bias, into fp32 and into the storage type."""
    x = layernorm_rows(h, h16)
    n, _ = R.split_width(h)
    gamma = R.walsh_gain(h, 3, -1.0)
    beta = 4.0 * R.pattern(h, n // 2 - 1) + 2.0
    xd = torch.from_numpy(x).to(dev, h16)
    g, b = torch.from_numpy(gamma).float().to(dev), torch.from_numpy(beta).float().to(dev)
    for eps in (1e-12, 1e-6, 1e-5):
        exp = R.layernorm(x, gamma, beta, eps)
        got = nv.layernorm(xd, g, b, eps, torch.float32).cpu().numpy()
        assert (msg := first_mismatch(got, exp, lambda i: f'row {i[0]}')) is None, (eps, 'fp32', msg)
        got = nv.layernorm(xd, g, b, eps).float().cpu().numpy()
        assert (msg := first_mismatch(got, R.round16(exp, h16), lambda i: f'row {i[0]}')) is None, (eps, h16, msg)


# ---------------------------------------------------------------------------------- rotary (b2e_debug_rotary)
# name: (family, hidden, heads, kv_heads or None, head_dim)
ROTARY = {'esm-d64': ('esm', 256, 4, None, 64), 'esm-d32': ('esm', 256, 8, None, 32),
          'modernbert': ('modernbert', 256, 4, None, 64), 'mistral-gqa4': ('mistral', 512, 4, 1, 128),
          'qwen3-gqa2': ('qwen3', 512, 4, 2, 128)}
ROT_S = 300


def rotary_encoder(name: str, storage: str, dev):
    """A 2-layer encoder whose rotary step is under test (its weight matrices play no part), and per layer the rotary
    base HF uses for it: ModernBERT layer 0 attends globally (global_rope_theta), layer 1 in a window (local)."""
    from distllm_b200.embed.encoders import native as N
    from distllm_b200.embed.encoders import weights as W

    fam, h, heads, kv, d = ROTARY[name]
    common = dict(hidden_size=h, num_hidden_layers=2, num_attention_heads=heads, intermediate_size=256)
    if fam == 'esm':
        from transformers import EsmConfig
        cfg = EsmConfig(vocab_size=33, max_position_embeddings=1026, position_embedding_type='rotary',
                        token_dropout=False, mask_token_id=32, pad_token_id=1, layer_norm_eps=1e-5,
                        emb_layer_norm_before=False, **common)
        cls, sd, thetas = N.NativeEsm2Encoder, W.random_esm_state_dict(cfg), (10000.0, 10000.0)
    elif fam == 'modernbert':
        from transformers import ModernBertConfig
        cfg = ModernBertConfig(vocab_size=50, max_position_embeddings=512, local_attention=128, pad_token_id=0,
                               bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2, **common)
        desc = W.modernbert_desc(cfg)
        cls, sd, thetas = N.NativeModernBertEncoder, W.random_modernbert_state_dict(cfg), (desc.rope_theta,
                                                                                        desc.rope_theta_local)
        assert thetas[0] != thetas[1]
    elif fam == 'mistral':
        from transformers import MistralConfig
        cfg = MistralConfig(vocab_size=50, num_key_value_heads=kv, head_dim=128, max_position_embeddings=512,
                            sliding_window=None, **common)
        cls, sd = N.NativeMistralEncoder, W.random_mistral_state_dict(cfg)
        thetas = (W.rope_theta_of(cfg),) * 2
    else:
        from transformers import Qwen3Config
        cfg = Qwen3Config(vocab_size=50, num_key_value_heads=kv, head_dim=128, max_position_embeddings=512,
                          rms_norm_eps=1e-6, rope_parameters={'rope_type': 'default', 'rope_theta': 1e6}, **common)
        cls, sd = N.NativeQwen3Encoder, W.random_qwen3_state_dict(cfg)
        thetas = (1e6, 1e6)
    return cls(cfg, sd, device=dev, storage=storage), cfg, sd, thetas


def layout_positions(mask: torch.Tensor, packed: bool) -> np.ndarray:
    """Position of each of the B*S qkv rows in the encoder's token layout; -1 for rows the step must not touch (past
    the last attended token of the packed layout)."""
    b, s = mask.shape
    lens = mask.sum(1).tolist()
    if packed and all(n > 0 and bool(mask[i, :n].all()) for i, n in enumerate(lens)):
        pos = np.full(b * s, -1)
        t = 0
        for n in lens:
            pos[t:t + n] = np.arange(n)
            t += n
        return pos
    return np.tile(np.arange(s), b)


def rotary_reference(x: np.ndarray, pos: np.ndarray, theta: float, d: int, gamma=None, eps=0.0):
    """HF's rotation of q / k heads x [T, heads, d] (float64 of the 16-bit inputs) at positions pos, with HF's fp32
    table: inv_freq = 1 / theta^(arange(0, d, 2) / d), angle = fl32(p * inv_freq), then cos / sin exactly; gamma:
    Qwen3's per-head RMSNorm first.  Returns (reference, bound): the device's fp32 table and arithmetic stay within
    bound of the reference before the one 16-bit rounding.

    The bound: the CUDA math library's maximum ulp errors for powf and sincosf are stated in the CUDA C++
    Programming Guide, which is not available offline here, so they are not quoted.  Instead the table's deviation
    from HF's formula is allowed 8 fp32 ulps of the angle (inv_freq through powf and a division on either side, one
    product each) plus 8 of the result (sincosf, torch's cos); the rotation adds one rounding per product and one per
    sum (2^-23 of |x1| + |x2|), Qwen3's norm 2^-20 relative (rsqrtf, three products)."""
    half = d // 2
    c, s, tau = (a[:, None, :] for a in R.rotary_table(pos, theta, d))
    rel = 2.0 ** -23
    if gamma is not None:
        r = 1.0 / np.sqrt((x * x).mean(-1, keepdims=True) + np.float32(eps))
        x = x * r * gamma
        rel = 2.0 ** -20
    x1, x2 = x[..., :half], x[..., half:]
    ref = np.concatenate([x1 * c - x2 * s, x2 * c + x1 * s], -1)
    b = (np.abs(x1) + np.abs(x2)) * (tau + rel)
    return ref, np.concatenate([b, b], -1)


def rotary_check(got: np.ndarray, ref: np.ndarray, bound: np.ndarray, dtype) -> str | None:
    """got = round16(v) for some v within bound of ref: got in [round16(ref - bound), round16(ref + bound)]
    (rounding is monotonic), so one 16-bit ulp away from round16(ref) only where the bound straddles a rounding
    boundary."""
    msg = R.interval_check(got, ref, bound, dtype)
    return None if msg is None else msg + ' (index: row, head, element)'


def rotary_masks():
    ragged = (torch.arange(ROT_S)[None] < torch.tensor([ROT_S, 257, 2, 1])[:, None]).long()
    left = torch.ones(3, ROT_S, dtype=torch.int64)
    left[1, :100] = 0
    return {'ragged': ragged, 'left': left}


def run_rotary(enc, layer, qkv, mask, packed):
    lib = enc._lib
    set_packing(lib, packed)
    try:
        return nv.debug_rotary_(enc, layer, qkv, mask.to(qkv.device))
    finally:
        set_packing(lib, default_packing())


@pytest.mark.parametrize('storage', ['bf16', 'f16'])
@pytest.mark.parametrize('name', list(ROTARY))
def test_rotary_exact(dev, name, storage):
    """One-hot q and k heads (x = e_j, j varying over heads and rows, both halves) give round16(HF cos) and
    +-round16(HF sin) at the two rotated elements and 0 elsewhere; random heads stay within the bound; position-0 rows
    come back unchanged bit for bit (not Qwen3: its heads are normalised), v heads and rows past the last packed
    token too.  Every layer (ModernBERT: its full and its sliding table), packed and padded layouts, ragged and
    left-padded masks, every row of every sequence (positions 0, 1, S-1, first and last row of each packed
    sequence)."""
    enc, cfg, sd, thetas = rotary_encoder(name, storage, dev)
    fam, h, heads, kv, d = ROTARY[name]
    kv = kv or heads
    n_rot, n_v = heads + kv, kv
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    g = torch.Generator().manual_seed(len(name))
    try:
        for mname, mask in rotary_masks().items():
            b, s = mask.shape
            t = b * s
            for packed in (True, False):
                pos = layout_positions(mask, packed)
                live = pos >= 0
                for layer in (0, 1):
                    gamma = None
                    if fam == 'qwen3':
                        gq = sd[f'layers.{layer}.self_attn.q_norm.weight'].double().numpy()
                        gk = sd[f'layers.{layer}.self_attn.k_norm.weight'].double().numpy()
                        gamma = np.stack([gq] * heads + [gk] * kv)[None]
                    case = (name, storage, mname, f'packed={packed}', f'layer={layer}')
                    for kind in ('onehot', 'random'):
                        x = torch.randn(t, n_rot + n_v, d, generator=g).to(dtype)
                        if kind == 'onehot':
                            j = (np.arange(t)[:, None] * 5 + np.arange(n_rot)[None] * 11) % d
                            oh = np.zeros((t, n_rot, d))
                            np.put_along_axis(oh, j[..., None], 1.0, -1)
                            x[:, :n_rot] = torch.from_numpy(oh).to(dtype)
                        before = x.clone()
                        got = run_rotary(enc, layer, x.reshape(t, -1).contiguous().to(dev), mask, packed)
                        got = got.reshape(t, n_rot + n_v, d).cpu()
                        assert torch.equal(got[:, n_rot:], before[:, n_rot:]), (*case, kind, 'v heads changed')
                        assert torch.equal(got[~torch.from_numpy(live)], before[~torch.from_numpy(live)]), \
                            (*case, kind, 'rows past the last token changed')
                        if fam != 'qwen3':
                            p0 = torch.from_numpy(pos == 0)
                            assert torch.equal(got[p0], before[p0]), (*case, kind, 'position-0 rows changed')
                        xq = before[live, :n_rot].double().numpy()
                        ref, bound = rotary_reference(xq, pos[live], thetas[layer], d, gamma, cfg.rms_norm_eps
                                                      if fam == 'qwen3' else 0.0)
                        gq = got[live, :n_rot].double().numpy()
                        msg = rotary_check(gq, ref, bound, dtype)
                        assert msg is None, (*case, kind, msg)
                        if kind == 'onehot' and fam != 'qwen3':
                            # every element but the two rotated ones is exactly 0 (+-0)
                            assert ((gq == 0) | (np.abs(ref) > 0)).all(), (*case, 'non-zero off the rotated pair')
    finally:
        enc.close()


def ragged_mask(s: int) -> torch.Tensor:
    lens = [s, max(s - 1, 0), s // 2 + 1, 2, 1, 0]
    return (torch.arange(s)[None] < torch.tensor([min(n, s) for n in lens])[:, None]).long()


@pytest.mark.parametrize('s', [1, 64, 65, 129, 1100])
@pytest.mark.parametrize('h', R.WIDTHS)
def test_pool_mean_exact(dev, h, s):
    """Integer hidden states in fp32, bf16 and f16 (exact in each), both pool kinds, the reference's mask mutation on
    and off.  With |x| <= 15 the numerators reach beyond 2^8 and 2^11: the 16-bit paths round them to the input type
    nearest-even before the division, as torch sums in the embedding dtype."""
    g = torch.Generator().manual_seed(h * 3 + s)
    mask = ragged_mask(s)
    x = torch.randint(-15, 16, (mask.shape[0], s, h), generator=g).double()
    x[0] = x[0].abs()            # one row of large same-signed sums
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        for kind, code, mutate in (('ref', nv.POOL_MEAN_REF, True), ('ref', nv.POOL_MEAN_REF, False),
                                   ('per_row', nv.POOL_MEAN_PER_ROW, False)):
            w = R.pool_weights(mask, kind)
            num = np.einsum('bs,bsh->bh', w, x.numpy())
            if dtype != torch.float32:
                num = R.round16(num, dtype)
            count = np.maximum(w.sum(1).astype(np.float32), R.POOL_EPS)
            exp = num.astype(np.float32) / count[:, None]
            m = mask.to(dev)
            got = nv.pool_mean(x.to(dev, dtype), m, code, mutate).cpu().numpy()
            msg = first_mismatch(got, exp, lambda i: f'sequence {i[0]}')
            assert msg is None, (dtype, kind, mutate, msg)
            assert torch.equal(m.cpu(), torch.from_numpy(w).long() if mutate else mask), (dtype, kind, mutate)


@pytest.mark.parametrize('h', R.WIDTHS + (4, 132))
def test_l2_normalize_divides(dev, h):
    """x / max(||x||, 1e-12) bit for bit, as F.normalize computes it, on integer rows whose sum of squares fp32 holds
    exactly; the rows include elements where x * (1 / ||x||) differs (checked on the host)."""
    x = R.l2_test_rows(h)
    exp = R.l2_exact(x)
    got = nv.l2_normalize_(torch.from_numpy(x).to(dev)).cpu().numpy()
    assert (msg := first_mismatch(got, exp, lambda i: f'row {i[0]}')) is None, msg


@pytest.mark.parametrize('h', [256, 384, 768, 4096])
def test_adjacent_cosine_exact(dev, h):
    """1 - dot / (sqrt(na) sqrt(nb)) on integer rows, bit for bit against oracle/semantic.py's fp32 arithmetic, for
    every input type; a document boundary gives NaN."""
    g = np.random.default_rng(h + 1)
    x = g.integers(-15, 16, (41, h)).astype(np.float32)
    x[7] = x[6]                      # distance 0
    x[9] = -x[8]                     # distance 2
    doc = torch.zeros(41, dtype=torch.int32)
    doc[20:] = 1
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        exp = osem.calculate_distances_between_buffer(x).astype(np.float32)
        got = nv.adjacent_cosine_dist(torch.from_numpy(x).to(dev, dtype)).cpu().numpy()
        assert (msg := first_mismatch(got, exp, lambda i: f'pair {i[0]}')) is None, (dtype, msg)
        got = nv.adjacent_cosine_dist(torch.from_numpy(x).to(dev, dtype), doc.to(dev)).cpu().numpy()
        assert np.isnan(got[19]) and (np.delete(got, 19) == np.delete(exp, 19)).all(), dtype


# ---------------------------------------------------------------------------------- (c) row-path encoders
def masks(s: int) -> dict[str, torch.Tensor]:
    """The encoders' masks: right-padded ragged rows, all rows full, left padding, and a hole, a one-token row and an
    empty row (the layout falls back to the padded one; the empty row's length 0 kills column S-1 for the
    reference's mean pooler and makes the last-token pooler take S-1)."""
    if s == 1:
        return {'S1': torch.ones(3, 1, dtype=torch.int64)}
    out = {'ragged': ragged_mask(s)[:5]}                      # rows of lengths S, S-1, S/2+1, 2, 1
    if s > 2:
        full = torch.ones(4, s, dtype=torch.int64)             # every row full: the last-token pooler takes S-1
        left = torch.ones(4, s, dtype=torch.int64)
        left[1, : s // 2] = 0                                  # left padding
        left[2, : s - 1] = 0
        holes = torch.ones(6, s, dtype=torch.int64)
        holes[5] = 0                                           # an empty row
        holes[1, 1: s // 3] = 0                                # a hole
        holes[2, 1:] = 0                                       # the first token only
        holes[3, s - 2:] = 0
        out.update(full=full, left=left, holes=holes)
    return out


# full mask set and S values at the widths with a half pass, at the BERT-base width and for ESM C (whose widths both end
# on a partial pass), S = 129 elsewhere
FULL_WIDTHS = (384, 640, 768)
SEQS = (1, 64, 65, 129, 1100)


def encoder_cases():
    out = []
    for fam, widths in R.FAMILY_WIDTHS.items():
        for h in widths:
            for live in (('word', 'pos', 'type') if fam == 'bert' else ('word',)):
                for storage in ('bf16', 'f16'):
                    out.append(pytest.param(fam, h, live, storage, id=f'{fam}-{h}-{live}-{storage}'))
    return out


def make_inputs(fam: str, live: str, mask: torch.Tensor, seed: int):
    g = torch.Generator().manual_seed(seed)
    b, s = mask.shape
    ids = torch.randint(0, R.VOCAB, (b, s), generator=g)
    ids[:, ::7] = R.VOCAB - 1      # the decoders' zero embedding row: RMSNorm of a zero row is 0 (eps keeps it finite)
    types = None
    if fam == 'bert':
        types = torch.randint(0, 2, (b, s), generator=g) if live == 'type' else torch.zeros(b, s, dtype=torch.int64)
    return ids, types


def default_packing() -> bool:
    """The packing state of a process that never called b2e_debug_set_packing (B2E_PACKED=0 turns it off)."""
    return os.environ.get('B2E_PACKED', '1')[:1] != '0'


def set_packing(lib, on: bool) -> None:
    lib.b2e_debug_set_packing.argtypes = [C.c_int]
    nv.check(lib.b2e_debug_set_packing(int(on)), lib)


@pytest.mark.parametrize('fam,h,live,storage', encoder_cases())
def test_row_path_encoder_exact(dev, fam, h, live, storage):
    from distllm_b200.embed.encoders import native as N

    cls = {'bert': N.NativeBertEncoder, 'esm': N.NativeEsm2Encoder, 'modernbert': N.NativeModernBertEncoder,
           'mistral': N.NativeMistralEncoder, 'qwen3': N.NativeQwen3Encoder, 'esmc': N.NativeEsmcEncoder}[fam]
    cfg, sd, reference = R.row_path_model(fam, h, live)
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    enc = cls(cfg, sd, device=dev, storage=storage)
    full = h in FULL_WIDTHS or fam == 'esmc'
    seqs = SEQS if full else (65, 129)
    try:
        for s in seqs:
            for mname, mask in masks(s).items():
                if not full and s == 65 and mname != 'holes':
                    continue
                ids, types = make_inputs(fam, live, mask, seed=h + s)
                y = reference(ids, mask, types, dtype)
                lens = mask.sum(1).tolist()
                prefix = all(mask[i, :n].all() and n > 0 for i, n in enumerate(lens))
                cu = np.concatenate([[0], np.cumsum(lens)])

                def at(i, packed):
                    row = f' (packed row {cu[i[0]] + i[1]})' if packed and prefix and len(i) == 3 else ''
                    return f'(b, s) = {i[:2]}{row}' if len(i) == 3 else f'sequence {i[0]}'

                case = (fam, h, live, storage, f'S={s}', mname)
                for out_dtype in (torch.float32, dtype):
                    got = enc.encode(ids, mask, types, out_dtype).float().cpu().numpy()
                    exp = y if out_dtype == torch.float32 else R.round16(y, dtype)
                    msg = first_mismatch(got, exp, lambda i: at(i, False))
                    assert msg is None, (*case, 'encode', out_dtype, msg)
                refs = {}
                for kind, code in (('ref', nv.POOL_MEAN_REF), ('per_row', nv.POOL_MEAN_PER_ROW)):
                    v = R.mean_pool(y, R.pool_weights(mask, kind))
                    refs[code] = (v, R.finalize_l2(v))
                v = R.last_token(y, mask)
                refs[nv.POOL_LAST_TOKEN] = (v, R.l2_exact(v))
                for packed in (True, False):
                    set_packing(enc._lib, packed)
                    for code, pair in refs.items():
                        for l2 in (False, True):
                            got = enc.encode_pooled(ids, mask, types, code, l2).cpu().numpy()
                            msg = first_mismatch(got, pair[l2], lambda i: at(i, packed))
                            assert msg is None, (*case, 'pooled', code, f'l2={l2}', f'packed={packed}', msg)
    finally:
        set_packing(enc._lib, default_packing())
        enc.close()
