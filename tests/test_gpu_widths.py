"""-m gpu: every hidden width the row kernels are built for (DISPATCH_H in csrc/b2e_api.cu), in every family that
accepts it, against float64 / fp32 references.

The row kernels keep NV = H / 256 passes of 8 floats per lane in registers and size their shared buffers by H, so each
width is its own code.  Kernel by kernel (LayerNorm, both mean poolers, last-token pooling) at all ten widths in both
builds; the GEMM at each width's four projection shapes with a NaN-filled output; head_dim-64 attention at 16 to 64
heads; then a 2-layer model of every (family, width) pair b2e_check_model accepts against the CPU oracle, at full
depth, after one layer, and packed against padded.  tests/test_widths_cpu.py checks the acceptance matrix itself."""

from __future__ import annotations

import ctypes as C
import json

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from oracle import pooling as opool
from tools.workloads import add_outliers

from conftest import cosine_rows

pytestmark = pytest.mark.gpu

WIDTHS = (256, 384, 512, 640, 768, 1024, 1280, 2048, 2560, 4096)


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(params=[torch.float16, torch.bfloat16], ids=['f16', 'bf16'])
def h16(request):
    """The 16-bit storage type = which build of the library the call lands in."""
    return request.param


# ---------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize('eps', [1e-12, 1e-5])
@pytest.mark.parametrize('h', WIDTHS)
def test_layernorm_every_width(dev, h, eps, h16):
    """1003 rows (the last block of 8 warps is not full); every other row sits on a common offset of 1e3 with std 1,
    where a one-pass E[x^2] - E[x]^2 variance in fp32 loses the whole statistic."""
    g = torch.Generator(device=dev).manual_seed(h + int(eps < 1e-6))
    x = torch.randn(1003, h, device=dev, generator=g) * 3 + 1
    x[1::2] = torch.randn(501, h, device=dev, generator=g) + 1e3
    x = x.to(h16)
    gamma = torch.rand(h, device=dev, generator=g) + 0.5
    beta = torch.randn(h, device=dev, generator=g)
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    var = (xd - mean).pow(2).mean(-1, keepdim=True)
    ref = (xd - mean) / torch.sqrt(var + eps) * gamma.double() + beta.double()
    got = nv.layernorm(x, gamma, beta, eps, torch.float32).double()
    torch.testing.assert_close(got[0::2], ref[0::2], rtol=1e-4, atol=1e-4)
    # the offset rows: the two-pass statistics keep them to ~1e-4; in fp32, E[x^2] ~ 1e6 alone is rounded to 0.0625
    torch.testing.assert_close(got[1::2], ref[1::2], rtol=1e-4, atol=1e-3)
    t = 2 ** -10 if h16 == torch.float16 else 2 ** -7
    torch.testing.assert_close(nv.layernorm(x, gamma, beta, eps).double(), ref, rtol=t, atol=t)


# ---------------------------------------------------------------------------------- mean pooling
def ragged_lens(s: int) -> list[int]:
    """Seven rows: full, one short of full, half, and the 0 / 1 / 2-token rows both poolers zero out."""
    return [min(n, s) for n in (s, max(s - 1, 0), s // 2, 0, 1, 2, 2)]


def round_through(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    return x.to(dtype).double() if dtype != torch.float32 else x


@pytest.mark.parametrize('s', [1, 63, 64, 65, 1100])
@pytest.mark.parametrize('h', WIDTHS)
def test_pool_mean_every_width(dev, h, s):
    """Both pool kinds for float32, bfloat16 and float16 hidden states: S from one split (pool_nsplit 1) to the cap of
    16; the reference's cross-row quirk (mean.py:36) edits the mask exactly as oracle.pooling.average_pool does.  The
    reference is the oracle in float64; for 16-bit inputs its sum is rounded to the input type, as torch sums
    `embeddings * mask` in the embedding dtype in the reference."""
    g = torch.Generator().manual_seed(h * 7 + s)
    lens = ragged_lens(s)
    mask = (torch.arange(s)[None] < torch.tensor(lens)[:, None]).long()
    base = torch.randn(len(lens), s, h, generator=g)
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        emb = base.to(dtype)
        m_ref = mask.clone()
        ref = opool.average_pool(emb.double(), m_ref)
        count = m_ref.sum(1, keepdim=True).double().clamp(min=1e-9)
        ref = round_through(ref * count, dtype) / count
        m = mask.to(dev)
        got = nv.pool_mean(emb.to(dev), m).double().cpu()
        rt = 1e-5 if dtype == torch.float32 else (2 ** -10 if dtype == torch.float16 else 2 ** -7)
        torch.testing.assert_close(got, ref, rtol=rt, atol=1e-6, msg=lambda e: f'{dtype} REF: {e}')
        assert torch.equal(m.cpu(), m_ref), dtype
        # per row: mean over positions 1 .. len-2 of the row itself; the mask is left alone
        w2 = mask.double()
        w2[:, 0] = 0
        for i, n in enumerate(lens):
            w2[i, n - 1 if n > 0 else s - 1] = 0
        ref2 = round_through((emb.double() * w2[..., None]).sum(1), dtype) / w2.sum(1, keepdim=True).clamp(min=1e-9)
        m2 = mask.to(dev)
        got2 = nv.pool_mean(emb.to(dev), m2, nv.POOL_MEAN_PER_ROW, mutate_mask=False).double().cpu()
        torch.testing.assert_close(got2, ref2, rtol=rt, atol=1e-6, msg=lambda e: f'{dtype} PER_ROW: {e}')
        assert torch.equal(m2.cpu(), mask), dtype
        assert not got2[torch.tensor(lens) <= 2].any()


@pytest.mark.parametrize('h', WIDTHS)
def test_pool_last_token_every_width(dev, h):
    """Bit-exact against oracle.pooling.last_token_pool, right padding (each row's own last token) and left padding
    (column S-1 for every row), for every input type."""
    g = torch.Generator().manual_seed(h + 3)
    s = 70
    base = torch.randn(5, s, h, generator=g)
    right = (torch.arange(s)[None] < torch.tensor([70, 1, 2, 69, 33])[:, None]).long()
    left = (torch.arange(s)[None] >= torch.tensor([0, 69, 68, 1, 37])[:, None]).long()
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        emb = base.to(dtype)
        for mask in (right, left):
            got = nv.pool_last_token(emb.to(dev), mask.to(dev)).cpu()
            assert torch.equal(got, opool.last_token_pool(emb, mask.clone()).float()), (dtype, mask[:, -1])


# ---------------------------------------------------------------------------------- GEMM
def intermediate_of(h: int) -> int:
    """The FFN width of the real model at this hidden size where one exists (bge-large / e5-large: 4096,
    esm2_t36_3B: 10240, ESM-2 650M: 5120), else 4H."""
    return {1024: 4096, 1280: 5120, 2560: 10240}.get(h, 4 * h)


PROJECTIONS = ('qkv', 'out', 'ffn_up', 'ffn_down')


@pytest.mark.parametrize('proj', PROJECTIONS)
@pytest.mark.parametrize('h', WIDTHS)
def test_gemm_projection_shapes(dev, h, proj, h16):
    """The four linear layers of a BERT / ESM-2 block at width H with their epilogues: QKV 3H x H (bias), attention
    out H x H (bias + residual), FFN up I x H (bias + GELU), FFN down H x I (bias + residual), for M = 1, 1000 and
    16 897 rows (one partial tile; 132 SMs walking several tiles each).  The output is NaN before the call, so a tile
    the persistent scheduler never writes fails; the reference is float64 from the same 16-bit operands."""
    i = intermediate_of(h)
    n, k, epi = {'qkv': (3 * h, h, nv.EPI_BIAS), 'out': (h, h, nv.EPI_BIAS_RESID),
                 'ffn_up': (i, h, nv.EPI_BIAS_GELU), 'ffn_down': (h, i, nv.EPI_BIAS_RESID)}[proj]
    lib = nv.load(nv.storage_of(h16))
    g = torch.Generator(device=dev).manual_seed(h + n + k)
    w = (torch.randn(n, k, device=dev, generator=g) / k ** 0.5).to(h16)
    bias = torch.randn(n, device=dev, generator=g) * 0.1
    tol = 2e-3 if h16 == torch.float16 else 1.2e-2
    for m in (1, 1000, 16897):
        a = torch.randn(m, k, device=dev, generator=g).to(h16)
        resid = torch.randn(m, n, device=dev, generator=g).to(h16) if epi == nv.EPI_BIAS_RESID else None
        out = torch.full((m, n), float('nan'), device=dev, dtype=h16)
        nv.check(lib.b2e_gemm_h16(a.data_ptr(), w.data_ptr(), bias.data_ptr(), nv._ptr(resid), out.data_ptr(),
                                  m, n, k, epi, nv.stream_ptr(dev)), lib)
        pre = a.double() @ w.double().T + bias.double()
        ref = pre
        bound = tol * (1 + pre.abs())
        if epi == nv.EPI_BIAS_GELU:
            ref = torch.nn.functional.gelu(pre)
            bound = tol * (1 + ref.abs()) + 4e-4 * pre.abs()     # the epilogue's erf approximation: <= 3e-4 |x|
        if resid is not None:
            ref = ref + resid.double()
            bound = tol * (1 + ref.abs())
        got = out.double()
        assert torch.isfinite(got).all(), (m, n, k, 'tiles left unwritten', (~torch.isfinite(got)).nonzero()[:4])
        err = (got - ref).abs()
        assert (err <= bound).all(), (m, n, k, float(err.max()), (err > bound).nonzero()[:4])
        del a, resid, out, pre, ref, bound, got, err


# ---------------------------------------------------------------------------------- head_dim-64 attention
def ref_attention(qkv, mask, b, s, heads, window=None):
    """float64 softmax(q k^T / 8 + key padding) v, optionally banded |i - j| <= window (ModernBERT's local layers)."""
    q, k, v = qkv.double().view(b, s, 3, heads, 64).unbind(2)
    q, k, v = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    vis = (mask != 0)[:, None, None, :]
    if window is not None:
        i = torch.arange(s, device=qkv.device)
        vis = vis & ((i[:, None] - i[None, :]).abs() <= window)[None, None]
    scores = (q @ k.transpose(-1, -2) / 8.0).masked_fill(~vis, torch.finfo(torch.float64).min)
    return (torch.softmax(scores, -1) @ v).permute(0, 2, 1, 3).reshape(b * s, heads * 64)


@pytest.mark.parametrize('window', [None, 64], ids=['full', 'window64'])
@pytest.mark.parametrize('heads', [16, 32, 40, 64])
def test_attention_d64_many_heads(dev, heads, window, h16):
    """The head counts of the 1024 / 2048 / 2560 / 4096 widths (BERT, ESM-2, ModernBERT) on a ragged batch whose rows
    end inside, at and one past a 128-row query tile; padded query rows must stay finite."""
    b, s = 4, 300
    g = torch.Generator(device=dev).manual_seed(heads * 10 + (window or 0))
    qkv = torch.randn(b * s, 3 * heads * 64, device=dev, generator=g).to(h16)
    mask = (torch.arange(s, device=dev)[None] < torch.tensor([300, 129, 128, 1], device=dev)[:, None]).long()
    if window is None:
        ctx = nv.attention_d64(qkv, mask, b, s, heads)
    else:
        ctx = nv.attention_d64_window(qkv, mask, b, s, heads, window)
    ref = ref_attention(qkv, mask, b, s, heads, window)
    assert torch.isfinite(ctx.float()).all()
    valid = mask.bool().view(-1)
    got, ref = ctx.double()[valid], ref[valid]
    cos = torch.nn.functional.cosine_similarity(got.view(-1, 64), ref.reshape(-1, 64), dim=-1)
    live = ref.reshape(-1, 64).norm(dim=-1) > 1e-3
    assert (1 - cos[live]).max().item() <= 1e-3
    t = (3e-3 if h16 == torch.float16 else 1.2e-2) * 2
    torch.testing.assert_close(got, ref, rtol=t, atol=t)


# ---------------------------------------------------------------------------------- models at every width
# (family, H, heads, I) per case; head_dim 64 unless heads says otherwise (BERT 768 at 24 x 32), Mistral 128 with
# heads // 4 kv heads.  I is the real model's where one exists: bge-large / e5-large (BERT 1024: 4096), esm2_t36_3B
# (ESM-2 2560: 10240), ModernBERT-base (768: 1152), ModernBERT-large (1024: 2624, zero-padded to 2688 on the device);
# elsewhere a small legal 1024.  The first case of each family is its control, a width other tests already cover:
# BERT 768 (12 x 64), ESM-2 1280, ModernBERT 768 and Mistral 512.
MODEL_CASES = [
    ('bert', 768, 12, 3072), ('bert', 256, 4, 1024), ('bert', 384, 6, 1024), ('bert', 512, 8, 1024),
    ('bert', 640, 10, 1024), ('bert', 768, 24, 1024), ('bert', 1024, 16, 4096), ('bert', 1280, 20, 1024),
    ('bert', 2048, 32, 1024), ('bert', 2560, 40, 1024), ('bert', 4096, 64, 1024),
    ('esm', 1280, 20, 5120), ('esm', 256, 4, 1024), ('esm', 384, 6, 1024), ('esm', 512, 8, 1024),
    ('esm', 640, 10, 1024), ('esm', 768, 12, 1024), ('esm', 1024, 16, 1024), ('esm', 2048, 32, 1024),
    ('esm', 2560, 40, 10240), ('esm', 4096, 64, 1024),
    ('modernbert', 768, 12, 1152), ('modernbert', 256, 4, 1024), ('modernbert', 512, 8, 1024),
    ('modernbert', 1024, 16, 2624), ('modernbert', 1280, 20, 1024), ('modernbert', 2048, 32, 1024),
    ('modernbert', 2560, 40, 1024), ('modernbert', 4096, 64, 1024),
    ('mistral', 512, 4, 1024), ('mistral', 256, 2, 1024), ('mistral', 768, 6, 1024), ('mistral', 1024, 8, 1024),
    ('mistral', 1280, 10, 1024), ('mistral', 2048, 16, 1024), ('mistral', 2560, 20, 1024),
    ('mistral', 4096, 32, 1024),
]
# Per-family bound on 1 - cos for every check (tokens, pooled rows, after one layer).  The controls' worst value over
# both weight sets and both builds, measured on an H100 80GB HBM3 at a 700 W power limit: BERT 768 2.2e-5, ESM-2 1280
# 2.3e-5, ModernBERT 768 1.5e-5, Mistral 512 5.1e-6; the bounds are about 10x those.  The widest widths come closest:
# ModernBERT 4096 6.9e-5 (4.5x its control), BERT 4096 3.5e-5, ESM-2 4096 3.3e-5; every Mistral width <= 3.6e-6.
# At 1e-3, a LayerNorm that skips gamma / beta on its last pass at H >= 2048 passed every case with N(0, 0.02) weights,
# and a finalize that drops one of three row splits passed ESM-2 2048; these bounds catch both.
COS_TOL = {'bert': 2.2e-4, 'esm': 2.3e-4, 'modernbert': 1.5e-4, 'mistral': 5e-5}
B, S, LENS = 6, 192, [192, 129, 128, 127, 2, 1]
VOCAB = 1000


def case_id(case):
    fam, h, heads, _ = case
    return f'{fam}-{h}' + ('x32' if fam != 'mistral' and h // heads == 32 else '')


def model_config(fam, h, heads, inter):
    common = dict(hidden_size=h, num_hidden_layers=2, num_attention_heads=heads, intermediate_size=inter,
                  initializer_range=0.02)
    if fam == 'bert':
        from transformers import BertConfig
        return BertConfig(vocab_size=VOCAB, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12,
                          **common)
    if fam == 'esm':
        from transformers import EsmConfig
        return EsmConfig(vocab_size=33, max_position_embeddings=1026, position_embedding_type='rotary',
                         token_dropout=True, mask_token_id=32, pad_token_id=1, layer_norm_eps=1e-5,
                         emb_layer_norm_before=False, **common)
    if fam == 'modernbert':
        from transformers import ModernBertConfig
        # local_attention 128: layer 0 attends globally, layer 1 within |i - j| <= 64
        return ModernBertConfig(vocab_size=VOCAB, max_position_embeddings=512, local_attention=128, norm_eps=1e-5,
                                pad_token_id=0, bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2,
                                **common)
    from transformers import MistralConfig
    return MistralConfig(vocab_size=VOCAB, num_key_value_heads=max(1, heads // 4), head_dim=128,
                         max_position_embeddings=512, rms_norm_eps=1e-5, sliding_window=None, **common)


def model_parts(fam):
    """(native encoder class, random state dict maker, oracle forward)"""
    from distllm_b200.embed.encoders import native as N
    from distllm_b200.embed.encoders import weights as W
    from oracle import bert as obert
    from oracle import esm as oesm
    from oracle import mistral as omis
    from oracle import modernbert as omb

    return {'bert': (N.NativeBertEncoder, W.random_bert_state_dict, obert.bert_forward),
            'esm': (N.NativeEsm2Encoder, W.random_esm_state_dict, oesm.esm_forward),
            'modernbert': (N.NativeModernBertEncoder, W.random_modernbert_state_dict, omb.modernbert_forward),
            'mistral': (N.NativeMistralEncoder, W.random_mistral_state_dict, omis.mistral_forward)}[fam]


_ORACLE: dict = {}


def oracle_case(case, weights):
    """Inputs, weights and fp32 oracle states of one (family, width, weights), computed once for the module.  The
    oracle modules cast every parameter to fp32 themselves, so fp32 is their precision here.  ``return_all`` gives
    the state after each layer: what the same checkpoint truncated to l layers returns (num_hidden_layers = l)."""
    key = (case, weights)
    if key in _ORACLE:
        return _ORACLE[key]
    fam, h, heads, inter = case
    cfg = model_config(*case)
    _, make_sd, forward = model_parts(fam)
    sd = make_sd(cfg, seed=h + heads, device='cpu')
    if weights == 'outliers':
        add_outliers(sd, fam, seed=h)
    g = torch.Generator().manual_seed(h + 1)
    mask = (torch.arange(S)[None] < torch.tensor(LENS)[:, None]).long()
    types = None
    if fam == 'esm':
        ids = torch.randint(4, 24, (B, S), generator=g).masked_fill(mask == 0, 1)
        ids[:, 0] = 0
        ids[0, 40:52] = 32        # <mask> tokens: token dropout rescales rows 0 and 1 differently
        ids[1, 100] = 32
    else:
        ids = torch.randint(5, VOCAB, (B, S), generator=g)
    if fam == 'bert':
        types = (torch.arange(S)[None] >= torch.tensor(LENS)[:, None] // 2).long() * mask
        states = forward(sd, cfg, ids, mask, types, return_all=True)[1:]
    else:
        states = forward(sd, cfg, ids, mask, return_all=True)
    out = dict(cfg=cfg, sd=sd, ids=ids, mask=mask, types=types, one=states[0], full=states[-1])
    _ORACLE.clear()            # cases run grouped by (family, width): keep one model's tensors at a time
    _ORACLE[key] = out
    return out


def worst(got: np.ndarray, ref: np.ndarray, what: str) -> float:
    """1 - min cosine over rows the reference does not zero out; rows it zeros must be zero too."""
    assert np.isfinite(got).all(), what
    live = np.linalg.norm(ref, axis=-1) > 0
    assert not got[~live].any(), what
    return float(1 - cosine_rows(got[live], ref[live]).min())


def set_layers(enc, n: int) -> None:
    enc._lib.b2e_debug_set_layers.argtypes = [C.c_void_p, C.c_int]
    nv.check(enc._lib.b2e_debug_set_layers(enc._handle, n), enc._lib)


def packed_vs_padded(enc, ids, mask, types) -> float:
    """1 - min cos between the padding-free token layout and the padded one (b2e_debug_set_packing)."""
    lib = enc._lib
    lib.b2e_debug_set_packing.argtypes = [C.c_int]
    out = 0.0
    try:
        for kind in (nv.POOL_MEAN_REF, nv.POOL_MEAN_PER_ROW, nv.POOL_LAST_TOKEN):
            lib.b2e_debug_set_packing(1)
            packed = enc.encode_pooled(ids, mask, types, kind, True).clone()
            lib.b2e_debug_set_packing(0)
            padded = enc.encode_pooled(ids, mask, types, kind, True).clone()
            assert torch.isfinite(packed).all()
            live = padded.norm(dim=-1) > 0
            assert torch.equal(live, packed.norm(dim=-1) > 0)
            cos = torch.nn.functional.cosine_similarity(packed[live].double(), padded[live].double())
            out = max(out, 1 - cos.min().item())
    finally:
        lib.b2e_debug_set_packing(1)
    return out


def storages(fam):
    return ['f16'] if fam == 'mistral' else ['bf16', 'f16']


@pytest.mark.parametrize('case,weights,storage',
                         [pytest.param(c, w, st, id=f'{case_id(c)}-{w}-{st}')
                          for c in MODEL_CASES for w in ('normal', 'outliers') for st in storages(c[0])])
def test_model_width_vs_oracle(case, weights, storage, record_property):
    """2 layers on a ragged batch (lengths 192, 129, 128, 127, 2, 1): token states at attended positions, pooled rows
    (mean with the reference's quirk and last token; ESM-2 mean only), the same after one layer, and the packed token
    layout against the padded one."""
    fam, h = case[0], case[1]
    o = oracle_case(case, weights)
    cls = model_parts(fam)[0]
    ids, mask, types = o['ids'], o['mask'], o['types']
    valid = mask.bool().numpy()
    kinds = [(nv.POOL_MEAN_REF, opool.average_pool)]
    if fam != 'esm':
        kinds.append((nv.POOL_LAST_TOKEN, opool.last_token_pool))
    margins = {}
    enc = cls(o['cfg'], o['sd'], storage=storage)
    try:
        for depth, ref_hidden in (('L2', o['full']), ('L1', o['one'])):
            set_layers(enc, 0 if depth == 'L2' else 1)
            hidden = enc.encode(ids, mask, types).cpu().numpy()
            margins[f'{depth}/tokens'] = worst(hidden[valid], ref_hidden.numpy()[valid], f'{depth} tokens')
            for kind, pool in kinds:
                got = enc.encode_pooled(ids, mask, types, kind, False).cpu().numpy()
                margins[f'{depth}/pool{kind}'] = worst(got, pool(ref_hidden, mask.clone()).numpy(),
                                                       f'{depth} pool {kind}')
        set_layers(enc, 0)
        packed = packed_vs_padded(enc, ids, mask, types)
    finally:
        enc.close()
    record_property('one_minus_cos', json.dumps({'packed': packed, **margins}))
    assert packed < 1e-6, packed
    bad = {k: v for k, v in margins.items() if not v < COS_TOL[fam]}
    assert not bad, (fam, h, weights, storage, bad, COS_TOL[fam])
