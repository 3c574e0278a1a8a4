"""-m gpu: each native kernel, called through the C ABI, against a torch fp32 reference or the
golden vectors produced by the reference.  The 16-bit kernels run in BOTH builds of the library (h16 =
float16 -> libb2e.so, bfloat16 -> libb2e_bf16.so); tolerances follow the storage type's rounding
(2^-11 resp. 2^-8 relative)."""

from __future__ import annotations

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(params=[torch.float16, torch.bfloat16], ids=['f16', 'bf16'])
def h16(request):
    """The 16-bit storage type = which build of the library the call lands in."""
    return request.param


def close(got, ref, h16, scale: float = 1.0):
    """assert_close with the storage type's rounding: `scale` x (3e-3 for half, 1.2e-2 for bfloat16)."""
    t = (3e-3 if h16 == torch.float16 else 1.2e-2) * scale
    torch.testing.assert_close(got, ref, rtol=t, atol=t)


GEMM_SHAPES = [(128, 256, 64), (300, 768, 768), (1000, 2304, 768), (517, 3072, 768), (517, 768, 3072),
               (200, 384, 128), (1, 768, 768), (20000, 768, 768)]


@pytest.mark.parametrize('m,n,k', GEMM_SHAPES)
@pytest.mark.parametrize('epi', [nv.EPI_BIAS, nv.EPI_BIAS_GELU, nv.EPI_BIAS_RESID])
def test_gemm_epilogues(dev, m, n, k, epi, h16):
    g = torch.Generator(device=dev).manual_seed(m * 7 + n + k + epi)
    a = (torch.randn(m, k, device=dev, generator=g) * 0.5).to(h16)
    w = (torch.randn(n, k, device=dev, generator=g) * 0.05).to(h16)
    bias = torch.randn(n, device=dev, generator=g) * 0.1
    resid = torch.randn(m, n, device=dev, generator=g).to(h16)
    out = nv.gemm_h16(a, w, bias, resid if epi == nv.EPI_BIAS_RESID else None, epi)
    ref = a.float() @ w.float().T + bias
    if epi == nv.EPI_BIAS_GELU:
        ref = torch.nn.functional.gelu(ref)
    if epi == nv.EPI_BIAS_RESID:
        ref = ref + resid.float()
    assert out.dtype == h16 and out.shape == (m, n)
    close(out.float(), ref, h16)


def test_gemm_rejects_bad_shapes(dev, h16):
    a = torch.zeros(8, 100, device=dev, dtype=h16)
    w = torch.zeros(128, 100, device=dev, dtype=h16)
    with pytest.raises(nv.NativeError, match='K=100'):
        nv.gemm_h16(a, w, torch.zeros(128, device=dev))
    with pytest.raises(nv.NativeError, match='N=100'):
        nv.gemm_h16(torch.zeros(8, 64, device=dev, dtype=h16),
                     torch.zeros(100, 64, device=dev, dtype=h16), torch.zeros(100, device=dev))


@pytest.fixture(params=[None, 5, 0, 69, 64, 193], ids=['shipping', 'two-wg-poly', 'two-wg', 'four-wg-poly', 'four-wg-vote', 'four-wg-epilogue-role'])
def att_variant(request, h16):
    """Which variant of the head_dim-64 attention kernel (attention.cuh) the calls of a test reach: the library's
    default, two consumer warpgroups per CTA (5: one exponential in four as a polynomial, 0: every chunk reads its
    bias row, none is known from attn_prep to be fully attended), or four (69: polynomial exponentials, 64: every
    chunk reads its bias row, 193: the producer warp stores the output tiles with TMA)."""
    import ctypes

    lib = nv.load(nv.storage_of(h16))
    lib.b2e_debug_set_att3_variant.argtypes = [ctypes.c_int]
    if request.param is not None:
        assert lib.b2e_debug_set_att3_variant(request.param) == 0
    yield request.param
    lib.b2e_debug_set_att3_variant(-1)   # back to B2E_ATT3 / the built-in default


def ref_attention(qkv, mask, b, s, heads):
    q, k, v = qkv.float().view(b, s, 3, heads, 64).unbind(2)
    q, k, v = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    scores = q @ k.transpose(-1, -2) / 8.0
    bias = torch.zeros(b, 1, 1, s, device=qkv.device)
    bias.masked_fill_(mask.view(b, 1, 1, s) == 0, torch.finfo(torch.float32).min)
    p = torch.softmax(scores + bias, dim=-1)
    return (p @ v).permute(0, 2, 1, 3).reshape(b * s, heads * 64)


@pytest.mark.parametrize('b,s,heads,ragged', [(2, 128, 2, False), (2, 512, 12, False), (3, 200, 12, True),
                                              (2, 512, 12, True), (4, 37, 4, True), (5, 1, 4, False),
                                              (2, 129, 4, True), (1, 384, 12, True), (2, 640, 2, False),
                                              (1, 1026, 4, True), (3, 257, 2, True)])
def test_attention_matches_reference(dev, b, s, heads, ragged, h16, att_variant):
    g = torch.Generator(device=dev).manual_seed(b * 1000 + s)
    qkv = torch.randn(b * s, 3 * heads * 64, device=dev, generator=g).to(h16)
    mask = torch.ones(b, s, dtype=torch.int64, device=dev)
    if ragged:
        for i in range(b):
            mask[i, max(1, s - 17 * (i + 1)):] = 0
    ctx = nv.attention_d64(qkv, mask, b, s, heads)
    close(ctx.float(), ref_attention(qkv, mask, b, s, heads), h16, 2.0)


def test_attention_mask_with_holes_and_fully_masked_row(dev, h16, att_variant):
    """Arbitrary 0/1 masks (left padding, holes); an all-zero mask degenerates to a uniform
    distribution over the S keys exactly like HF's additive most-negative-finite mask."""
    b, s, heads = 3, 96, 4
    g = torch.Generator(device=dev).manual_seed(9)
    qkv = torch.randn(b * s, 3 * heads * 64, device=dev, generator=g).to(h16)
    mask = torch.ones(b, s, dtype=torch.int64, device=dev)
    mask[0, :40] = 0            # left padding
    mask[1, 10:20] = 0          # a hole
    mask[2, :] = 0              # nothing attended
    ctx = nv.attention_d64(qkv, mask, b, s, heads)
    ref = ref_attention(qkv, mask, b, s, heads)
    assert torch.isfinite(ctx.float()).all()
    close(ctx.float(), ref, h16, 2.0)


def test_attention_many_items_per_cta(dev, h16, att_variant):
    """More work items than SMs: several waves of CTAs over ragged sequences, the K/V ring reused per CTA."""
    b, s, heads = 40, 300, 12
    g = torch.Generator(device=dev).manual_seed(77)
    qkv = torch.randn(b * s, 3 * heads * 64, device=dev, generator=g).to(h16)
    lens = torch.randint(1, s + 1, (b,), generator=torch.Generator().manual_seed(5))
    mask = (torch.arange(s)[None] < lens[:, None]).long().to(dev)
    ctx = nv.attention_d64(qkv, mask, b, s, heads)
    ref = ref_attention(qkv, mask, b, s, heads)
    valid = mask.bool().view(-1)
    close(ctx.float()[valid], ref[valid], h16, 2.0)
    assert torch.isfinite(ctx.float()).all()


def test_attention_large_scores_trigger_rescale(dev, h16, att_variant):
    """Scores that grow along the key axis force the lazy online-softmax rescale path."""
    b, s, heads = 2, 512, 2
    g = torch.Generator(device=dev).manual_seed(78)
    qkv = torch.randn(b * s, 3 * heads * 64, device=dev, generator=g)
    # keys later in the sequence get larger norms -> row maxima jump by far more than 2^8
    ramp = torch.linspace(0.2, 6.0, s, device=dev).repeat(b)[:, None]
    qkv[:, heads * 64:2 * heads * 64] *= ramp
    qkv = qkv.to(h16)
    mask = torch.ones(b, s, dtype=torch.int64, device=dev)
    ctx = nv.attention_d64(qkv, mask, b, s, heads)
    close(ctx.float(), ref_attention(qkv, mask, b, s, heads), h16, 3.0)


@pytest.mark.parametrize('h', [256, 768, 1024, 1280])
def test_layernorm(dev, h, h16):
    g = torch.Generator(device=dev).manual_seed(h)
    x = (torch.randn(1003, h, device=dev, generator=g) * 3 + 1).to(h16)
    gamma = torch.randn(h, device=dev, generator=g)
    beta = torch.randn(h, device=dev, generator=g)
    ref = torch.nn.functional.layer_norm(x.float(), (h,), gamma, beta, 1e-12)
    torch.testing.assert_close(nv.layernorm(x, gamma, beta, 1e-12, torch.float32), ref, rtol=1e-4, atol=1e-4)
    close(nv.layernorm(x, gamma, beta, 1e-12).float(), ref, h16, 2.0)


@pytest.mark.parametrize('case', ['ragged', 'full', 'single', 'left_padded_like'])
def test_pool_mean_matches_reference_vectors(dev, pool_golden, case):
    emb = torch.from_numpy(pool_golden[f'{case}/emb']).to(dev)
    mask = torch.from_numpy(pool_golden[f'{case}/mask']).to(dev)
    got = nv.pool_mean(emb, mask)
    np.testing.assert_allclose(got.cpu().numpy(), pool_golden[f'{case}/mean'], rtol=1e-5, atol=1e-6)
    # the caller's mask is rewritten exactly like distllm/embed/poolers/mean.py:35-36
    np.testing.assert_array_equal(mask.cpu().numpy(), pool_golden[f'{case}/mask_after'])


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_pool_mean_half_inputs(dev, dtype):
    from oracle import pooling as opool

    g = torch.Generator().manual_seed(4)
    emb = torch.randn(6, 50, 512, generator=g).to(dtype)
    lens = torch.tensor([50, 3, 17, 17, 1, 44])
    mask = (torch.arange(50)[None] < lens[:, None]).long()
    ref = opool.average_pool(emb.float(), mask.clone())
    got = nv.pool_mean(emb.to(dev), mask.to(dev))
    assert got.dtype == torch.float32
    torch.testing.assert_close(got.cpu(), ref, rtol=1e-2, atol=1e-2)


def test_pool_mean_per_row_mode_and_no_mutation(dev):
    g = torch.Generator().manual_seed(5)
    emb = torch.randn(4, 30, 256, generator=g)
    lens = [30, 7, 12, 2]
    mask = (torch.arange(30)[None] < torch.tensor(lens)[:, None]).long()
    ref = torch.stack([emb[i, 1:n - 1].mean(0) if n > 2 else torch.zeros(256) for i, n in enumerate(lens)])
    m = mask.to(dev)
    got = nv.pool_mean(emb.to(dev), m, nv.POOL_MEAN_PER_ROW, mutate_mask=False)
    torch.testing.assert_close(got.cpu(), ref, rtol=1e-5, atol=1e-6)
    assert torch.equal(m.cpu(), mask)


@pytest.mark.parametrize('case', ['full', 'single', 'left_padded_like', 'leftpad'])
def test_pool_last_token_matches_reference_vectors(dev, pool_golden, case):
    emb = torch.from_numpy(pool_golden[f'{case}/emb']).to(dev)
    mask = torch.from_numpy(pool_golden[f'{case}/mask']).to(dev)
    got = nv.pool_last_token(emb, mask)
    np.testing.assert_array_equal(got.cpu().numpy(), pool_golden[f'{case}/last'])


def test_adjacent_cosine_matches_reference_vectors(dev, semantic_golden):
    emb = torch.from_numpy(semantic_golden['emb']).to(dev)
    ranges = [tuple(r) for r in semantic_golden['doc_ranges']]
    doc_id = torch.empty(len(emb), dtype=torch.int32)
    for k, (lo, hi) in enumerate(ranges):
        doc_id[lo:hi] = k
    d = nv.adjacent_cosine_dist(emb, doc_id.to(dev)).cpu().numpy()
    for k, (lo, hi) in enumerate(ranges):
        np.testing.assert_allclose(d[lo:hi - 1], semantic_golden[f'dist/{k}'], rtol=0, atol=5e-7)
        if hi < len(emb):
            assert np.isnan(d[hi - 1]), 'pairs across a document boundary must be NaN'
    # no doc ids: plain consecutive distances; 0/1-row inputs: nothing to compute
    plain = nv.adjacent_cosine_dist(emb).cpu().numpy()
    assert not np.isnan(plain).any() and plain.shape == (len(emb) - 1,)
    assert nv.adjacent_cosine_dist(emb[:1]).shape == (0,)


def test_product_split_equals_oracle_split_on_same_embeddings(dev, semantic_golden):
    """Discrete output: on identical embeddings the native distance kernel + host percentile split
    must give exactly the reference's row groups."""
    from distllm_b200.embed.embedders.semantic_chunk import build_chunks
    from oracle import semantic as osem

    emb = semantic_golden['emb']
    ranges = [tuple(int(v) for v in r) for r in semantic_golden['doc_ranges']]
    dev_emb = torch.from_numpy(emb).to(dev)
    for pct in (50, 90, 95):
        got = []
        for lo, hi in ranges:
            d = nv.adjacent_cosine_dist(dev_emb[lo:hi].contiguous()).cpu().numpy().astype(np.float64)
            got.extend((lo + s, lo + e) for s, e in build_chunks(d, pct))
        assert got == osem.split_rows(emb, ranges, pct)


def test_l2_normalize(dev):
    x = torch.randn(33, 768, device=dev)
    x[5] = 0
    ref = torch.nn.functional.normalize(x, p=2, dim=-1)
    torch.testing.assert_close(nv.l2_normalize_(x.clone()), ref, rtol=1e-6, atol=1e-7)


# ---------------------------------------------------------------------------- Mistral-family kernels
@pytest.mark.parametrize('m,i,k', [(128, 128, 64), (300, 768, 512), (1000, 1792, 1024), (5, 256, 4096)])
def test_gemm_swiglu_epilogue(dev, m, i, k, h16):
    """gate/up rows interleaved in blocks of 64 -> silu(gate) * up, no bias, [M, I] out."""
    from distllm_b200.embed.encoders.weights import interleave_gate_up

    g = torch.Generator(device=dev).manual_seed(m + i + k)
    a = (torch.randn(m, k, device=dev, generator=g) * 0.5).to(h16)
    gate = (torch.randn(i, k, device=dev, generator=g) * 0.08).to(h16)
    up = (torch.randn(i, k, device=dev, generator=g) * 0.08).to(h16)
    out = nv.gemm_h16(a, interleave_gate_up(gate, up).contiguous(), None, None, nv.EPI_SWIGLU)
    ref = torch.nn.functional.silu(a.float() @ gate.float().T) * (a.float() @ up.float().T)
    assert out.dtype == h16 and out.shape == (m, i)
    close(out.float(), ref, h16, 1.3)


def test_gemm_without_bias(dev, h16):
    g = torch.Generator(device=dev).manual_seed(4)
    a = torch.randn(200, 256, device=dev, generator=g).to(h16)
    w = (torch.randn(512, 256, device=dev, generator=g) * 0.05).to(h16)
    out = nv.gemm_h16(a, w, None)
    close(out.float(), a.float() @ w.float().T, h16)


def ref_attention_causal(qkv, mask, b, s, heads, kv_heads, window):
    d = 128
    q = qkv[:, :heads * d].float().view(b, s, heads, d).permute(0, 2, 1, 3)
    k = qkv[:, heads * d:(heads + kv_heads) * d].float().view(b, s, kv_heads, d).permute(0, 2, 1, 3)
    v = qkv[:, (heads + kv_heads) * d:].float().view(b, s, kv_heads, d).permute(0, 2, 1, 3)
    k = k.repeat_interleave(heads // kv_heads, dim=1)
    v = v.repeat_interleave(heads // kv_heads, dim=1)
    i = torch.arange(s, device=qkv.device)[:, None]
    j = torch.arange(s, device=qkv.device)[None, :]
    vis = j <= i
    if window:
        vis = vis & (i - j < window)
    vis = vis[None, None] & (mask != 0)[:, None, None, :]
    scores = (q @ k.transpose(-1, -2)) * d ** -0.5
    p = torch.softmax(scores.masked_fill(~vis, float('-inf')), dim=-1)
    alive = vis.any(-1)                      # [B,1,S]: query rows with at least one visible key
    p = torch.nan_to_num(p, nan=0.0)
    out = (p @ v).permute(0, 2, 1, 3).reshape(b * s, heads * d)
    return out, alive.expand(b, heads, s)[:, 0].reshape(b * s)


CAUSAL_CASES = [
    # b, s, heads, kv_heads, window, padding
    (2, 128, 2, 1, 0, 'none'), (2, 256, 4, 2, 0, 'none'), (3, 200, 4, 1, 0, 'right'),
    (2, 513, 2, 2, 0, 'right'), (2, 320, 4, 2, 80, 'right'), (2, 320, 4, 2, 80, 'left'),
    (1, 1100, 2, 1, 0, 'none'), (1, 1100, 2, 1, 300, 'left'), (4, 37, 2, 1, 16, 'right'),
    (5, 1, 2, 2, 0, 'none'), (2, 640, 8, 2, 128, 'none'), (2, 300, 4, 4, 1, 'none'),
    (2, 400, 2, 1, 64, 'right'), (2, 400, 2, 1, 65, 'left'),
]


@pytest.mark.parametrize('b,s,heads,kv_heads,window,padding', CAUSAL_CASES)
def test_attention_causal_d128_matches_reference(dev, b, s, heads, kv_heads, window, padding, h16):
    g = torch.Generator(device=dev).manual_seed(b * 1000 + s + window)
    qkv = torch.randn(b * s, (heads + 2 * kv_heads) * 128, device=dev, generator=g).to(h16)
    mask = torch.ones(b, s, dtype=torch.int64, device=dev)
    for r in range(b):
        n_pad = min(s - 1, 23 * r + (5 if padding != 'none' else 0)) if padding != 'none' else 0
        if padding == 'right' and n_pad:
            mask[r, s - n_pad:] = 0
        if padding == 'left' and n_pad:
            mask[r, :n_pad] = 0
    ctx = nv.attention_causal_d128(qkv, mask, b, s, heads, kv_heads, window)
    ref, alive = ref_attention_causal(qkv, mask, b, s, heads, kv_heads, window)
    assert torch.isfinite(ctx.float()).all()
    # rows that see no key at all (queries inside left padding) are unspecified; everything else,
    # including padded query positions that still see attended keys, must match
    close(ctx.float()[alive], ref[alive], h16, 2.0)


def test_attention_causal_d128_many_items_and_rescale(dev, h16):
    """More items than SMs with mixed lengths, and key norms that grow along the sequence so the lazy
    rescale path runs on top of the causal/window edge masking."""
    b, s, heads, kv_heads, window = 24, 700, 8, 2, 333
    g = torch.Generator(device=dev).manual_seed(91)
    qkv = torch.randn(b * s, (heads + 2 * kv_heads) * 128, device=dev, generator=g)
    ramp = torch.linspace(0.2, 4.0, s, device=dev).repeat(b)[:, None]
    qkv[:, heads * 128:(heads + kv_heads) * 128] *= ramp
    qkv = qkv.to(h16)
    lens = torch.randint(1, s + 1, (b,), generator=torch.Generator().manual_seed(6))
    mask = (torch.arange(s)[None] < lens[:, None]).long().to(dev)
    ctx = nv.attention_causal_d128(qkv, mask, b, s, heads, kv_heads, window)
    ref, alive = ref_attention_causal(qkv, mask, b, s, heads, kv_heads, window)
    sel = alive & mask.bool().view(-1)
    assert torch.isfinite(ctx.float()).all()
    close(ctx.float()[sel], ref[sel], h16, 3.0)


# ---------------------------------------------------------------------------- exact inner-product top-k
def check_topk_against_oracle(queries, corpus, k, scores, idx, atol=2e-5):
    from oracle import search as osearch

    q = queries.shape[0]
    ref_s, ref_i = osearch.topk_inner_product(queries.cpu().numpy(), corpus.float().cpu().numpy(), k)
    kk = ref_s.shape[1]
    got_s, got_i = scores.cpu().numpy(), idx.cpu().numpy()
    # scores: fp32 dot products in a different summation order
    np.testing.assert_allclose(got_s[:, :kk], ref_s, rtol=0, atol=atol)
    assert (np.diff(got_s[:, :kk], axis=1) <= 0).all()
    if kk < k:   # fewer rows than k: the tail is marked empty
        assert (got_i[:, kk:] == -1).all() and np.isinf(got_s[:, kk:]).all()
    # indices: identical wherever the oracle's neighbouring scores are not within rounding of each other
    full = queries.cpu().numpy().astype(np.float64) @ corpus.float().cpu().numpy().astype(np.float64).T
    for r in range(q):
        assert len(set(got_i[r, :kk].tolist())) == kk
        np.testing.assert_allclose(full[r, got_i[r, :kk]], ref_s[r], rtol=0, atol=atol)
        clear = np.abs(np.diff(ref_s[r])) > 5 * atol
        stable = np.concatenate([[True], clear]) & np.concatenate([clear, [True]])
        assert (got_i[r, :kk][stable] == ref_i[r][stable]).all()


@pytest.mark.parametrize('q,n,h,k', [(1, 1000, 768, 10), (7, 5000, 768, 100), (16, 20000, 768, 5),
                                     (33, 3000, 256, 64), (3, 17, 128, 8), (2, 5, 768, 10),
                                     (5, 40000, 1280, 256), (4, 2000, 4096, 20), (1, 1, 768, 1)])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_topk_inner_product_matches_oracle(dev, q, n, h, k, dtype):
    from oracle import search as osearch

    g = torch.Generator(device=dev).manual_seed(q * 31 + n + k)
    if dtype == torch.bfloat16 and h % 256:
        with pytest.raises(nv.NativeError, match='multiple of 256'):
            nv.topk_ip(torch.zeros(q, h, device=dev), torch.zeros(n, h, device=dev, dtype=dtype), k)
        return
    corpus = torch.randn(n, h, device=dev, generator=g)
    corpus = corpus / corpus.norm(dim=1, keepdim=True)
    queries = torch.randn(q, h, device=dev, generator=g)
    queries = queries / queries.norm(dim=1, keepdim=True)
    corpus = corpus.to(dtype).contiguous()
    scores, idx = nv.topk_ip(queries, corpus, k)
    check_topk_against_oracle(queries, corpus, k, scores, idx)


@pytest.mark.parametrize('q,n,h,k', [(1, 40000, 768, 10), (16, 100000, 768, 100), (5, 70001, 1280, 256),
                                     (33, 50000, 256, 64), (3, 32768, 128, 1), (7, 33000, 4096, 20)])
@pytest.mark.parametrize('normalised', [True, False])
def test_topk_tensor_core_scan_matches_oracle(dev, q, n, h, k, normalised):
    """b2e_topk_ip_tc: TF32 scan on the tensor cores, exact fp32 decision -- the SAME contract as b2e_topk_ip."""
    g = torch.Generator(device=dev).manual_seed(q * 17 + n + k)
    corpus = torch.randn(n, h, device=dev, generator=g)
    queries = torch.randn(q, h, device=dev, generator=g)
    if normalised:
        corpus = corpus / corpus.norm(dim=1, keepdim=True)
        queries = queries / queries.norm(dim=1, keepdim=True)
        atol = 2e-5
    else:   # row norms spread over a factor of four: the margin is sized by the LARGEST norm
        corpus = corpus * (0.5 + 1.5 * torch.rand(n, 1, device=dev, generator=g))
        atol = 2e-5 * float(corpus.norm(dim=1).max() * queries.norm(dim=1).max())
    corpus = corpus.contiguous()
    max_norm = nv.max_row_norm(corpus)
    assert abs(max_norm - float(corpus.norm(dim=1).max())) <= 1e-5 * max_norm
    scores, idx = nv.topk_ip(queries, corpus, k, max_norm=max_norm)
    # normalised rows (what the reference indexes: faiss.normalize_L2, search.py:258-278) must stay on the fast
    # path; with spread-out norms the one global bound may be too loose and the call may redo itself exactly
    if normalised:
        assert not nv.topk_tc_fell_back()
    check_topk_against_oracle(queries, corpus, k, scores, idx, atol=atol)
    # and the two paths return the same bits: the contract of b2e_topk_ip_tc (include/b2e.h)
    s2, i2 = nv.topk_ip(queries, corpus, k)
    assert torch.equal(scores, s2) and torch.equal(idx, i2)


def test_topk_tensor_core_scan_falls_back_on_degenerate_corpus(dev):
    """Thousands of rows tie with the k-th best (a corpus of duplicates): the candidate buffer overflows, the call
    is redone by the exact scan on the device -- same scores and indices as b2e_topk_ip bit for bit.  Among
    identical rows the lowest ids come back: the first ten copies of the best vector, best + 8 m."""
    g = torch.Generator(device=dev).manual_seed(5)
    base = torch.randn(8, 768, device=dev, generator=g)
    base = base / base.norm(dim=1, keepdim=True)
    corpus = base.repeat(6000, 1).contiguous()      # 48 000 rows, 8 distinct
    queries = torch.randn(3, 768, device=dev, generator=g)
    scores, idx = nv.topk_ip(queries, corpus, 10, max_norm=1.0)
    assert nv.topk_tc_fell_back()
    s2, i2 = nv.topk_ip(queries, corpus, 10)
    assert torch.equal(scores, s2) and torch.equal(idx, i2)
    # every copy of one vector scores the same bits, so the ten best are the ten lowest copies of the best one
    best = (corpus[:8] @ queries.T).argmax(dim=0)
    assert torch.equal(idx.cpu(), (best[:, None] + 8 * torch.arange(10, device=dev)).cpu())
    assert (scores == scores[:, :1]).all()
    # a too-small norm bound can only shrink the margin, never corrupt memory; with the true bound it is exact
    corpus2 = torch.randn(40000, 768, device=dev, generator=g)
    s3, i3 = nv.topk_ip(queries, corpus2, 10, max_norm=nv.max_row_norm(corpus2))
    check_topk_against_oracle(queries, corpus2, 10, s3, i3, atol=2e-5 * 28 * float(queries.norm(dim=1).max()))


def test_topk_rejects_bad_arguments(dev):
    c = torch.zeros(10, 768, device=dev)
    qq = torch.zeros(2, 768, device=dev)
    with pytest.raises(nv.NativeError, match='k=300'):
        nv.topk_ip(qq, c, 300)
    with pytest.raises(nv.NativeError, match='H=100'):
        nv.topk_ip(torch.zeros(2, 100, device=dev), torch.zeros(10, 100, device=dev), 3)


# ---------------------------------------------------------------------------------- binary retrieval
@pytest.mark.parametrize('n,h,q,k,mult', [(5000, 768, 3, 10, 2), (20000, 1280, 9, 5, 4), (40, 256, 2, 8, 2),
                                          (3000, 64 * 3, 1, 100, 2)])
def test_ubinary_search_matches_oracle(n, h, q, k, mult):
    """b2e_pack_ubinary / b2e_search_ubinary vs the CPU restatement of packbits + IndexBinaryFlat + rescoring
    (oracle/search.py): packed bits and result indices bit-exact (integer / index work), scores to fp32 rounding."""
    from oracle import search as osearch

    rng = np.random.default_rng(n + h)
    corpus = rng.standard_normal((n, h)).astype(np.float32)
    corpus[rng.integers(0, n, 50)] = 0.0          # zero rows pack to all-zero bits
    if n > 100:
        corpus[100:110] = corpus[7]                # exact duplicates: Hamming ties resolved by row id
    queries = rng.standard_normal((q, h)).astype(np.float32)
    queries[0] = corpus[7] + 0.05 * rng.standard_normal(h).astype(np.float32)
    bits = nv.pack_ubinary(torch.from_numpy(corpus).cuda())
    ref_bits = osearch.quantize_ubinary(corpus)
    assert np.array_equal(bits.cpu().numpy(), ref_bits)
    scores, indices = nv.search_ubinary(torch.from_numpy(queries).cuda(), bits, k, mult)
    ref_s, ref_i = osearch.search_ubinary(queries, ref_bits, k, mult)
    kk = ref_i.shape[1]
    got_i, got_s = indices.cpu().numpy(), scores.cpu().numpy()
    # rescored scores are sums of up to h floats: order of summation differs -> compare with a tolerance, and
    # indices wherever the reference scores are not tied within that tolerance
    np.testing.assert_allclose(got_s[:, :kk], ref_s, rtol=1e-5, atol=1e-4)
    for r in range(q):
        gap = np.abs(np.diff(ref_s[r])) > 1e-3
        stable = np.concatenate(([True], gap)) & np.concatenate((gap, [True]))
        assert np.array_equal(got_i[r, :kk][stable], ref_i[r][stable]), (r, got_i[r], ref_i[r])
        assert set(got_i[r, :kk]) == set(ref_i[r])
    if kk < k:
        assert (got_i[:, kk:] == -1).all() and np.isinf(got_s[:, kk:]).all()


def test_exact_index_ubinary_through_the_retriever_surface():
    from distllm_b200.rag.search import ExactIndex
    from distllm_b200.rag.search import ExactIndexConfig
    from oracle import search as osearch

    rng = np.random.default_rng(9)
    corpus = rng.standard_normal((4000, 768)).astype(np.float32)
    index = ExactIndex(corpus, config=ExactIndexConfig(precision='ubinary', rescore_multiplier=3))
    assert index.corpus.dtype == torch.uint8 and index.corpus.shape == (4000, 96) and len(index) == 4000
    q = ExactIndex.transform(corpus[[5, 77]] + 0.1 * rng.standard_normal((2, 768)).astype(np.float32))
    res = index.search(q, top_k=4)
    ref_s, ref_i = osearch.search_ubinary(q, osearch.quantize_ubinary(corpus), 4, 3)
    assert [r[0] for r in res.total_indices] == [5, 77]
    assert res.total_indices == ref_i.tolist()
    np.testing.assert_allclose(np.array(res.total_scores), ref_s, rtol=1e-5, atol=1e-4)
    kept = index.search(q, top_k=4, score_threshold=float(ref_s[0, 1]))
    assert kept.total_indices[0] == ref_i[0, :2].tolist()


@pytest.mark.parametrize('m,i,k', [(300, 1152, 768), (1000, 2688, 1024)])
def test_gemm_geglu_epilogue(dev, m, i, k, h16):
    """ModernBERT's gated MLP: Wi rows = input | gate (transformers/models/modernbert/modeling_modernbert.py
    :88-91), interleaved in blocks of 64 for the epilogue: out = gelu(x Wi_in^T) * (x Wi_gate^T)."""
    from distllm_b200.embed.encoders.weights import interleave_gate_up

    g = torch.Generator(device=dev).manual_seed(m + i)
    a = (torch.randn(m, k, device=dev, generator=g) * 0.5).to(h16)
    w_in = (torch.randn(i, k, device=dev, generator=g) * 0.08).to(h16)
    w_gate = (torch.randn(i, k, device=dev, generator=g) * 0.08).to(h16)
    out = nv.gemm_h16(a, interleave_gate_up(w_in, w_gate).contiguous(), None, None, nv.EPI_GEGLU)
    ref = torch.nn.functional.gelu(a.float() @ w_in.float().T) * (a.float() @ w_gate.float().T)
    assert out.dtype == h16 and out.shape == (m, i)
    close(out.float(), ref, h16, 1.3)


@pytest.mark.parametrize('b,s,heads,window', [(2, 512, 4, 64), (3, 333, 2, 64), (1, 1500, 2, 64), (2, 200, 4, 16),
                                              (2, 700, 2, 300)])
def test_attention_d64_sliding_window(dev, b, s, heads, window, h16, att_variant):
    """Bidirectional sliding window |i - j| <= window (ModernBERT's local layers) on ragged batches; rows of
    padding tiles must stay finite."""
    g = torch.Generator(device=dev).manual_seed(b * 100 + s + window)
    qkv = torch.randn(b * s, 3 * heads * 64, device=dev, generator=g).to(h16)
    mask = torch.ones(b, s, dtype=torch.int64, device=dev)
    for r in range(1, b):
        mask[r, max(1, s - 90 * r):] = 0
    ctx = nv.attention_d64_window(qkv, mask, b, s, heads, window)
    q, k, v = qkv.float().view(b, s, 3, heads, 64).unbind(2)
    q, k, v = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    i = torch.arange(s, device=dev)
    vis = ((i[:, None] - i[None, :]).abs() <= window)[None, None] & (mask != 0)[:, None, None, :]
    scores = (q @ k.transpose(-1, -2) / 8.0).masked_fill(~vis, torch.finfo(torch.float32).min)
    ref = (torch.softmax(scores, -1) @ v).permute(0, 2, 1, 3).reshape(b * s, heads * 64)
    valid = mask.bool().view(-1)
    assert torch.isfinite(ctx.float()).all()
    close(ctx.float()[valid], ref[valid], h16, 2.0)


# ------------------------------------------------------------------------- profiling instantiations
def test_profiling_instantiations_write_timelines_and_change_no_result(dev):
    """The clock64 timelines live in separate instantiations (attention: variant bit 8; bias GEMM: selected while a
    clock buffer is set): they must fill their buffers and give the production kernels' results bit for bit."""
    import ctypes

    lib = nv.load('bf16')
    lib.b2e_debug_set_att3_variant.argtypes = [ctypes.c_int]
    lib.b2e_debug_set_att3_clock.argtypes = [ctypes.c_void_p]
    lib.b2e_debug_set_clock_buffer.argtypes = [ctypes.c_void_p]
    g = torch.Generator(device=dev).manual_seed(11)
    b, s, heads = 6, 512, 4
    qkv = torch.randn(b * s, 3 * heads * 64, device=dev, generator=g).to(torch.bfloat16)
    mask = torch.ones(b, s, dtype=torch.int64, device=dev)
    try:
        for plain, timed in ((65, 321), (5, 261)):
            lib.b2e_debug_set_att3_variant(plain)
            want = nv.attention_d64(qkv, mask, b, s, heads).clone()
            buf = torch.zeros(4 * 512, dtype=torch.int64, device=dev)
            assert lib.b2e_debug_set_att3_clock(buf.data_ptr()) == 0
            nv.attention_d64(qkv, mask, b, s, heads)          # production kernel: no stamps even with a buffer set
            torch.cuda.synchronize()
            assert int((buf != 0).sum()) == 0
            lib.b2e_debug_set_att3_variant(timed)
            got = nv.attention_d64(qkv, mask, b, s, heads).clone()
            torch.cuda.synchronize()
            assert lib.b2e_debug_set_att3_clock(None) == 0
            assert torch.equal(got, want)
            assert int((buf.view(4, 2, 256)[0, 0] != 0).sum()) > 8   # the first softmax role recorded its chunks
    finally:
        lib.b2e_debug_set_att3_clock(None)
        lib.b2e_debug_set_att3_variant(-1)
    # bias GEMM
    a = (torch.randn(4096, 768, device=dev, generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(768, 768, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(768, device=dev, generator=g)
    want = nv.gemm_h16(a, w, bias).clone()
    buf = torch.zeros(4 * 256, dtype=torch.int64, device=dev)
    try:
        assert lib.b2e_debug_set_clock_buffer(buf.data_ptr()) == 0
        got = nv.gemm_h16(a, w, bias).clone()
        torch.cuda.synchronize()
    finally:
        assert lib.b2e_debug_set_clock_buffer(None) == 0
    assert torch.equal(got, want) and int((buf != 0).sum()) > 8
    buf.zero_()
    nv.gemm_h16(a, w, bias)
    torch.cuda.synchronize()
    assert int((buf != 0).sum()) == 0
