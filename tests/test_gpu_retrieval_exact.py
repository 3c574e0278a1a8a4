"""-m gpu: the retrieval kernels on inputs whose arithmetic is exact (oracle/exact.py), compared with the
reference BIT FOR BIT -- scores and row ids, the -inf / -1 tail included.

A retriever's answer is which rows come back and in what order, so ties matter: the same chunk stored twice
has two identical embeddings and bit-identical scores.  The contract (include/b2e.h, oracle/search.py) is
descending score, equal scores by ascending row id; for ubinary, equal rescored scores keep the candidate
order (Hamming distance, then id).  The cases plant ties at the k-th place where each scan's visiting order
differs from index order: inside one 4-row group of the wide CUDA-core scan (rows are offered 0, 2, 1, 3),
one warp apart, in different CTAs and grid-stride sweeps with the higher id reached first, several rows where
only one fits, and distinct vectors with equal dot products."""

from __future__ import annotations

import pytest
import torch

from distllm_b200 import _native as nv
from oracle import exact

pytestmark = pytest.mark.gpu

BIG = 1 << 31


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def reference(queries, corpus, k):
    """(scores [Q, k] f32, indices [Q, k] i64) of oracle/search.py, padded with -inf / -1 past min(k, N)."""
    if corpus.shape[0] * corpus.shape[1] <= 1 << 22:
        s, i = exact.numpy_reference(queries, corpus, k)
    else:   # the same computation in float64 on the device
        s, i = exact.topk_inner_product(queries, corpus, k)
    return pad(s.cpu(), i.cpu(), k)


def pad(s, i, k):
    q, kk = s.shape
    out_s = torch.full((q, k), -float('inf'), dtype=torch.float32)
    out_i = torch.full((q, k), -1, dtype=torch.int64)
    out_s[:, :kk], out_i[:, :kk] = s + 0.0, i   # + 0.0: a zero score is +0, as the kernels' sums give it
    return out_s, out_i


def assert_same(got, ref, what=''):
    """Scores and indices equal bit for bit; on failure name the first differing (query, place)."""
    gs, gi = (t.cpu() for t in got)
    rs, ri = ref
    assert gs.shape == rs.shape and gi.shape == ri.shape, (gs.shape, rs.shape)
    bad = (gi != ri) | (gs.view(torch.int32) != rs.view(torch.int32))
    if bad.any():
        q, p = (int(x) for x in bad.nonzero()[0])
        raise AssertionError(f'{what}: query {q} place {p}: got index {int(gi[q, p])} score {float(gs[q, p])}, '
                             f'oracle index {int(ri[q, p])} score {float(rs[q, p])} '
                             f'({int(bad.sum())} places differ)')


def run(scan, queries, corpus, k):
    """scan: 'f32' / 'bf16' = b2e_topk_ip on that corpus type, 'tc' = b2e_topk_ip_tc (float32 corpus)."""
    if scan == 'tc':
        return nv.topk_ip(queries, corpus, k, max_norm=nv.max_row_norm(corpus))
    return nv.topk_ip(queries, corpus.to(torch.bfloat16) if scan == 'bf16' else corpus, k)


def int_queries(q, h, g, lead_one=True):
    queries = exact.int_matrix(q, h, 8, g)
    if lead_one:
        queries[:, 0] = 1
    return queries


def tie_positions(pattern, q, n, sms):
    """Rows tied at the k-th place for each of q queries (lists of distinct rows, all < n)."""
    sweep = 2 * sms * 64                     # rows one grid-stride sweep of the narrow scan covers
    out = []
    for qi in range(q):
        a = 64 * (3 + 11 * qi)               # a 4-row (and 8-row) aligned anchor per query
        far_lo = sweep - 64 * (1 + qi) + 5   # a late CTA of the first sweep ...
        far_hi = 2 * sweep + 8 * qi + 3      # ... and CTA 0 of a later sweep: the higher id is reached first
        rows = {'row_group': [a + 1, a + 2],
                'warp4': [a + 5, a + 1],
                'warp8': [a + 11, a + 3],
                'far': [far_hi, far_lo],
                'several': [a + 3, a + 2, far_hi, a + 1, a + 9],
                'equal_dot': [a + 2, a + 1, a + 6]}[pattern]
        out.append(rows)
    flat = [r for rows in out for r in rows]
    assert len(set(flat)) == len(flat) and max(flat) < n
    return out


def tie_case(q, n, h, k, pattern, seed, sms, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    queries = int_queries(q, h, g)
    corpus = exact.int_matrix(n, h, 4, g)
    rows = tie_positions(pattern, q, n, sms)
    exact.planted_ties(queries, corpus, k, rows, g, equal_dot=(pattern == 'equal_dot'))
    # the case is what it claims: k - 1 rows strictly better, every planted row tied at the k-th place
    s = exact.score_matrix(queries, corpus)
    for qi in range(q):
        t = float(queries[qi].double() @ queries[qi].double()) - 1
        assert int((s[qi] > t).sum()) == k - 1 and int((s[qi] == t).sum()) == len(rows[qi])
    return queries, corpus, rows


PATTERNS = ['row_group', 'warp4', 'warp8', 'far', 'several', 'equal_dot']
QS = [1, 4, 5, 16, 17, 33]
KS = [1, 2, 100, 255, 256]


@pytest.mark.parametrize('scan', ['f32', 'bf16', 'tc'])
@pytest.mark.parametrize('q', QS)
@pytest.mark.parametrize('pattern', PATTERNS)
def test_topk_ties_at_the_kth_place_go_to_the_lowest_row_id(dev, sms, pattern, q, scan):
    k = KS[(PATTERNS.index(pattern) + QS.index(q)) % len(KS)]
    n, h = 100_003, 256
    queries, corpus, rows = tie_case(q, n, h, k, pattern, 1000 * q + k, sms, dev)
    got = run(scan, queries, corpus, k)
    if scan == 'tc':   # planted rows far above the background: the tensor-core decision itself is tested
        assert not nv.topk_tc_fell_back()
    ref = reference(queries, corpus, k)
    assert ref[1][:, -1].tolist() == [min(r) for r in rows]
    assert_same(got, ref, f'{scan} {pattern} Q={q} k={k}')


@pytest.mark.parametrize('scan', ['f32', 'bf16'])
def test_wide_scan_tie_inside_one_row_group(dev, scan):
    """5 queries (the 16-query scan), k = 1, rows 1 and 2 identical and best: the answer is row 1."""
    g = torch.Generator(device=dev).manual_seed(3)
    corpus = exact.int_matrix(1000, 256, 2, g)
    queries = int_queries(5, 256, g)
    corpus[1] = corpus[2] = 8 * torch.sign(queries[0])
    queries[1:] = queries[0]
    got = run(scan, queries, corpus, 1)
    assert got[1].cpu().flatten().tolist() == [1] * 5
    assert_same(got, reference(queries, corpus, 1), scan)


# --------------------------------------------------------------------------------------------- shapes
# entries in {-1, 0, 1}: thousands of rows share every score, so every place of the answer is a tie
SHAPES = [
    (1, 1, 1, 128), (4, 2, 1, 256), (5, 100, 99, 768), (16, 255, 254, 128), (17, 256, 255, 256),
    (33, 100, 100, 128), (1, 256, 256, 768), (5, 2, 3, 8192), (4, 255, 256, 256), (33, 256, 257, 768),
    (16, 1, 2, 128), (17, 2, 2, 256), (5, 256, 257, 8192), (1, 100, 32_767, 256), (5, 256, 32_768, 768),
    (17, 2, 32_767, 128), (4, 255, 32_768, 256), (33, 1, 32_768, 256), (16, 100, 100_003, 768),
    (1, 255, 100_003, 128), (5, 1, 100_003, 256), (33, 256, 100_003, 128), (4, 2, 100_003, 768),
    (17, 100, 32_768, 8192), (4, 256, 32_767, 8192), (1, 2, 32_768, 8192),
]


@pytest.mark.parametrize('scan', ['f32', 'bf16', 'tc'])
@pytest.mark.parametrize('q,k,n,h', SHAPES)
def test_topk_shapes_with_ties_everywhere(dev, q, k, n, h, scan):
    if scan == 'bf16' and h % 256:
        pytest.skip('a bfloat16 corpus needs H % 256 == 0')
    g = torch.Generator(device=dev).manual_seed(q * 7919 + k * 31 + n + h)
    corpus = exact.int_matrix(n, h, 1, g)
    queries = exact.int_matrix(q, h, 1, g)
    if n % 2:   # the same values times a power of two are just as exact
        queries *= 2.0 ** -4
        corpus *= 2.0 ** -3
    assert_same(run(scan, queries, corpus, k), reference(queries, corpus, k), f'{scan} Q={q} k={k} N={n} H={h}')


@pytest.mark.parametrize('scan', ['f32', 'bf16', 'tc'])
@pytest.mark.parametrize('q,k,n', [(1, 1, 40_000), (1, 256, 100_003), (5, 100, 40_000), (17, 256, 40_000)])
def test_topk_all_zero_query_returns_the_first_k_rows(dev, q, k, n, scan):
    g = torch.Generator(device=dev).manual_seed(n + k)
    corpus = exact.int_matrix(n, 768, 8, g)
    queries = int_queries(q, 768, g)
    queries[q // 2] = 0
    got = run(scan, queries, corpus, k)
    if scan == 'tc':   # every score ties: the candidate list cannot hold them, the exact scan redoes the call
        assert nv.topk_tc_fell_back()
    assert got[1][q // 2].tolist() == list(range(k)) and not got[0][q // 2].any()
    assert_same(got, reference(queries, corpus, k), scan)


@pytest.mark.parametrize('q,k', [(3, 10), (17, 256)])
def test_topk_tensor_core_scan_falls_back_on_duplicates_and_stays_exact(dev, q, k):
    """48 000 rows, 8 distinct: thousands tie with the k-th best, the candidate list overflows, and the exact
    scan must name the lowest ids among the duplicates -- the same answer as the direct CUDA-core call."""
    g = torch.Generator(device=dev).manual_seed(q)
    corpus = exact.int_matrix(8, 768, 8, g).repeat(6000, 1).contiguous()
    queries = int_queries(q, 768, g, lead_one=False)
    ref = reference(queries, corpus, k)
    got = run('tc', queries, corpus, k)
    assert nv.topk_tc_fell_back()
    assert_same(got, ref, 'tc')
    assert_same(run('f32', queries, corpus, k), ref, 'f32')


# ------------------------------------------------------------------------------------------- ubinary
def ubinary_case(q, n, h, k, mult, g):
    """Integer queries; around each query's sign pattern, rows at Hamming distance 0..3 whose flips fall on a
    few positions, so that distances tie, rescored scores tie between different candidates (a flip where
    q == 0 changes the distance, not the score), and duplicates occur."""
    queries = exact.int_matrix(q, h, 8, g)
    corpus = exact.int_matrix(n, h, 8, g)
    cpu = torch.Generator().manual_seed(int(torch.randint(0, 2**31, (1,), generator=g, device=g.device)))
    per = min(n // max(q, 1), 2 * k * mult)
    slots = torch.randperm(n, generator=cpu)[:per * q].view(q, per) if per else torch.empty(q, 0, dtype=torch.long)
    for qi in range(q):
        qv = queries[qi].cpu()
        pool = torch.cat([(qv == 0).nonzero().flatten()[:3], (qv == 3).nonzero().flatten()[:3],
                          (qv == -3).nonzero().flatten()[:2]])
        for r in slots[qi].tolist():
            row = qv.clone()
            for p in pool[torch.randperm(len(pool), generator=cpu)[:int(torch.randint(0, 4, (1,), generator=cpu))]]:
                row[p] = -1.0 if row[p] > 0 else 1.0      # flip the packed bit
            corpus[r] = row.to(corpus.device)
    return queries, corpus


@pytest.mark.parametrize('q,n,h,k,mult', [(1, 5000, 256, 10, 2), (5, 40_000, 768, 100, 2), (9, 20_000, 256, 1, 4),
                                          (17, 3000, 1280, 50, 1), (2, 3, 256, 4, 2), (3, 8, 768, 10, 1),
                                          (8, 100_003, 8192, 20, 3)])
def test_ubinary_search_is_exact_with_ties(dev, q, n, h, k, mult):
    g = torch.Generator(device=dev).manual_seed(n + h + k)
    queries, corpus = ubinary_case(q, n, h, k, mult, g)
    bits = nv.pack_ubinary(corpus)
    assert torch.equal(bits, exact.pack_bits(corpus))
    got = nv.search_ubinary(queries, bits, k, mult)
    if n * h <= 1 << 22:
        from oracle import search as osearch

        s, i = osearch.search_ubinary(queries.cpu().numpy(), bits.cpu().numpy(), k, mult)
        ref = pad(torch.from_numpy(s), torch.from_numpy(i).to(torch.int64), k)
    else:
        s, i = exact.search_ubinary(queries, bits, k, mult)
        ref = pad(s.cpu(), i.cpu(), k)
    assert_same(got, ref, f'ubinary Q={q} N={n}')


def test_ubinary_candidate_overflow_is_flagged(dev):
    """5000 rows tie at distance 0 for query 0 (more than the candidate buffer): its row is NaN / -2 and
    ExactIndex raises; query 1, in the same call, is unaffected and exact."""
    from distllm_b200.rag.search import ExactIndex
    from distllm_b200.rag.search import ExactIndexConfig

    g = torch.Generator(device=dev).manual_seed(11)
    queries = exact.int_matrix(2, 256, 8, g)
    corpus = exact.int_matrix(20_000, 256, 8, g)
    corpus[3000:8000] = queries[0]
    corpus[100:110] = queries[1]
    bits = nv.pack_ubinary(corpus)
    s, i = nv.search_ubinary(queries, bits, 5, 2)
    assert torch.isnan(s[0]).all() and (i[0] == -2).all()
    rs, ri = exact.search_ubinary(queries[1:], bits, 5, 2)
    assert_same((s[1:], i[1:]), pad(rs.cpu(), ri.cpu(), 5), 'query 1')
    index = ExactIndex(corpus.cpu().numpy(), config=ExactIndexConfig(precision='ubinary', rescore_multiplier=2))
    with pytest.raises(nv.NativeError, match='candidate buffer'):
        index.search(queries.cpu().numpy(), top_k=5)


# ---------------------------------------------------------------------------------------- ExactIndex
@pytest.mark.parametrize('precision,corpus_dtype,n', [('float32', 'float32', 32_767), ('float32', 'float32', 32_768),
                                                      ('float32', 'bfloat16', 40_000), ('ubinary', 'float32', 40_000)])
def test_exact_index_search_returns_the_oracle_answer(dev, sms, precision, corpus_dtype, n):
    from distllm_b200.rag.search import ExactIndex
    from distllm_b200.rag.search import ExactIndexConfig

    q, h, k = 6, 256, 20
    if precision == 'ubinary':
        g = torch.Generator(device=dev).manual_seed(5)
        queries, corpus = ubinary_case(q, n, h, k, 2, g)
        bits = exact.pack_bits(corpus)
        rs, ri = exact.search_ubinary(queries, bits, k, 2)
    else:
        queries, corpus, _ = tie_case(q, n, h, k, 'equal_dot', 17, sms, dev)
        rs, ri = reference(queries, corpus.to(torch.bfloat16) if corpus_dtype == 'bfloat16' else corpus, k)
    index = ExactIndex(corpus.cpu().numpy(), config=ExactIndexConfig(precision=precision, corpus_dtype=corpus_dtype))
    res = index.search(queries.cpu().numpy(), top_k=k)
    if precision == 'float32' and corpus_dtype == 'float32' and n >= 32_768:
        assert index.max_norm is not None and not nv.topk_tc_fell_back()
    assert res.total_indices == ri.tolist()
    assert res.total_scores == rs.tolist()


# ------------------------------------------------------------------------------------ past 2^31 elements
def need_free(gib: float):
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2**30:
        pytest.skip(f'needs {gib:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free')


def test_float32_corpus_past_2_31_elements(dev):
    """2^22 + 129 rows x 512 (8.6 GB): every query's better rows and tied rows lie beyond element 2^31.  The
    narrow (Q <= 4) and wide CUDA-core scans and the tensor-core scan all return the oracle's answer."""
    need_free(10.5)
    n, h, k = (1 << 22) + 129, 512, 6
    g = torch.Generator(device=dev).manual_seed(31)
    corpus = exact.int_matrix(n, h, 4, g)
    queries = int_queries(6, h, g)
    top = 1 << 22
    assert top * h == BIG
    rows = [[top + 1, top + 2], [top + 7, top + 3], [top + 40, top + 39, top + 38], [top + 128, top + 64],
            [top + 90, top + 89], [top + 100, top + 127]]
    corpus[top:] = 0
    exact.planted_ties(queries, corpus[top:], k, [[r - top for r in rr] for rr in rows], g)
    for queries_now in (queries[:3], queries):   # narrow scan, then the wide one
        ref = reference(queries_now, corpus, k)
        assert (ref[1] >= top).all() and ref[1][:, -1].tolist() == [min(r) for r in rows[:len(queries_now)]]
        assert_same(run('f32', queries_now, corpus, k), ref, f'f32 Q={len(queries_now)}')
    got = run('tc', queries, corpus, k)
    assert not nv.topk_tc_fell_back()
    assert_same(got, ref, 'tc')
    del corpus, got
    torch.cuda.empty_cache()


def test_bfloat16_corpus_past_2_31_elements(dev):
    """2^23 + 3 rows x 256 bfloat16 (4.3 GB): the three best rows are the last three, beyond element 2^31;
    rows 2^23 + 1 and 2^23 + 2 are identical and tie at k = 2 (the 4-row group trap of the wide scan)."""
    need_free(6.5)
    n, h, top = (1 << 23) + 3, 256, 1 << 23
    assert top * h == BIG
    g = torch.Generator(device=dev).manual_seed(23)
    corpus = torch.empty((n, h), dtype=torch.bfloat16, device=dev)
    step = 1 << 20
    for lo in range(0, n, step):
        corpus[lo:lo + step] = exact.int_matrix(min(step, n - lo), h, 4, g).to(torch.bfloat16)
    q0 = int_queries(1, h, g)[0]
    row = exact.base_row(q0)
    corpus[top] = (row + torch.eye(h, device=dev)[0]).to(torch.bfloat16)   # scores one more than the tie
    corpus[top + 1] = corpus[top + 2] = row.to(torch.bfloat16)
    for q in (2, 5):
        queries = q0.repeat(q, 1).contiguous()
        ref = reference(queries, corpus, 2)
        assert ref[1].tolist() == [[top, top + 1]] * q
        assert_same(nv.topk_ip(queries, corpus, 2), ref, f'bf16 Q={q}')
    del corpus
    torch.cuda.empty_cache()


def test_ubinary_corpus_past_2_31_bytes(dev):
    """2^24 + 8 packed rows x 128 bytes (2.1 GB) generated directly as bits; the 8 candidates (k = 4, multiplier
    2) are the last 8 rows, with tied distances and tied rescored scores among them."""
    need_free(4.0)
    n, h, top = (1 << 24) + 8, 1024, 1 << 24
    assert top * (h // 8) == BIG
    g = torch.Generator(device=dev).manual_seed(24)
    bits = torch.empty((n, h // 8), dtype=torch.uint8, device=dev).random_(0, 256, generator=g)
    q = exact.int_matrix(1, h, 8, g)[0]
    zero, three = (q == 0).nonzero().flatten(), (q == 3).nonzero().flatten()
    rows = q.repeat(8, 1)
    rows[2, zero[0]] = 1.0                       # distance 1, same score as the query's own pattern
    rows[3, three[0]] = -1.0                     # distance 1, score - 3
    rows[4, three[1]] = -1.0                     # distance 1, score - 3 (a different row)
    rows[5, zero[1]] = 1.0
    rows[5, three[2]] = -1.0                     # distance 2, score - 3
    rows[6, zero[0]] = rows[6, zero[1]] = 1.0    # distance 2, same score as the query's pattern
    rows[7] = rows[4]                            # a duplicate of row 4
    bits[top:] = exact.pack_bits(rows)
    queries = torch.stack([q, 2 * q])
    rs, ri = exact.search_ubinary(queries, bits, 4, 2)
    assert (ri >= top).all()
    assert_same(nv.search_ubinary(queries, bits, 4, 2), (rs.cpu(), ri.cpu()), 'ubinary')
    del bits
    torch.cuda.empty_cache()
