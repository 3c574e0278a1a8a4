"""-m gpu: the squared-L2 search (b2e_topk_l2, the CUDA-core scan, and b2e_topk_l2_tc, the TF32 scan with the
exact fp32 decision) on inputs whose arithmetic is exact (oracle/exact.py), compared with tools/oracle_l2.py's
topk_l2 BIT FOR BIT -- distances and row ids, the +inf / -1 tail included -- and the faiss_index_v1 retriever
end to end.  The contract (include/b2e.h): ascending squared distance, equal distances by ascending row id."""

from __future__ import annotations

import json

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from oracle import exact
from oracle import search as osearch
from tools import oracle_l2 as ol2

pytestmark = pytest.mark.gpu

BIG = 1 << 31
SCANS = ['fma', 'tc']


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def reference(queries, corpus, k):
    """(distances [Q, k] f32, indices [Q, k] i64) of the oracle, padded with +inf / -1 past min(k, N)."""
    if corpus.shape[0] * corpus.shape[1] <= 1 << 22:
        d, i = ol2.numpy_reference(queries, corpus, k)
    else:   # the same computation in float64 on the device
        d, i = ol2.topk_l2_torch(queries, corpus, k)
    d, i = d.cpu(), i.cpu()
    q, kk = d.shape
    out_d = torch.full((q, k), float('inf'), dtype=torch.float32)
    out_i = torch.full((q, k), -1, dtype=torch.int64)
    out_d[:, :kk], out_i[:, :kk] = d + 0.0, i
    return out_d, out_i


def assert_same(got, ref, what=''):
    gd, gi = (t.cpu() for t in got)
    rd, ri = ref
    assert gd.shape == rd.shape and gi.shape == ri.shape, (gd.shape, rd.shape)
    bad = (gi != ri) | (gd.view(torch.int32) != rd.view(torch.int32))
    if bad.any():
        q, p = (int(x) for x in bad.nonzero()[0])
        raise AssertionError(f'{what}: query {q} place {p}: got index {int(gi[q, p])} distance {float(gd[q, p])}, '
                             f'oracle index {int(ri[q, p])} distance {float(rd[q, p])} '
                             f'({int(bad.sum())} places differ)')


def run(scan, queries, corpus, k):
    """'fma' = b2e_topk_l2 (CUDA cores), 'tc' = b2e_topk_l2_tc on the norms built as an index builds them."""
    if scan == 'tc':
        norms, max_norm = nv.row_norms(corpus)
        return nv.topk_l2(queries, corpus, k, norms=norms, max_norm=max_norm * 1.0001)
    return nv.topk_l2(queries, corpus, k)


def pad_cols(x, h):
    return torch.nn.functional.pad(x, (0, h - x.shape[1])).contiguous() if x.shape[1] < h else x


def test_row_norms_are_the_squared_norms_and_their_maximum(dev):
    g = torch.Generator(device=dev).manual_seed(1)
    x = exact.int_matrix(5000, 768, 8, g)
    norms, m = nv.row_norms(x)
    ref = (x.double() ** 2).sum(dim=1)
    assert torch.equal(norms.double(), ref) and m == float(ref.max().sqrt().float())
    assert nv.max_row_norm(x) == m


# --------------------------------------------------------------------------------------------- shapes
# entries in {-1, 0, 1}: thousands of rows share every distance, so every place of the answer is a tie
SHAPES = [
    (1, 1, 1, 128), (4, 2, 1, 256), (5, 100, 99, 768), (16, 255, 254, 128), (17, 256, 255, 960),
    (64, 100, 100, 128), (1, 256, 256, 4096), (5, 10, 3, 960), (33, 256, 257, 768), (64, 1, 2, 128),
    (1, 100, 32_767, 256), (5, 256, 32_768, 768), (17, 2, 32_767, 128), (4, 255, 32_768, 960),
    (33, 1, 32_768, 256), (16, 100, 100_003, 768), (1, 255, 100_003, 128), (5, 1, 100_003, 960),
    (64, 256, 100_003, 128), (4, 2, 100_003, 4096), (17, 100, 40_000, 4096), (64, 10, 40_000, 960),
]


@pytest.mark.parametrize('scan', SCANS)
@pytest.mark.parametrize('q,k,n,h', SHAPES)
def test_l2_shapes_with_ties_everywhere(dev, q, k, n, h, scan):
    g = torch.Generator(device=dev).manual_seed(q * 7919 + k * 31 + n + h)
    corpus = exact.int_matrix(n, h, 1, g)
    queries = exact.int_matrix(q, h, 1, g)
    if n % 2:   # the same values times a power of two are just as exact
        queries *= 2.0 ** -3
        corpus *= 2.0 ** -3
    ref = reference(queries, corpus, k)
    hp = -(-h // 128) * 128     # 960 -> 1024 zero columns, as the index pads them: (0 - 0)^2 adds nothing
    assert_same(run(scan, pad_cols(queries, hp), pad_cols(corpus, hp), k), ref, f'{scan} Q={q} k={k} N={n} H={h}')


# ------------------------------------------------------------------------------------- planted ties
def tie_positions(pattern, q, n, sms):
    """Rows tied at the k-th place for each of q queries: inside one row group of the scans, one warp apart, in
    a late CTA of the first grid-stride sweep and CTA 0 of a later one (the higher id reached first), several."""
    sweep = 2 * sms * 64
    out = []
    for qi in range(q):
        a = 64 * (3 + 11 * qi)
        far_lo = sweep - 64 * (1 + qi) + 5
        far_hi = 2 * sweep + 8 * qi + 3
        out.append({'row_group': [a + 1, a + 2],
                    'warp4': [a + 5, a + 1],
                    'warp8': [a + 11, a + 3],
                    'far': [far_hi, far_lo],
                    'several': [a + 3, a + 2, far_hi, a + 1, a + 9]}[pattern])
    flat = [r for rows in out for r in rows]
    assert len(set(flat)) == len(flat) and max(flat) < n
    return out


PATTERNS = ['row_group', 'warp4', 'warp8', 'far', 'several']
QS = [1, 4, 5, 16, 17, 33]
KS = [1, 2, 100, 255, 256]


@pytest.mark.parametrize('scan', SCANS)
@pytest.mark.parametrize('q', QS)
@pytest.mark.parametrize('pattern', PATTERNS)
def test_l2_ties_at_the_kth_place_go_to_the_lowest_row_id(dev, sms, pattern, q, scan):
    k = KS[(PATTERNS.index(pattern) + QS.index(q)) % len(KS)]
    n, h = 100_003, 256
    g = torch.Generator(device=dev).manual_seed(1000 * q + k)
    queries = exact.int_matrix(q, h, 8, g)
    corpus = exact.int_matrix(n, h, 4, g)
    rows = tie_positions(pattern, q, n, sms)
    ol2.planted_ties(queries, corpus, k, rows, g, permute=(q % 2 == 1))
    dist = ol2.l2_matrix(queries, corpus)
    for qi in range(q):   # the case is what it claims
        assert int((dist[qi] < 15).sum()) == k - 1 and int((dist[qi] == 15).sum()) == len(rows[qi])
    got = run(scan, queries, corpus, k)
    if scan == 'tc':   # planted rows far closer than the background: the tensor-core decision itself is tested
        assert not nv.topk_tc_fell_back()
    ref = reference(queries, corpus, k)
    assert ref[1][:, -1].tolist() == [min(r) for r in rows]
    assert_same(got, ref, f'{scan} {pattern} Q={q} k={k}')


@pytest.mark.parametrize('scan', SCANS)
@pytest.mark.parametrize('q,k,n', [(1, 1, 40_000), (1, 256, 100_003), (5, 100, 40_000), (17, 256, 40_000)])
def test_l2_all_zero_query_returns_the_rows_of_smallest_norm(dev, q, k, n, scan):
    g = torch.Generator(device=dev).manual_seed(n + k)
    corpus = exact.int_matrix(n, 768, 2, g)
    queries = exact.int_matrix(q, 768, 8, g)
    queries[q // 2] = 0
    got = run(scan, queries, corpus, k)
    norms = (corpus.double() ** 2).sum(dim=1).cpu()
    order = torch.sort(norms, stable=True).indices[:k]
    assert got[1][q // 2].cpu().tolist() == order.tolist()
    assert got[0][q // 2].cpu().double().tolist() == norms[order].tolist()
    assert_same(got, reference(queries, corpus, k), scan)


@pytest.mark.parametrize('q,k', [(3, 10), (17, 256)])
def test_l2_tensor_core_scan_falls_back_on_duplicates_and_stays_exact(dev, q, k):
    """48 000 rows, 8 distinct: thousands tie with the k-th nearest, the candidate list overflows, and the exact
    scan must name the lowest ids among the duplicates -- the same answer as the direct CUDA-core call."""
    g = torch.Generator(device=dev).manual_seed(q)
    corpus = exact.int_matrix(8, 768, 8, g).repeat(6000, 1).contiguous()
    queries = exact.int_matrix(q, 768, 8, g)
    ref = reference(queries, corpus, k)
    got = run('tc', queries, corpus, k)
    assert nv.topk_tc_fell_back()
    assert_same(got, ref, 'tc')
    assert_same(run('fma', queries, corpus, k), ref, 'fma')


# ------------------------------------------------------------------------------------ past 2^31 elements
def need_free(gib: float):
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2**30:
        pytest.skip(f'needs {gib:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free')


def test_l2_float32_corpus_past_2_31_elements(dev):
    """2^22 + 129 rows x 512 (8.6 GB): every query's closer rows and tied rows lie beyond element 2^31.  The
    narrow (Q <= 4) and wide CUDA-core scans and the tensor-core scan all return the oracle's answer."""
    need_free(10.5)
    n, h, k = (1 << 22) + 129, 512, 6
    g = torch.Generator(device=dev).manual_seed(31)
    corpus = exact.int_matrix(n, h, 4, g)
    queries = exact.int_matrix(6, h, 8, g)
    top = 1 << 22
    assert top * h == BIG
    rows = [[top + 1, top + 2], [top + 7, top + 3], [top + 40, top + 39, top + 38], [top + 128, top + 64],
            [top + 90, top + 89], [top + 100, top + 127]]
    corpus[top:] = 8    # far from every query, and no closer ones below 2^31 either
    ol2.planted_ties(queries, corpus[top:], k, [[r - top for r in rr] for rr in rows], g)
    for queries_now in (queries[:3], queries):   # narrow scan, then the wide one
        ref = reference(queries_now, corpus, k)
        assert (ref[1] >= top).all() and ref[1][:, -1].tolist() == [min(r) for r in rows[:len(queries_now)]]
        assert_same(run('fma', queries_now, corpus, k), ref, f'fma Q={len(queries_now)}')
    got = run('tc', queries, corpus, k)
    assert not nv.topk_tc_fell_back()
    assert_same(got, ref, 'tc')
    del corpus, got
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------ real-valued embeddings
def test_l2_scans_agree_on_normalised_float_embeddings(dev):
    """1 M normalised float rows x 768: the two scans return the same distances and row ids bit for bit (the
    contract of b2e_topk_l2_tc, include/b2e.h), and the tensor-core search never needs its fallback."""
    n, h = 1_000_000, 768
    g = torch.Generator(device=dev).manual_seed(7)
    corpus = torch.randn(n, h, device=dev, generator=g)
    corpus /= corpus.norm(dim=1, keepdim=True)
    for q, k in [(1, 10), (4, 100), (16, 10), (64, 256)]:
        queries = torch.randn(q, h, device=dev, generator=g)
        queries /= queries.norm(dim=1, keepdim=True)
        fd, fi = run('fma', queries, corpus, k)
        td, ti = run('tc', queries, corpus, k)
        assert not nv.topk_tc_fell_back()
        assert torch.equal(td, fd) and torch.equal(ti, fi), (q, k)
        assert bool((fd[:, 1:] >= fd[:, :-1]).all())
    del corpus
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize('metric', ['l2', 'inner_product'])
def test_faiss_index_v1_retriever_end_to_end(tmp_path, metric):
    """A tiny BERT checkpoint -> embedding_worker -> huggingface writer (text + fp32 embeddings) -> a
    faiss_index_v1 RetrieverConfig -> search returns the oracle's rows, get_texts their text."""
    from distllm_b200.distributed_embedding import embedding_worker
    from distllm_b200.rag.search import FaissIndexV1
    from distllm_b200.rag.search import RetrieverConfig
    from distllm_b200.registry import registry
    from oracle.make_golden import tiny_bert_texts
    from oracle.make_golden import write_tiny_bert_checkpoint

    write_tiny_bert_checkpoint(tmp_path / 'ckpt')
    texts = tiny_bert_texts()
    (tmp_path / 'texts.jsonl').write_text('\n'.join(json.dumps({'text': t}) for t in texts) + '\n')
    enc = {'name': 'auto', 'pretrained_model_name_or_path': str(tmp_path / 'ckpt'), 'half_precision': False,
           'quantization': False}
    embedding_worker(tmp_path / 'texts.jsonl', tmp_path / 'out',
                     dataset_kwargs={'name': 'jsonl', 'batch_size': 4, 'num_data_workers': 0, 'pin_memory': False},
                     encoder_kwargs=enc, pooler_kwargs={'name': 'mean'},
                     embedder_kwargs={'name': 'full_sequence'}, writer_kwargs={'name': 'huggingface'})
    (ds_dir,) = [p for p in (tmp_path / 'out').iterdir() if p.is_dir()]
    cfg = RetrieverConfig(faiss_config={'name': 'faiss_index_v1', 'dataset_dir': str(ds_dir), 'metric': metric},
                          encoder_config=enc, pooler_config={'name': 'mean'}, batch_size=3)
    retriever = cfg.get_retriever()
    assert isinstance(retriever.faiss_index, FaissIndexV1)
    assert retriever.faiss_index.dataset.column_names[:2] == ['text', 'embeddings']
    emb = retriever.get_embeddings(list(range(len(texts)))).astype(np.float32)
    assert emb.shape == (len(texts), 256)
    queries = [texts[3], texts[10] + ' ' + texts[0], 'protein folding']
    k = 5
    res, q_emb = retriever.search(queries, top_k=k)
    if metric == 'l2':   # queries as pooled, not normalised
        assert not np.allclose(np.linalg.norm(q_emb, axis=1), 1.0)
        ref_s, ref_i = ol2.topk_l2(q_emb, emb, k)
    else:
        assert np.allclose(np.linalg.norm(q_emb, axis=1), 1.0, atol=1e-6)
        ref_s, ref_i = osearch.topk_inner_product(q_emb, emb, k)
    assert np.array(res.total_indices).tolist() == ref_i.tolist()
    np.testing.assert_allclose(np.array(res.total_scores), ref_s, rtol=1e-5, atol=1e-4)
    for row in res.total_indices:
        assert retriever.get_texts(row) == [texts[i] for i in row]
    # a threshold at the third result keeps the first three: distances <= it (l2), scores >= it (inner product)
    cut = res.total_scores[1][2]
    kept, _ = retriever.search(queries, top_k=k, score_threshold=cut)
    assert kept.total_indices[1] == res.total_indices[1][:3]
    registry.clear()
