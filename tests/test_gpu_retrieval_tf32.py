"""-m gpu: the TF32 tensor-core searches (b2e_topk_ip_tc, b2e_topk_l2_tc) on inputs the tensor cores round.

Their contract is the CUDA-core scans' results bit for bit.  That rests on a margin: the TF32 scan's error must
stay below eps, and the histogram, threshold and selection must keep every row that could reach the k-th place.
Inputs of small integers (test_gpu_retrieval_exact.py) never exercise it, so these tests read the last pass's
intermediate state through b2e_debug_topk_tc_state and hold it to oracle/tf32.py:
  (a) the premise: every scan score within the scan's share of the margin, and the conversion model identified;
  (b) every stage against its restatement: r and eps, the histogram, the threshold, the candidate set, and the
      soundness of what was left out;
  (c) corpora the TF32 scan ranks wrongly (oracle/tf32.py: adversarial) end to end, against the CUDA-core scans
      and the planted answer."""

from __future__ import annotations

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from oracle import exact
from oracle import tf32 as ot
from tools import oracle_l2 as ol2

pytestmark = pytest.mark.gpu

CHUNK = 1 << 14


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


def tc_search(metric, queries, corpus, k):
    """The tensor-core search with the norms and bound an index builds (FaissIndexV1): (result, norms, max_norm)"""
    norms, m = nv.row_norms(corpus)
    m *= 1.0001
    if metric == 'ip':
        return nv.topk_ip(queries, corpus, k, max_norm=m), norms, m
    return nv.topk_l2(queries, corpus, k, norms=norms, max_norm=m), norms, m


def cuda_core(metric, queries, corpus, k):
    return nv.topk_ip(queries, corpus, k) if metric == 'ip' else nv.topk_l2(queries, corpus, k)


def last_pass_state(n):
    return nv.topk_tc_state(-(-n // 128) * 128)


def inputs(kind, n, h, q, seed, dev):
    if kind == 'adversarial':
        p = ot.adversarial(n, h, q, min(4, ot.offsets(h, ot.TRUNC) - 3), ot.TRUNC, seed, device=dev)
        return p.queries, p.corpus
    g = torch.Generator(device=dev).manual_seed(seed)
    corpus = torch.randn(n, h, device=dev, generator=g)
    queries = torch.randn(q, h, device=dev, generator=g)
    if kind in ('normalised', 'spread'):
        corpus /= corpus.norm(dim=1, keepdim=True)
        queries /= queries.norm(dim=1, keepdim=True)
    if kind == 'spread':
        corpus *= 0.5 + 1.5 * torch.rand(n, 1, device=dev, generator=g)
    return queries, corpus.contiguous()


def matching_models(scan, queries, corpus, h):
    """The conversion models whose float64 sum of converted products every scan score [Q, N] matches within the
    accumulation allowance, and for each model the largest deviation / allowance."""
    out = {}
    for model in ot.MODELS:
        s, a = ot.tf32_scores(queries, corpus, model, CHUNK)
        out[model] = float(((scan - s).abs() / (ot.accumulation_allowance(h, a) + 1e-30)).max())
    return [m for m, v in out.items() if v <= 1.0], out


@pytest.fixture(scope='module')
def hw_model(dev):
    """The conversion the tensor cores apply, identified on an adversarial pattern at H = 768."""
    n, h, q = 40_000, 768, 16
    p = ot.adversarial(n, h, q, 16, ot.TRUNC, 99, device=dev)
    tc_search('ip', p.queries, p.corpus, 1)
    scan = torch.from_numpy(last_pass_state(n)['scores'][:n, :q]).to(dev, torch.float64).T
    models, dev_ratio = matching_models(scan, p.queries, p.corpus, h)
    print(f'\nTF32 conversion on this device: {models} (deviation / allowance {dev_ratio})')
    assert len(models) == 1, dev_ratio
    return models[0]


# ------------------------------------------------------------------------------------------ (a) premise
HS = [128, 768, 1024, 4096, 8192]
KINDS = ['normal', 'normalised', 'spread', 'adversarial']
NS = [32_768, 32_769, 100_003]
QS = [1, 5, 16]
PREMISE = [(h, kind, NS[(i + j) % 3], QS[(i + 2 * j) % 3]) for i, h in enumerate(HS) for j, kind in enumerate(KINDS)]


@pytest.mark.parametrize('h,kind,n,q', PREMISE)
def test_scan_error_is_within_its_share_of_the_margin(dev, hw_model, h, kind, n, q):
    """|S - q.x| <= 1.5 2^-9 r - (H / 32 + 5) 2^-24 sum |q_i x_i| for every row and query: the scan's share of eps,
    less what the fp32 rescore may itself be off.  The L2 search runs the same scan: its scores are the same bits."""
    queries, corpus = inputs(kind, n, h, q, 7 * h + n + q, dev)
    tc_search('ip', queries, corpus, 10)
    st = last_pass_state(n)
    tc_search('l2', queries, corpus, 10)
    st2 = last_pass_state(n)
    assert np.array_equal(st['scores'][:n, :q].view(np.uint32), st2['scores'][:n, :q].view(np.uint32))
    assert not st['scores'][n:].any()                    # rows past N: the TMA zero-fills them
    scan = torch.from_numpy(st['scores'][:n, :q]).to(dev, torch.float64).T
    ex = exact.score_matrix(queries, corpus, CHUNK)
    r = torch.from_numpy(st['meta']['r'][:q].astype(np.float64)).to(dev)[:, None]
    allowed = 1.5 * 2.0 ** -9 * r - ot.rescore_error(h, ot.abs_score_matrix(queries, corpus, CHUNK))
    err = (scan - ex).abs()
    ratio = float((err / (1.5 * 2.0 ** -9 * r)).max())
    print(f'\nH={h} {kind} N={n} Q={q}: largest |S - q.x| / eps = {ratio:.4f}')
    assert bool((err <= allowed).all()), ratio
    if kind == 'adversarial':
        models, dev_ratio = matching_models(scan, queries, corpus, h)
        print(f'H={h}: conversion {models}, deviation / allowance {dev_ratio}')
        assert models == [hw_model], dev_ratio


# ------------------------------------------------------------------------------------------ (b) stages
STAGES = [
    ('ip', 'normalised', 32_769, 768, 16, 10), ('ip', 'adversarial', 100_003, 1024, 5, 100),
    ('ip', 'spread', 32_768, 4096, 1, 256), ('ip', 'normal', 50_000, 128, 16, 1),
    ('l2', 'normalised', 32_769, 768, 16, 10), ('l2', 'adversarial', 100_003, 1024, 5, 100),
    ('l2', 'spread', 32_768, 4096, 1, 256), ('l2', 'normal', 50_000, 128, 16, 1),
    ('l2', 'far', 50_021, 768, 16, 100),
]


@pytest.mark.parametrize('metric,kind,n,h,q,k', STAGES)
def test_each_stage_matches_its_restatement(dev, metric, kind, n, h, q, k):
    if kind == 'far':
        p = ot.adversarial(n, h, q, k, ot.TRUNC, 5, device=dev, far_background=True)
        queries, corpus = p.queries, p.corpus
    else:
        queries, corpus = inputs(kind, n, h, q, n + h + k, dev)
    (_, idx), norms, m = tc_search(metric, queries, corpus, k)
    fell_back = nv.topk_tc_fell_back()
    assert not fell_back or kind == 'spread'   # one global norm bound may be too loose for spread-out norms
    st = last_pass_state(n)
    scores = st['scores'][:n]
    norm2 = norms.cpu().numpy()
    m32 = np.float32(m)
    shift = ot.shift_of(m32) if metric == 'l2' else np.float32(0.0)
    qn = queries.double().norm(dim=1).cpu().numpy()
    qn32 = np.sqrt((queries.double() ** 2).sum(dim=1).float().cpu().numpy())
    if metric == 'ip':
        ex = exact.score_matrix(queries, corpus, CHUNK)
        err = ot.rescore_error(h, ot.abs_score_matrix(queries, corpus, CHUNK))
    else:   # distances, negated so that larger is better on both metrics
        d = ol2.l2_matrix(queries, corpus, CHUNK)
        ex, err = -d, ot.rescore_error(h + 64, d)
    idx = idx.cpu().numpy()
    for qi in range(q):
        rec = st['meta'][qi]
        r, eps, thr, need = rec['r'], rec['eps'], rec['thr'], int(rec['need'])
        # r bounds every score; eps is the formula of r (L2: and of |q|, which the device sums in its own order)
        assert qn[qi] * float(m32) <= r <= qn[qi] * float(m32) * 1.001
        if metric == 'ip':
            assert abs(eps - ot.eps_ip(r)) <= np.spacing(eps)
        else:
            assert abs(eps - ot.eps_l2(r, qn32[qi], m32, h)) <= 4 * np.spacing(eps)
        # the histogram: of these N rows' values and nothing else
        vals = scores[:, qi] if metric == 'ip' else ot.l2_values(scores[:, qi], norm2)
        bins = ot.bins_ip(vals, r) if metric == 'ip' else ot.bins_l2(vals, r, shift)
        hist = st['hist'][qi].astype(np.int64)
        assert hist.sum() == n and np.array_equal(hist, ot.histogram(bins))
        # the threshold: the bin of the need-th row from the top, minus 2 eps and one bin
        assert need == min(k, n)
        found = ot.found_bin(hist, need)
        assert np.sort(bins)[::-1][need - 1] == found
        assert min(abs(float(thr) - float(t)) for t in ot.thresholds(found, r, eps, shift)) <= np.spacing(abs(thr))
        # the candidates: exactly the rows at or above the threshold
        want = np.nonzero(vals >= thr)[0]
        assert int(st['n_cand'][qi]) == len(want)
        if fell_back:
            continue
        assert np.array_equal(np.sort(st['cand'][qi, :len(want)].astype(np.int64)), want)
        # sound: no row left out could reach the returned k-th place, even with the rescore's error on both sides
        kth = int(idx[qi, need - 1])
        out = torch.ones(n, dtype=torch.bool, device=dev)
        out[torch.from_numpy(want).to(dev)] = False
        reach = ex[qi][out] + err[qi][out]
        assert bool((reach < ex[qi, kth] - err[qi, kth]).all()), (qi, float(reach.max()), float(ex[qi, kth]))


# ------------------------------------------------------------------------------------ (c) adversarial
E2E = [(h, k, q) for h in (768, 4096) for k in (1, 10, 100, 256) for q in (1, 16, 17)]


def planted_answer(p, k):
    return torch.cat([p.winners[:, None], p.outrankers[:, :k - 1]], dim=1)


@pytest.mark.parametrize('metric', ['ip', 'l2'])
@pytest.mark.parametrize('h,k,q', E2E)
def test_adversarial_corpus_equals_the_cuda_core_scan(dev, hw_model, metric, h, k, q):
    """The TF32 scan ranks k rows above each query's winner; the search must still return the winner first,
    then the outrankers in exact order, bit for bit what the CUDA-core scan returns."""
    n = 50_021
    p = ot.adversarial(n, h, q, k, hw_model, seed=h + 3 * k + q, device=dev)
    (s, i), _, _ = tc_search(metric, p.queries, p.corpus, k)
    assert not nv.topk_tc_fell_back()
    s2, i2 = cuda_core(metric, p.queries, p.corpus, k)
    assert torch.equal(i.cpu(), planted_answer(p, k))
    assert torch.equal(s, s2) and torch.equal(i, i2)


@pytest.mark.parametrize('h,k', [(768, 10), (768, 100), (4096, 100)])
def test_l2_with_far_background_rows(dev, h, k):
    """max_norm ~ 10^3 |q|: the histogram spans [-r - M^2 / 2, r] and its shift dominates every bin."""
    n, q = 50_021, 16
    p = ot.adversarial(n, h, q, k, ot.TRUNC, seed=h + k, device=dev, far_background=True)
    (s, i), _, m = tc_search('l2', p.queries, p.corpus, k)
    assert m > 500 * float(p.queries.norm(dim=1).max())
    assert not nv.topk_tc_fell_back()
    s2, i2 = cuda_core('l2', p.queries, p.corpus, k)
    assert torch.equal(i.cpu(), planted_answer(p, k))
    assert torch.equal(s, s2) and torch.equal(i, i2)


@pytest.mark.parametrize('metric', ['inner_product', 'l2'])
def test_faiss_index_v1_retriever_on_an_adversarial_corpus(dev, hw_model, tmp_path, metric):
    from distllm_b200.rag.search import FaissIndexV1
    from distllm_b200.rag.search import FaissIndexV1Config
    from distllm_b200.rag.search import Retriever

    k, q = 10, 16
    p = ot.adversarial(40_000, 768, q, k, hw_model, seed=17, device=dev)
    index = FaissIndexV1(p.corpus, FaissIndexV1Config(dataset_dir=tmp_path, metric=metric), device=dev)
    res, _ = Retriever(None, None, index).search(query_embedding=p.queries, top_k=k)
    assert not nv.topk_tc_fell_back()
    assert res.total_indices == planted_answer(p, k).tolist()
