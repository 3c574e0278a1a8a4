"""The premise of tests/test_gpu_retrieval_exact.py, checked on the host: the integer inputs of oracle/exact.py
have fp32 inner products that do not depend on the summation order, survive bfloat16 unchanged, and the
references (oracle/search.py and its torch restatement in oracle/exact.py) order equal scores by row id."""

from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import exact
from oracle import search as osearch


@pytest.mark.parametrize('h', [128, 256, 768, 8192])
def test_integer_scores_are_exact_in_any_fp32_summation_order(h):
    g = torch.Generator().manual_seed(h)
    corpus = exact.int_matrix(64, h, 8, g).numpy()
    queries = exact.int_matrix(3, h, 8, g).numpy()
    queries[0] *= 2.0 ** -3                      # the same values scaled by a power of two stay exact
    ref = queries.astype(np.float64) @ corpus.astype(np.float64).T
    assert np.abs(ref).max() < 2 ** 24
    rng = np.random.default_rng(h)
    for _ in range(2):
        perm = rng.permutation(h)
        prod = (queries[:, None, perm] * corpus[None, :, perm]).astype(np.float32)
        seq = np.zeros(prod.shape[:2], dtype=np.float32)
        for j in range(h):                       # one fp32 rounding per addition, in a shuffled order
            seq = (seq + prod[:, :, j]).astype(np.float32)
        assert np.array_equal(seq.astype(np.float64), ref)
        # pairwise (tree) order, as a warp reduction sums (zero-padded to a power of two)
        width = 1 << (h - 1).bit_length()
        tree = np.zeros(prod.shape[:2] + (width,), dtype=np.float32)
        tree[:, :, :h] = prod
        while tree.shape[2] > 1:
            tree = (tree[:, :, 0::2] + tree[:, :, 1::2]).astype(np.float32)
        assert np.array_equal(tree[:, :, 0].astype(np.float64), ref)


def test_integer_inputs_round_trip_bfloat16_and_tf32():
    g = torch.Generator().manual_seed(1)
    x = exact.int_matrix(100, 256, 8, g)
    assert torch.equal(x.to(torch.bfloat16).float(), x)
    assert torch.equal((x * 2.0 ** -5).to(torch.bfloat16).float(), x * 2.0 ** -5)
    assert torch.equal(exact.int_matrix(10, 256, 8, g, dtype=torch.bfloat16).float().abs().max(), torch.tensor(8.0))
    # TF32 keeps 10 explicit mantissa bits: dropping the low 13 bits of an integer <= 2^11 changes nothing
    bits = x.view(torch.int32)
    assert torch.equal((bits & ~0x1FFF).view(torch.float32), x)


def test_oracle_orders_ties_by_row_id():
    q = np.array([[1.0, 0.0], [0.0, 0.0]], dtype=np.float32)
    corpus = np.array([[1, 5], [2, 0], [1, -3], [2, 7], [0, 0], [1, 0]], dtype=np.float32)
    s, i = osearch.topk_inner_product(q, corpus, 4)
    assert i.tolist() == [[1, 3, 0, 2], [0, 1, 2, 3]]
    assert s.tolist() == [[2, 2, 1, 1], [0, 0, 0, 0]]
    ts, ti = exact.topk_inner_product(torch.from_numpy(q), torch.from_numpy(corpus), 4)
    assert ti.tolist() == i.tolist() and ts.tolist() == s.tolist()


@pytest.mark.parametrize('q,n,h,k', [(3, 500, 128, 10), (5, 2000, 256, 256), (2, 7, 128, 10)])
def test_torch_reference_equals_oracle_on_tie_heavy_inputs(q, n, h, k):
    g = torch.Generator().manual_seed(n)
    corpus = exact.int_matrix(n, h, 1, g)        # entries in {-1, 0, 1}: thousands of equal scores
    queries = exact.int_matrix(q, h, 1, g)
    ref_s, ref_i = exact.numpy_reference(queries, corpus, k)
    got_s, got_i = exact.topk_inner_product(queries, corpus, k)
    assert torch.equal(got_s, ref_s) and torch.equal(got_i, ref_i)
    assert got_i.shape[1] == min(k, n)


@pytest.mark.parametrize('equal_dot', [False, True])
def test_planted_ties_have_exactly_k_minus_1_better_rows(equal_dot):
    g = torch.Generator().manual_seed(7)
    k, n, h = 20, 3000, 256
    queries = exact.int_matrix(3, h, 8, g)
    queries[:, 0] = 1
    corpus = exact.int_matrix(n, h, 4, g)
    tie_rows = [[401, 402, 405], [1000, 7, 2999], [64, 65, 66]]
    exact.planted_ties(queries, corpus, k, tie_rows, g, equal_dot=equal_dot)
    s = exact.score_matrix(queries, corpus)
    for qi, rows in enumerate(tie_rows):
        t = float(queries[qi].double() @ queries[qi].double()) - 1
        assert (s[qi] > t).sum() == k - 1 and (s[qi] == t).sum() == len(rows)
        assert (s[qi, rows] == t).all()
        vecs = corpus[rows]
        assert len({tuple(v.tolist()) for v in vecs}) == (len(rows) if equal_dot else 1)
    _, idx = exact.topk_inner_product(queries, corpus, k)
    assert idx[:, -1].tolist() == [min(r) for r in tie_rows]


@pytest.mark.parametrize('q,n,h,k,mult', [(3, 400, 256, 10, 2), (2, 5, 128, 4, 2), (4, 3000, 768, 50, 3)])
def test_torch_ubinary_reference_equals_oracle(q, n, h, k, mult):
    g = torch.Generator().manual_seed(n + h)
    corpus = exact.int_matrix(n, h, 8, g)
    corpus[n // 3:n // 3 + 5] = corpus[1]        # duplicates: equal distances and equal rescored scores
    queries = exact.int_matrix(q, h, 8, g)
    bits = exact.pack_bits(corpus)
    assert np.array_equal(bits.numpy(), osearch.quantize_ubinary(corpus.numpy()))
    assert torch.equal(exact.unpack_bits(bits), (corpus > 0).to(torch.uint8))
    ref_s, ref_i = osearch.search_ubinary(queries.numpy(), bits.numpy(), k, mult)
    got_s, got_i = exact.search_ubinary(queries, bits, k, mult, chunk=97)
    assert np.array_equal(got_s.numpy(), ref_s) and np.array_equal(got_i.numpy(), ref_i)
