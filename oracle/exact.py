"""Retrieval inputs whose inner products are exact in fp32, and torch restatements of oracle/search.py for
corpora too large for numpy on the host.  TEST INFRASTRUCTURE ONLY.

Every entry is a small integer, |x| <= 8, or such an integer times one power of two.  With H <= 8192 every
product and every partial sum is then an integer (times that power) below 2^24 in magnitude, so its fp32
value is the same in any summation order: in an FMA scan, in a TF32 tensor-core scan (integers up to 2^11
are exact in TF32), in a rescore, and in float64.  bfloat16 holds these integers exactly too.  A kernel's
scores can therefore be compared with the reference bit for bit, and which row wins an equal score is
decided by the contract alone (descending score, ties by ascending row id), not by rounding.
"""

from __future__ import annotations

import numpy as np
import torch

from oracle import search as osearch


def int_matrix(n: int, h: int, bound: int, gen: torch.Generator, dtype=torch.float32,
               device=None) -> torch.Tensor:
    """[n, h] integers uniform in [-bound, bound], stored as `dtype` (exact for bound <= 256)."""
    return torch.empty((n, h), dtype=dtype, device=device or gen.device).random_(-bound, bound + 1, generator=gen)


# ----------------------------------------------------------------------------- planted ties at the k-th place
def base_row(q: torch.Tensor) -> torch.Tensor:
    """The query with entry 0 zeroed.  With q[0] == 1, base_row(q) + s * e_0 scores |q|^2 - 1 + s: seventeen
    exact score levels (|s| <= 8) far above a background of smaller integers."""
    b = q.clone()
    b[0] = 0
    return b


def equal_dot_rows(q: torch.Tensor, count: int) -> torch.Tensor:
    """`count` distinct rows with the same inner product with q as base_row(q): row t adds +1 and -1 at two
    positions i, j > 0 with q[i] == q[j] (row 0 is base_row(q) itself)."""
    qc = q.cpu()
    groups: dict[int, list[int]] = {}
    for i in range(1, qc.numel()):
        v = int(qc[i])
        if -7 <= v <= 7:
            groups.setdefault(v, []).append(i)
    pairs = [(idx[2 * p], idx[2 * p + 1]) for idx in groups.values() for p in range(len(idx) // 2)]
    if len(pairs) < count - 1:
        raise ValueError('query has too few equal entries for distinct equal-dot rows')
    base = base_row(q)
    rows = base.repeat(count, 1)
    for t in range(1, count):
        i, j = pairs[t - 1]
        rows[t, i] += 1
        rows[t, j] -= 1
    return rows


def planted_ties(queries: torch.Tensor, corpus: torch.Tensor, k: int, tie_rows: list[list[int]],
                 gen: torch.Generator, equal_dot: bool = False) -> None:
    """Plant, in place, for every query qi: the rows tie_rows[qi] all scoring T_qi = |q|^2 - 1 exactly
    (duplicates of base_row(q), or distinct vectors with that same dot product when `equal_dot`), and k - 1
    rows elsewhere scoring strictly more (T + s, s in 1..8: many of them tied among themselves too).
    queries[:, 0] must be 1, and the background must score below every T (the caller checks with the
    reference)."""
    taken = {r for rows in tie_rows for r in rows}
    assert len(taken) == sum(len(rows) for rows in tie_rows), 'tie rows overlap'
    n = corpus.shape[0]
    cpu = torch.Generator().manual_seed(int(torch.randint(0, 2**31, (1,), generator=gen, device=gen.device)))
    perm = torch.randperm(n, generator=cpu)
    free = perm[~torch.isin(perm, torch.tensor(sorted(taken), dtype=torch.long))]
    at = 0
    for qi, rows in enumerate(tie_rows):
        q = queries[qi].to(corpus.dtype)
        vec = equal_dot_rows(q, len(rows)) if equal_dot else base_row(q).repeat(len(rows), 1)
        corpus[torch.tensor(rows, device=corpus.device)] = vec
        if k > 1:
            better = free[at:at + k - 1].to(corpus.device)
            at += k - 1
            up = base_row(q).repeat(k - 1, 1)
            up[:, 0] = torch.randint(1, 9, (k - 1,), generator=cpu).to(up.dtype).to(up.device)
            corpus[better] = up


# ------------------------------------------------------------------------- references on any torch device
def score_matrix(queries: torch.Tensor, corpus: torch.Tensor, chunk: int = 1 << 18) -> torch.Tensor:
    """[Q, N] float64 inner products, computed in row chunks (exact for the inputs above: integers < 2^53)."""
    q64 = queries.to(torch.float64)
    out = torch.empty((queries.shape[0], corpus.shape[0]), dtype=torch.float64, device=corpus.device)
    for lo in range(0, corpus.shape[0], chunk):
        out[:, lo:lo + chunk] = q64.to(corpus.device) @ corpus[lo:lo + chunk].to(torch.float64).T
    return out


def topk_inner_product(queries: torch.Tensor, corpus: torch.Tensor, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    """oracle/search.py:topk_inner_product in torch: (scores [Q, k'] f32, indices [Q, k'] i64), k' = min(k, N),
    descending float64 score cast to fp32, ties by ascending index (a stable descending sort)."""
    s = score_matrix(queries, corpus)
    vals, order = torch.sort(s, dim=1, descending=True, stable=True)
    kk = min(k, corpus.shape[0])
    return vals[:, :kk].to(torch.float32), order[:, :kk]


def pack_bits(x: torch.Tensor) -> torch.Tensor:
    """np.packbits(x > 0) per row in torch: [N, H] -> [N, H/8] uint8, first dimension in the MSB."""
    bits = (x > 0).to(torch.uint8).view(x.shape[0], -1, 8)
    weights = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], dtype=torch.uint8, device=x.device)
    return (bits * weights).sum(dim=2, dtype=torch.uint8)


def unpack_bits(b: torch.Tensor) -> torch.Tensor:
    shifts = torch.arange(7, -1, -1, device=b.device, dtype=torch.uint8)
    return ((b[..., None] >> shifts) & 1).reshape(b.shape[0], -1)


_POPCOUNT = torch.tensor([bin(i).count('1') for i in range(256)], dtype=torch.int16)


def search_ubinary(queries: torch.Tensor, corpus_bits: torch.Tensor, top_k: int, rescore_multiplier: int = 2,
                   chunk: int = 1 << 19) -> tuple[torch.Tensor, torch.Tensor]:
    """oracle/search.py:search_ubinary in torch: Hamming top-(top_k * multiplier) by (distance, id), then the
    float query against each candidate's bits in float64, a stable descending sort, top_k.  Chunked so that a
    packed corpus of several GB can be searched on the device."""
    dev = corpus_bits.device
    n = corpus_bits.shape[0]
    qbits = pack_bits(queries.to(dev))
    table = _POPCOUNT.to(dev)
    dist = torch.empty((queries.shape[0], n), dtype=torch.int16, device=dev)
    for qi in range(queries.shape[0]):
        for lo in range(0, n, chunk):
            x = torch.bitwise_xor(corpus_bits[lo:lo + chunk], qbits[qi][None])
            dist[qi, lo:lo + chunk] = table[x.int()].sum(dim=1, dtype=torch.int16)
    kk = min(top_k * rescore_multiplier, n)
    _, cand = torch.sort(dist, dim=1, stable=True)
    cand = cand[:, :kk]
    scores, indices = [], []
    for qi in range(queries.shape[0]):
        bits = unpack_bits(corpus_bits[cand[qi]]).to(torch.float64)
        s = bits @ queries[qi].to(dev, torch.float64)
        vals, order = torch.sort(s, descending=True, stable=True)
        scores.append(vals[:top_k].to(torch.float32))
        indices.append(cand[qi][order[:top_k]])
    return torch.stack(scores), torch.stack(indices)


def numpy_reference(queries: torch.Tensor, corpus: torch.Tensor, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    """oracle/search.py itself (numpy on the host), returned as torch tensors."""
    s, i = osearch.topk_inner_product(queries.cpu().numpy(), corpus.float().cpu().numpy(), k)
    return torch.from_numpy(s), torch.from_numpy(np.ascontiguousarray(i)).to(torch.int64)
