"""Squared-L2 restatement of the exact search the reference delegates to faiss, and retrieval inputs for it whose
arithmetic is exact.  TEST INFRASTRUCTURE ONLY.

distllm/rag/search.py:402-666 (FaissIndexV1 with metric='l2') builds a ``faiss.IndexFlatL2`` over the dataset's fp32
embeddings column: search returns, per query, the k rows with the smallest SQUARED Euclidean distance, ascending.
faiss is third-party and not vendored, so this restates IndexFlatL2's published behaviour, with ties broken by
ascending row id (the contract of include/b2e.h: b2e_topk_l2).

The inputs follow oracle/exact.py: small integers (|x| <= 8), or such integers times one power of two.  With
H <= 8192 every difference, square and partial sum is then an integer (times that power) below 2^24, so a kernel's
fp32 distances equal the float64 ones here bit for bit, in any summation order, and equal distances are decided by
the row id alone.
"""

from __future__ import annotations

import numpy as np
import torch


def topk_l2(queries: np.ndarray, corpus: np.ndarray, k: int) -> tuple[np.ndarray, np.ndarray]:
    """(distances [Q,k'], indices [Q,k']), k' = min(k, N): squared Euclidean distances in float64 cast to fp32,
    ascending, ties by ascending index."""
    c64 = corpus.astype(np.float64)
    dist = np.stack([((c64 - q[None, :]) ** 2).sum(axis=1) for q in queries.astype(np.float64)])
    k = min(k, corpus.shape[0])
    order = np.lexsort((np.arange(corpus.shape[0])[None, :].repeat(len(queries), 0), dist), axis=1)[:, :k]
    return np.take_along_axis(dist, order, axis=1).astype(np.float32), order


def numpy_reference(queries: torch.Tensor, corpus: torch.Tensor, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    """topk_l2 above (numpy on the host), returned as torch tensors."""
    s, i = topk_l2(queries.cpu().numpy(), corpus.float().cpu().numpy(), k)
    return torch.from_numpy(s), torch.from_numpy(np.ascontiguousarray(i)).to(torch.int64)


# ------------------------------------------------------------------------- references on any torch device
def l2_matrix(queries: torch.Tensor, corpus: torch.Tensor, chunk: int = 1 << 18) -> torch.Tensor:
    """[Q, N] float64 squared Euclidean distances |q|^2 + |x|^2 - 2 q.x, in row chunks (exact for the inputs
    above: integers < 2^53)."""
    q64 = queries.to(torch.float64).to(corpus.device)
    qn = (q64 * q64).sum(dim=1, keepdim=True)
    out = torch.empty((queries.shape[0], corpus.shape[0]), dtype=torch.float64, device=corpus.device)
    for lo in range(0, corpus.shape[0], chunk):
        x = corpus[lo:lo + chunk].to(torch.float64)
        out[:, lo:lo + chunk] = qn + (x * x).sum(dim=1)[None, :] - 2.0 * (q64 @ x.T)
    return out


def topk_l2_torch(queries: torch.Tensor, corpus: torch.Tensor, k: int) -> tuple[torch.Tensor, torch.Tensor]:
    """topk_l2 in torch, for corpora too large for numpy on the host: (distances [Q, k'] f32, indices [Q, k'] i64),
    k' = min(k, N), ascending float64 distance cast to fp32, ties by ascending index (a stable ascending sort)."""
    vals, order = torch.sort(l2_matrix(queries, corpus), dim=1, stable=True)
    kk = min(k, corpus.shape[0])
    return vals[:, :kk].to(torch.float32), order[:, :kk]


# ----------------------------------------------------------------------------- planted ties at the k-th place
def planted_ties(queries: torch.Tensor, corpus: torch.Tensor, k: int, tie_rows: list[list[int]],
                 gen: torch.Generator, permute: bool = True) -> None:
    """The squared-L2 counterpart of oracle/exact.py:planted_ties, in place: for every query qi, the rows
    tie_rows[qi] all lie at squared distance 15 from it, as q + P(d) for d = (3, 2, 1, 1, 0, ...) and a different
    coordinate permutation P per row (distinct vectors; the same vector q + d for every row when not `permute`), and
    k - 1 rows elsewhere lie strictly closer, at q + v e_j with v in {1, 2, 3} (distances 1, 4, 9: many tied among
    themselves too).  The background must lie farther than 15 from every query (the caller checks with the
    reference)."""
    taken = {r for rows in tie_rows for r in rows}
    assert len(taken) == sum(len(rows) for rows in tie_rows), 'tie rows overlap'
    n, h = corpus.shape
    cpu = torch.Generator().manual_seed(int(torch.randint(0, 2**31, (1,), generator=gen, device=gen.device)))
    perm = torch.randperm(n, generator=cpu)
    free = perm[~torch.isin(perm, torch.tensor(sorted(taken), dtype=torch.long))]
    d = torch.zeros(h, dtype=corpus.dtype)
    d[:4] = torch.tensor([3.0, 2.0, 1.0, 1.0])
    at = 0
    for qi, rows in enumerate(tie_rows):
        q = queries[qi].to(corpus.dtype).cpu()
        if permute:
            vec = torch.stack([q + d[torch.randperm(h, generator=cpu)] for _ in rows])
        else:
            vec = (q + d).repeat(len(rows), 1)
        corpus[torch.tensor(rows, device=corpus.device)] = vec.to(corpus.device)
        if k > 1:
            better = free[at:at + k - 1]
            at += k - 1
            up = q.repeat(k - 1, 1)
            j = torch.randint(0, h, (k - 1,), generator=cpu)
            up[torch.arange(k - 1), j] += torch.randint(1, 4, (k - 1,), generator=cpu).to(up.dtype)
            corpus[better.to(corpus.device)] = up.to(corpus.device)
