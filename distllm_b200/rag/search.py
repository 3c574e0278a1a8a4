"""Query side of the RAG search: embed the queries with the native encoder + pooler, then an exact
inner-product top-k over the device-resident embedding matrix.

Mirrors the float32 / exact branch of distllm/rag/search.py:

    FaissIndexV2.transform       :258-278   L2-normalise the query embeddings
    FaissIndexV2.search          :280-336   faiss.IndexFlatIP through semantic_search_faiss -> BatchedSearchResults
    _filter_search_by_score      :338-377   keep results with score >= threshold
    Retriever.search             :743-798
    Retriever.get_pooled_embeddings / _get_pooled_embeddings   :800-881 (sort by length, batches of `batch_size`,
                                            tokenizer(padding=True, truncation=True), encode, pool, fp32)

The index itself is the device-resident matrix: no faiss file.  ``precision='float32'`` is the exact
IndexFlatIP search (``b2e_topk_ip`` / ``b2e_topk_ip_tc``: TF32 scan on the tensor cores, exact fp32 decision); ``precision='ubinary'`` is the reference's binary branch
(search.py:34-56, :202-260, :280-336: packbits(x > 0) corpus, Hamming top-(k * rescore_multiplier), float
rescoring) on ``b2e_pack_ubinary`` / ``b2e_search_ubinary``, 1/32 of the HBM traffic per query.  The HNSW
(approximate) branch is not built -- ``search_algorithm='hnsw'`` raises.  There is no CPU fallback.
"""

from __future__ import annotations

from pathlib import Path
from typing import Literal
from typing import Optional

import numpy as np
import torch
from datasets.search import BatchedSearchResults
from pydantic import Field

from distllm_b200 import _native
from distllm_b200.utils import BaseConfig
from distllm_b200.utils import batch_data

MAX_TOP_K = 256


class ExactIndexConfig(BaseConfig):
    """The reference's ``FaissIndexV2Config`` (search.py:59-95) for the exact branches: same field names and
    defaults, so a reference YAML validates; the faiss file fields are accepted and unused."""

    name: Literal['exact_index', 'faiss_index_v2'] = 'exact_index'  # type: ignore[assignment]
    # HF dataset directory with the document text and the fp32 ``embeddings`` column
    dataset_dir: Optional[Path] = None  # noqa: UP007
    faiss_index_path: Optional[Path] = None  # noqa: UP007  (no index file: the matrix lives in HBM)
    dataset_chunk_paths: Optional[list[Path]] = None  # noqa: UP007
    precision: Literal['float32', 'ubinary'] = Field(
        'float32', description='The desired precision for the embeddings [float32, ubinary].')
    search_algorithm: Literal['exact'] = Field('exact', description='only the exact search is built')
    rescore_multiplier: int = Field(2, description='Oversampling factor for rescoring (ubinary).')
    num_quantization_workers: int = 1   # accepted for compatibility: packing is one kernel launch
    # not in the reference: storage of the float32-precision matrix on the device: 'float32' (exact) or
    # 'bfloat16' (half the HBM traffic; scores are exact fp32 dot products of the ROUNDED corpus)
    corpus_dtype: Literal['float32', 'bfloat16'] = 'float32'


class ExactIndex:
    """Device-resident embedding matrix + exact inner-product search (faiss.IndexFlatIP semantics)."""

    def __init__(self, embeddings: np.ndarray | torch.Tensor | None = None,
                 config: ExactIndexConfig | None = None, device: torch.device | str | None = None) -> None:
        self.config = config or ExactIndexConfig()
        if embeddings is None:
            if self.config.dataset_dir is None:
                raise ValueError('Provide an embedding matrix or a dataset_dir')
            from datasets import Dataset

            dataset = Dataset.load_from_disk(str(self.config.dataset_dir))
            dataset.set_format('numpy', columns=['embeddings'])
            embeddings = np.asarray(dataset['embeddings'], dtype=np.float32)
            self.dataset = dataset
        if not torch.cuda.is_available():
            raise _native.NativeError('no CUDA device: the exact index has no CPU fallback (sm_90a only)')
        dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        matrix = torch.as_tensor(embeddings)
        if matrix.ndim != 2:
            raise ValueError(f'embeddings must be [N, H], got {tuple(matrix.shape)}')
        self.precision = self.config.precision
        if self.precision == 'ubinary':
            # quantize_embeddings(..., 'ubinary') (search.py:34-56): packed on the device, chunk by chunk so that
            # the fp32 matrix never has to sit in HBM next to its 32x smaller packed form
            if matrix.shape[1] % 32:
                raise ValueError(f'ubinary needs an embedding size that is a multiple of 32, got {matrix.shape[1]}')
            self.corpus = torch.empty((matrix.shape[0], matrix.shape[1] // 8), dtype=torch.uint8, device=dev)
            step = 1 << 20
            for lo in range(0, matrix.shape[0], step):
                rows = matrix[lo:lo + step].to(device=dev, dtype=torch.float32).contiguous()
                self.corpus[lo:lo + step] = _native.pack_ubinary(rows)
            self.embedding_size = matrix.shape[1]
            return
        dtype = torch.float32 if self.config.corpus_dtype == 'float32' else torch.bfloat16
        self.corpus = matrix.to(device=dev, dtype=dtype)
        # the scans read one 16-byte vector per lane: rows are zero-padded to a multiple of 128 (float32) or 256
        # (bfloat16) columns (esmc-300m's 960), and queries alike in search; zeros add nothing to any inner product
        pad = -matrix.shape[1] % (128 if dtype == torch.float32 else 256)
        if pad:
            self.corpus = torch.nn.functional.pad(self.corpus, (0, pad))
        self.corpus = self.corpus.contiguous()
        self.embedding_size = matrix.shape[1]
        # bound of the row norms: sizes the TF32 margin of the tensor-core scan (b2e_topk_ip_tc).  Computed once
        # here, a hair above the measured maximum; None (bf16 corpus) keeps the CUDA-core scan.
        self.max_norm = None
        if dtype == torch.float32 and matrix.shape[0] > 0:
            self.max_norm = _native.max_row_norm(self.corpus) * 1.0001

    def __len__(self) -> int:
        return self.corpus.shape[0]

    @staticmethod
    def transform(embeddings: np.ndarray) -> np.ndarray:
        """faiss.normalize_L2: in place, rows with zero norm stay zero (search.py:258-278)."""
        norms = np.sqrt((embeddings.astype(np.float32) ** 2).sum(axis=1, keepdims=True))
        np.divide(embeddings, norms, out=embeddings, where=norms > 0)
        return embeddings

    def search(self, query_embedding: np.ndarray | torch.Tensor, top_k: int = 1,
               score_threshold: float = 0.0) -> BatchedSearchResults:
        """Top-k most similar rows per query (search.py:280-336)."""
        if not 1 <= top_k <= MAX_TOP_K:
            raise ValueError(f'top_k must be in [1, {MAX_TOP_K}], got {top_k}')
        queries = torch.as_tensor(query_embedding, dtype=torch.float32).to(self.corpus.device).contiguous()
        if queries.ndim == 1:
            queries = queries[None]
        if self.precision == 'ubinary':
            scores, indices = _native.search_ubinary(queries, self.corpus, top_k, self.config.rescore_multiplier)
            if bool((indices == -2).any()):
                raise _native.NativeError('ubinary search: more rows tie at the threshold Hamming distance than '
                                          'the candidate buffer holds (duplicate corpus rows?)')
        else:
            if queries.shape[-1] == self.embedding_size < self.corpus.shape[1]:
                queries = torch.nn.functional.pad(queries, (0, self.corpus.shape[1] - queries.shape[-1])).contiguous()
            scores, indices = _native.topk_ip(queries, self.corpus, top_k, max_norm=self.max_norm)
        scores, indices = scores.cpu(), indices.cpu()
        total_scores, total_indices = [], []
        for s_row, i_row in zip(scores.tolist(), indices.tolist()):
            keep = [(s, i) for s, i in zip(s_row, i_row) if i >= 0]   # fewer than top_k rows in the index
            total_scores.append([s for s, _ in keep])
            total_indices.append([i for _, i in keep])
        results = BatchedSearchResults(total_scores=total_scores, total_indices=total_indices)
        return filter_search_by_score(results, score_threshold)


def filter_search_by_score(results: BatchedSearchResults, score_threshold: float) -> BatchedSearchResults:
    """search.py:338-377: drop results whose inner product is below the threshold (0.0 keeps all)."""
    if not score_threshold:
        return results
    new_scores, new_indices = [], []
    for indices, scores in zip(results.total_indices, results.total_scores):
        kept = [(i, s) for i, s in zip(indices, scores) if s >= score_threshold]
        new_indices.append([i for i, _ in kept])
        new_scores.append([s for _, s in kept])
    return BatchedSearchResults(total_scores=new_scores, total_indices=new_indices)


class RetrieverConfig(BaseConfig):
    """Settings of a retriever (distllm/rag/search.py:669-712, with the exact index in place of faiss)."""

    faiss_config: ExactIndexConfig = Field(..., description='Settings for the exact index')
    encoder_config: dict = Field(..., description='Settings for the encoder (as in the embedding YAML)')
    pooler_config: dict = Field(..., description='Settings for the pooler')
    batch_size: int = Field(4, description='Batch size for the embedder model')

    def get_retriever(self) -> 'Retriever':
        from distllm_b200.embed import get_encoder
        from distllm_b200.embed import get_pooler

        encoder = get_encoder(dict(self.encoder_config))
        pooler = get_pooler(dict(self.pooler_config))
        return Retriever(encoder=encoder, pooler=pooler, faiss_index=ExactIndex(config=self.faiss_config),
                         batch_size=self.batch_size)


class Retriever:
    """Semantic similarity search: same call surface as distllm/rag/search.py:715-881."""

    def __init__(self, encoder, pooler, faiss_index: ExactIndex, batch_size: int = 4) -> None:
        self.encoder = encoder
        self.pooler = pooler
        self.faiss_index = faiss_index
        self.batch_size = batch_size

    def search(self, query: str | list[str] | None = None, query_embedding: np.ndarray | None = None,
               top_k: int = 1, score_threshold: float = 0.0) -> tuple[BatchedSearchResults, np.ndarray]:
        if query is None and query_embedding is None:
            raise ValueError('Provide at least one of query or query_embedding.')
        if query_embedding is None:
            query_embedding = self.get_pooled_embeddings(query)
        results = self.faiss_index.search(query_embedding=query_embedding, top_k=top_k,
                                          score_threshold=score_threshold)
        return results, query_embedding

    def get_pooled_embeddings(self, query: str | list[str]) -> np.ndarray:
        if isinstance(query, str):
            query = [query]
        # sorted by length, embedded in batches, put back in the caller's order (search.py:815-836)
        order = sorted(range(len(query)), key=lambda i: len(query[i]))
        batches = batch_data([query[i] for i in order], chunk_size=self.batch_size)
        pooled = np.concatenate([self._get_pooled_embeddings(b) for b in batches], axis=0)
        return pooled[np.argsort(order)]

    @torch.no_grad()
    def _get_pooled_embeddings(self, query: list[str]) -> np.ndarray:
        batch = self.encoder.tokenizer(query, padding=True, truncation=True, return_tensors='pt')
        inputs = batch.to(self.encoder.device)
        hidden = self.encoder.encode(inputs)
        pooled = self.pooler.pool(hidden, inputs['attention_mask'])
        pooled = pooled.cpu().numpy().astype(np.float32)
        return self.faiss_index.transform(pooled)
