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

``faiss_index_v1`` configs (FaissIndexV1, search.py:402-666) index the dataset's ``faiss_index_name`` column the
same way: ``metric='inner_product'`` is the exact float32 search above, ``metric='l2'`` is faiss IndexFlatL2
(``b2e_topk_l2`` / ``b2e_topk_l2_tc``: squared Euclidean distances, ascending, on the stored row norms), with
queries normalised only for ``inner_product`` and ``score <= threshold`` kept for ``l2`` (:561-603).  No
``.index`` file is read or written.
"""

from __future__ import annotations

from pathlib import Path
from typing import Annotated
from typing import Any
from typing import Literal
from typing import Optional
from typing import Union

import numpy as np
import torch
from datasets.search import BatchedSearchResults
from pydantic import Discriminator
from pydantic import Field
from pydantic import Tag

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


class FaissIndexV1Config(BaseConfig):
    """The reference's ``FaissIndexV1Config`` (search.py:402-429): same fields and defaults.  The column
    ``faiss_index_name`` of the dataset is indexed as float32 on the device; ``faiss_index_path`` is accepted and
    unused (no ``.index`` file is read or written)."""

    name: Literal['faiss_index_v1'] = 'faiss_index_v1'  # type: ignore[assignment]
    dataset_dir: Path = Field(..., description='HF dataset directory with the document text and fp32 embeddings')
    faiss_index_path: Optional[Path] = None  # noqa: UP007
    faiss_index_name: str = Field('embeddings', description='the dataset column that is indexed')
    metric: Literal['l2', 'inner_product'] = Field(
        'inner_product', description='faiss IndexFlatL2 (squared distances, ascending) or IndexFlatIP')


class ExactIndex:
    """Device-resident embedding matrix + exact inner-product search (faiss.IndexFlatIP semantics)."""

    metric = 'inner_product'

    def __init__(self, embeddings: np.ndarray | torch.Tensor | None = None,
                 config: ExactIndexConfig | None = None, device: torch.device | str | None = None) -> None:
        self.config = config or ExactIndexConfig()
        self.dataset = None
        if embeddings is None:
            embeddings = self._load_dataset('embeddings')
        matrix, dev = self._matrix(embeddings, device)
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
        self._upload(matrix, dtype, dev)
        # bound of the row norms: sizes the TF32 margin of the tensor-core scan (b2e_topk_ip_tc).  Computed once
        # here, a hair above the measured maximum; None (bf16 corpus) keeps the CUDA-core scan.
        self.max_norm = None
        if dtype == torch.float32 and matrix.shape[0] > 0:
            self.max_norm = _native.max_row_norm(self.corpus) * 1.0001

    def _load_dataset(self, column: str) -> np.ndarray:
        """Keep the dataset at config.dataset_dir (for get) and return its `column` as a float32 matrix."""
        if self.config.dataset_dir is None:
            raise ValueError('Provide an embedding matrix or a dataset_dir')
        from datasets import Dataset

        self.dataset = Dataset.load_from_disk(str(self.config.dataset_dir))
        # straight from Arrow: datasets' numpy formatter converts row by row (and imports torchvision's video
        # reader whenever torchvision is loaded)
        col = self.dataset.with_format('arrow')[:].column(column).combine_chunks()
        values = np.asarray(col.flatten().to_numpy(zero_copy_only=False), dtype=np.float32)
        return values.reshape(len(col), len(values) // max(len(col), 1))

    @staticmethod
    def _matrix(embeddings, device) -> tuple[torch.Tensor, torch.device]:
        if not torch.cuda.is_available():
            raise _native.NativeError('no CUDA device: the exact index has no CPU fallback (sm_90a only)')
        dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        matrix = torch.as_tensor(embeddings)
        if matrix.ndim != 2:
            raise ValueError(f'embeddings must be [N, H], got {tuple(matrix.shape)}')
        return matrix, dev

    def _upload(self, matrix: torch.Tensor, dtype: torch.dtype, dev: torch.device) -> None:
        self.corpus = matrix.to(device=dev, dtype=dtype)
        # the scans read one 16-byte vector per lane: rows are zero-padded to a multiple of 128 (float32) or 256
        # (bfloat16) columns (esmc-300m's 960), and queries alike in search; zeros add nothing to any inner product
        # (nor to any squared distance)
        pad = -matrix.shape[1] % (128 if dtype == torch.float32 else 256)
        if pad:
            self.corpus = torch.nn.functional.pad(self.corpus, (0, pad))
        self.corpus = self.corpus.contiguous()
        self.embedding_size = matrix.shape[1]

    def __len__(self) -> int:
        return self.corpus.shape[0]

    def get(self, indices: list[int], key: str) -> list[Any]:
        """The dataset's `key` values at `indices`, in the given order (search.py:384-399 and :651-666)."""
        if self.dataset is None:
            raise ValueError('this index was built from an in-memory matrix: it has no dataset to read '
                             f'{key!r} from (build it from a dataset_dir)')
        return list(self.dataset.select([int(i) for i in indices])[key])

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
        scores, indices = self._topk(queries, top_k)
        scores, indices = scores.cpu(), indices.cpu()
        total_scores, total_indices = [], []
        for s_row, i_row in zip(scores.tolist(), indices.tolist()):
            keep = [(s, i) for s, i in zip(s_row, i_row) if i >= 0]   # fewer than top_k rows in the index
            total_scores.append([s for s, _ in keep])
            total_indices.append([i for _, i in keep])
        results = BatchedSearchResults(total_scores=total_scores, total_indices=total_indices)
        return filter_search_by_score(results, score_threshold, self.metric)

    def _pad_queries(self, queries: torch.Tensor) -> torch.Tensor:
        if queries.shape[-1] == self.embedding_size < self.corpus.shape[1]:
            queries = torch.nn.functional.pad(queries, (0, self.corpus.shape[1] - queries.shape[-1])).contiguous()
        return queries

    def _topk(self, queries: torch.Tensor, top_k: int) -> tuple[torch.Tensor, torch.Tensor]:
        if self.precision == 'ubinary':
            scores, indices = _native.search_ubinary(queries, self.corpus, top_k, self.config.rescore_multiplier)
            if bool((indices == -2).any()):
                raise _native.NativeError('ubinary search: more rows tie at the threshold Hamming distance than '
                                          'the candidate buffer holds (duplicate corpus rows?)')
        else:
            scores, indices = _native.topk_ip(self._pad_queries(queries), self.corpus, top_k, max_norm=self.max_norm)
        return scores, indices


class FaissIndexV1(ExactIndex):
    """The reference's FaissIndexV1 (search.py:432-666) on the device: the dataset's ``faiss_index_name`` column as
    a float32 matrix in HBM, searched exactly as faiss IndexFlatIP (``metric='inner_product'``) or IndexFlatL2
    (``metric='l2'``: squared distances, ascending, ties by row id).  An in-memory matrix may replace the dataset
    (then ``get`` has nothing to read)."""

    def __init__(self, embeddings: np.ndarray | torch.Tensor | None = None,
                 config: FaissIndexV1Config | None = None, device: torch.device | str | None = None) -> None:
        if config is None:
            raise ValueError('FaissIndexV1 needs a FaissIndexV1Config')
        self.config = config
        self.metric = config.metric
        self.precision = 'float32'
        self.dataset = None
        if embeddings is None:
            embeddings = self._load_dataset(config.faiss_index_name)
        matrix, dev = self._matrix(embeddings, device)
        self._upload(matrix, torch.float32, dev)
        # built once with the index: the bound of the row norms sizes the tensor-core scans' margins, and the l2
        # scan ranks rows on the stored squared norms
        self.max_norm, self.norms = None, None
        if matrix.shape[0] > 0:
            norms, max_norm = _native.row_norms(self.corpus)
            self.max_norm = max_norm * 1.0001
            if self.metric == 'l2':
                self.norms = norms

    def transform(self, embeddings: np.ndarray) -> np.ndarray:
        """search.py:561-578: faiss.normalize_L2 for ``inner_product``; ``l2`` queries are used as they are."""
        return ExactIndex.transform(embeddings) if self.metric == 'inner_product' else embeddings

    def _topk(self, queries: torch.Tensor, top_k: int) -> tuple[torch.Tensor, torch.Tensor]:
        queries = self._pad_queries(queries)
        if self.metric == 'l2':
            if self.norms is None:
                return _native.topk_l2(queries, self.corpus, top_k)
            return _native.topk_l2(queries, self.corpus, top_k, norms=self.norms, max_norm=self.max_norm)
        return _native.topk_ip(queries, self.corpus, top_k, max_norm=self.max_norm)


def filter_search_by_score(results: BatchedSearchResults, score_threshold: float,
                           metric: str = 'inner_product') -> BatchedSearchResults:
    """search.py:338-377 and :580-637: drop results worse than the threshold -- an inner product below it, a
    squared L2 distance (``metric='l2'``) above it.  A threshold of 0.0 keeps all."""
    if not score_threshold:
        return results
    lower_is_better = metric == 'l2'
    new_scores, new_indices = [], []
    for indices, scores in zip(results.total_indices, results.total_scores):
        kept = [(i, s) for i, s in zip(indices, scores)
                if (s <= score_threshold if lower_is_better else s >= score_threshold)]
        new_indices.append([i for i, _ in kept])
        new_scores.append([s for _, s in kept])
    return BatchedSearchResults(total_scores=new_scores, total_indices=new_indices)


def _index_config_kind(value: Any) -> str:
    """'v1' for a faiss_index_v1 config, else 'exact' (whose Literal name then rejects anything unknown)."""
    name = value.get('name') if isinstance(value, dict) else getattr(value, 'name', None)
    return 'v1' if name == 'faiss_index_v1' else 'exact'


IndexConfig = Annotated[
    Union[Annotated[ExactIndexConfig, Tag('exact')], Annotated[FaissIndexV1Config, Tag('v1')]],
    Discriminator(_index_config_kind),
]


class RetrieverConfig(BaseConfig):
    """Settings of a retriever (distllm/rag/search.py:669-712, with the exact index in place of faiss).  The
    ``faiss_config`` is told apart by its ``name``: ``exact_index`` (the default) and ``faiss_index_v2`` build an
    ExactIndex, ``faiss_index_v1`` a FaissIndexV1."""

    faiss_config: IndexConfig = Field(..., description='Settings for the exact index')
    encoder_config: dict = Field(..., description='Settings for the encoder (as in the embedding YAML)')
    pooler_config: dict = Field(..., description='Settings for the pooler')
    batch_size: int = Field(4, description='Batch size for the embedder model')

    def get_retriever(self) -> 'Retriever':
        from distllm_b200.embed import get_encoder
        from distllm_b200.embed import get_pooler

        encoder = get_encoder(dict(self.encoder_config))
        pooler = get_pooler(dict(self.pooler_config))
        if isinstance(self.faiss_config, FaissIndexV1Config):
            index = FaissIndexV1(config=self.faiss_config)
        else:
            index = ExactIndex(config=self.faiss_config)
        return Retriever(encoder=encoder, pooler=pooler, faiss_index=index, batch_size=self.batch_size)


class Retriever:
    """Semantic similarity search: same call surface as distllm/rag/search.py:715-881."""

    def __init__(self, encoder, pooler, faiss_index: ExactIndex | FaissIndexV1, batch_size: int = 4) -> None:
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

    def get(self, indices: list[int], key: str) -> list[Any]:
        """The dataset's `key` values at `indices`, in the given order (search.py:883-897)."""
        return self.faiss_index.get(indices, key)

    def get_embeddings(self, indices: list[int]) -> np.ndarray:
        """[len(indices), H] rows of the dataset's ``embeddings`` column (search.py:899-912)."""
        return np.array(self.get(indices, 'embeddings'))

    def get_texts(self, indices: list[int]) -> list[str]:
        """The ``text`` of the rows at `indices` (search.py:914-928)."""
        return self.get(indices, 'text')
