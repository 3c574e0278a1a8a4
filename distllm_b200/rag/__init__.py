"""Retrieval query path on the native kernels (SURVEY 8(f) rank 2)."""

from distllm_b200.rag.search import ExactIndex
from distllm_b200.rag.search import ExactIndexConfig
from distllm_b200.rag.search import FaissIndexV1
from distllm_b200.rag.search import FaissIndexV1Config
from distllm_b200.rag.search import Retriever
from distllm_b200.rag.search import RetrieverConfig

__all__ = ['ExactIndex', 'ExactIndexConfig', 'FaissIndexV1', 'FaissIndexV1Config', 'Retriever', 'RetrieverConfig']
