"""faiss_index_v1 retrieval without a device: the squared-L2 oracle and its planted ties, the V1 config as the
reference's evaluate YAMLs write it, the metric-dependent threshold, and Retriever.get / get_texts /
get_embeddings on an on-disk HF dataset."""

from __future__ import annotations

import numpy as np
import pytest
import torch
import yaml
from datasets import Dataset
from datasets.search import BatchedSearchResults

from distllm_b200.rag.search import ExactIndex
from distllm_b200.rag.search import ExactIndexConfig
from distllm_b200.rag.search import FaissIndexV1
from distllm_b200.rag.search import FaissIndexV1Config
from distllm_b200.rag.search import Retriever
from distllm_b200.rag.search import RetrieverConfig
from distllm_b200.rag.search import filter_search_by_score
from oracle import exact
from tools import oracle_l2 as ol2


@pytest.mark.parametrize('q,n,h,k', [(1, 1, 4, 1), (3, 50, 16, 7), (5, 300, 128, 256), (2, 40, 960, 3)])
def test_l2_oracle_equals_float64_brute_force_on_integers(q, n, h, k):
    g = torch.Generator().manual_seed(q + n + h + k)
    queries = exact.int_matrix(q, h, 8, g).numpy()
    corpus = exact.int_matrix(n, h, 2, g).numpy()
    corpus[n // 2:] = corpus[:n - n // 2]        # duplicate rows: every distance appears at least twice
    d, i = ol2.topk_l2(queries, corpus, k)
    kk = min(k, n)
    for qi in range(q):
        brute = [(float(((queries[qi].astype(np.float64) - corpus[r].astype(np.float64)) ** 2).sum()), r)
                 for r in range(n)]
        brute.sort()
        assert i[qi].tolist() == [r for _, r in brute[:kk]]
        assert d[qi].tolist() == [dd for dd, _ in brute[:kk]]
    # the torch restatement (the GPU tests' reference for large corpora) agrees bit for bit
    td, ti = ol2.topk_l2_torch(torch.from_numpy(queries), torch.from_numpy(corpus), k)
    assert torch.equal(ti, torch.from_numpy(i).to(torch.int64)) and torch.equal(td, torch.from_numpy(d))


@pytest.mark.parametrize('permute', [True, False])
@pytest.mark.parametrize('k', [1, 2, 17, 256])
def test_planted_l2_ties_leave_k_minus_1_closer_rows_and_go_to_the_lowest_id(k, permute):
    g = torch.Generator().manual_seed(k)
    q, n, h = 3, 2000, 128
    queries = exact.int_matrix(q, h, 8, g)
    corpus = exact.int_matrix(n, h, 4, g)
    rows = [[900, 17, 1500], [3, 4], [1999, 1000, 5, 600]]
    ol2.planted_ties(queries, corpus, k, rows, g, permute=permute)
    dist = ol2.l2_matrix(queries, corpus)
    for qi in range(q):
        assert int((dist[qi] < 15).sum()) == k - 1 and int((dist[qi] == 15).sum()) == len(rows[qi])
        tied = corpus[torch.tensor(rows[qi])]
        assert (len(torch.unique(tied, dim=0)) == len(rows[qi])) == permute
    d, i = ol2.numpy_reference(queries, corpus, k)
    assert i[:, -1].tolist() == [min(r) for r in rows] and (d[:, -1] == 15).all()


# the retriever blocks of the reference's examples/evaluate/*.yaml (amp_pubmedbert_mistral,
# amp_pubmedbert_mixtral, pro_pubmedbert_mixtral), with the cluster path replaced by a local directory
EVALUATE_RETRIEVERS = {
    'amp_pubmedbert_mistral': """
faiss_config:
  name: faiss_index_v1
  dataset_dir: {dataset_dir}
encoder_config:
  name: auto
  pretrained_model_name_or_path: pritamdeka/S-PubMedBert-MS-MARCO
pooler_config:
  name: mean
""",
    'amp_pubmedbert_mixtral': """
faiss_config:
  name: faiss_index_v1
  dataset_dir: {dataset_dir}
encoder_config:
  name: auto
  pretrained_model_name_or_path: pritamdeka/S-PubMedBert-MS-MARCO
pooler_config:
  name: mean
""",
    'pro_pubmedbert_mixtral': """
faiss_config:
  name: faiss_index_v1
  dataset_dir: {dataset_dir}
encoder_config:
  name: auto
  pretrained_model_name_or_path: pritamdeka/S-PubMedBert-MS-MARCO
pooler_config:
  name: mean
""",
}


@pytest.mark.parametrize('which', sorted(EVALUATE_RETRIEVERS))
def test_reference_evaluate_retriever_blocks_validate(tmp_path, which):
    path = tmp_path / 'r.yaml'
    path.write_text(EVALUATE_RETRIEVERS[which].format(dataset_dir=tmp_path / 'ds'))
    cfg = RetrieverConfig.from_yaml(path)
    fc = cfg.faiss_config
    assert isinstance(fc, FaissIndexV1Config)
    assert (fc.dataset_dir, fc.faiss_index_path, fc.faiss_index_name, fc.metric) == \
        (tmp_path / 'ds', None, 'embeddings', 'inner_product')
    cfg.write_yaml(tmp_path / 'back.yaml')
    assert RetrieverConfig.from_yaml(tmp_path / 'back.yaml') == cfg


def test_index_config_is_chosen_by_name(tmp_path):
    def faiss(fc):
        return RetrieverConfig(faiss_config=fc, encoder_config={}, pooler_config={}).faiss_config

    assert type(faiss({})) is ExactIndexConfig
    assert type(faiss({'name': 'faiss_index_v2', 'precision': 'ubinary'})) is ExactIndexConfig
    v1 = faiss({'name': 'faiss_index_v1', 'dataset_dir': str(tmp_path), 'metric': 'l2',
                'faiss_index_path': str(tmp_path / 'x.index'), 'faiss_index_name': 'emb'})
    assert type(v1) is FaissIndexV1Config and (v1.metric, v1.faiss_index_name) == ('l2', 'emb')
    for bad in ({'name': 'faiss_index_v1'}, {'name': 'faiss_index_v1', 'dataset_dir': '.', 'metric': 'cosine'},
                {'name': 'hnsw_index'}):
        with pytest.raises(ValueError):
            faiss(bad)
    assert yaml.safe_load(yaml.safe_dump({'m': v1.metric}))['m'] == 'l2'


def test_threshold_keeps_le_for_l2_and_ge_for_inner_product():
    res = BatchedSearchResults(total_scores=[[0.5, 1.0, 1.5, 2.0], [3.0]], total_indices=[[7, 3, 9, 1], [4]])
    l2 = filter_search_by_score(res, 1.0, 'l2')
    assert l2.total_indices == [[7, 3], []] and l2.total_scores == [[0.5, 1.0], []]
    ip = filter_search_by_score(res, 1.5, 'inner_product')
    assert ip.total_indices == [[9, 1], [4]] and ip.total_scores == [[1.5, 2.0], [3.0]]
    assert filter_search_by_score(res, 1.5).total_indices == ip.total_indices   # the default stays inner product
    for metric in ('l2', 'inner_product'):   # 0.0 keeps everything, as in the reference
        assert filter_search_by_score(res, 0.0, metric) is res


def test_v1_transform_normalises_only_for_inner_product(tmp_path):
    x = np.array([[3.0, 4.0], [0.0, 0.0]], dtype=np.float32)
    index = object.__new__(FaissIndexV1)   # transform needs no device
    index.metric = 'l2'
    assert np.array_equal(index.transform(x.copy()), x)
    index.metric = 'inner_product'
    assert np.allclose(index.transform(x.copy()), [[0.6, 0.8], [0.0, 0.0]])


def test_get_texts_and_embeddings_from_an_on_disk_dataset(tmp_path):
    n, h = 40, 8
    emb = np.arange(n * h, dtype=np.float32).reshape(n, h) / 7
    Dataset.from_dict({'text': [f'chunk {i}' for i in range(n)], 'path': [f'doc{i % 3}' for i in range(n)],
                       'embeddings': emb.tolist()}).save_to_disk(str(tmp_path / 'ds'))
    index = object.__new__(FaissIndexV1)   # the dataset side of the index needs no device
    index.config = FaissIndexV1Config(dataset_dir=tmp_path / 'ds', metric='l2')
    column = index._load_dataset('embeddings')
    assert column.dtype == np.float32 and np.array_equal(column, emb)
    assert index.dataset.column_names == ['text', 'path', 'embeddings']
    retriever = Retriever(encoder=None, pooler=None, faiss_index=index)
    order = [31, 2, 2, 17, 0]
    assert retriever.get_texts(order) == [f'chunk {i}' for i in order]
    assert retriever.get(order, 'path') == [f'doc{i % 3}' for i in order]
    got = retriever.get_embeddings(order)
    assert got.shape == (5, h) and np.array_equal(got.astype(np.float32), emb[order])
    assert retriever.get_texts([]) == []
    bare = object.__new__(ExactIndex)
    bare.dataset = None
    with pytest.raises(ValueError, match='in-memory matrix'):
        Retriever(encoder=None, pooler=None, faiss_index=bare).get_texts([1])
