"""-m gpu: the small encoders -- head_dim-32 attention and the 384 / 640-wide row kernels.

all-MiniLM-L6-v2, bge-small-en-v1.5 and e5-small-v2 are BERT checkpoints of H = 384 (12 heads x 32, I = 1536);
esm2_t30_150M is ESM-2 at H = 640 (20 heads x 32, I = 2560).  Kernel by kernel against torch, the whole forward pass
against the reference's golden vectors (tests/golden/*_d32_golden.npz, tools/make_golden_small.py) and at full depth
against the CPU oracle, and end to end through the plugin API from a checkpoint directory."""

from __future__ import annotations

import numpy as np
import pytest
import torch
from transformers import BatchEncoding

from distllm_b200 import _native as nv
from oracle import pooling as opool
from tools.workloads import add_outliers

from conftest import GOLDEN
from conftest import cosine_rows

pytestmark = pytest.mark.gpu
COS_TOL = 1e-3


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


@pytest.fixture(params=[torch.float16, torch.bfloat16], ids=['f16', 'bf16'])
def h16(request):
    return request.param


@pytest.fixture(params=['bf16', 'f16'])
def storage(request):
    return request.param


def close(got, ref, h16, scale: float = 1.0):
    t = (3e-3 if h16 == torch.float16 else 1.2e-2) * scale
    torch.testing.assert_close(got, ref, rtol=t, atol=t)


def bert_d32_config(layers: int = 2, **kw):
    from transformers import BertConfig

    from tools.make_golden_small import BERT_D32

    return BertConfig(**{**BERT_D32, 'num_hidden_layers': layers, **kw})


def esm_d32_config(layers: int = 2, **kw):
    from transformers import EsmConfig

    from tools.make_golden_small import ESM_D32

    return EsmConfig(**{**ESM_D32, 'num_hidden_layers': layers, **kw})


# ---------------------------------------------------------------------------------- attention, head_dim 32
def ref_attention_d32(qkv, mask, b, s, heads):
    q, k, v = qkv.float().view(b, s, 3, heads, 32).unbind(2)
    q, k, v = (t.permute(0, 2, 1, 3) for t in (q, k, v))
    bias = torch.zeros(b, 1, 1, s, device=qkv.device)
    bias.masked_fill_(mask.view(b, 1, 1, s) == 0, torch.finfo(torch.float32).min)
    p = torch.softmax(q @ k.transpose(-1, -2) / 32 ** 0.5 + bias, dim=-1)
    return (p @ v).permute(0, 2, 1, 3).reshape(b * s, heads * 32)


def check_attention_rows(ctx, ref, h16, rows=None):
    """1 - cos <= 1e-3 per output row (per head) and the d64 kernel tests' elementwise tolerance."""
    got, ref = ctx.float(), ref
    if rows is not None:
        got, ref = got[rows], ref[rows]
    assert torch.isfinite(got).all()
    cos = torch.nn.functional.cosine_similarity(got.view(-1, 32), ref.reshape(-1, 32), dim=-1)
    live = ref.reshape(-1, 32).norm(dim=-1) > 1e-3
    assert (1 - cos[live]).max().item() <= 1e-3
    close(got, ref, h16, 2.0)


@pytest.mark.parametrize('s', [1, 63, 64, 65, 129, 512, 1026])
@pytest.mark.parametrize('padding', ['none', 'right', 'left'])
def test_attention_d32_matches_reference(dev, s, padding, h16):
    b, heads = 3, 12
    g = torch.Generator(device=dev).manual_seed(s * 10 + len(padding))
    qkv = torch.randn(b * s, 3 * heads * 32, device=dev, generator=g).to(h16)
    lens = [s, max(1, s - 17), max(1, s // 3)] if padding != 'none' else [s] * b
    pos = torch.arange(s, device=dev)[None]
    lens_t = torch.tensor(lens, device=dev)[:, None]
    mask = (pos < lens_t if padding != 'left' else pos >= s - lens_t).long()
    ctx = nv.attention_d32(qkv, mask, b, s, heads)
    ref = ref_attention_d32(qkv, mask, b, s, heads)
    rows = None if padding == 'left' else mask.bool().view(-1)   # queries inside left padding: finite, never read
    check_attention_rows(ctx, ref, h16, rows if padding == 'right' else None)


def test_attention_d32_fully_masked_row_and_holes(dev, h16):
    """An all-zero mask row degenerates to a uniform softmax over the S keys (HF's additive mask); holes anywhere."""
    b, s, heads = 3, 200, 4
    g = torch.Generator(device=dev).manual_seed(9)
    qkv = torch.randn(b * s, 3 * heads * 32, device=dev, generator=g).to(h16)
    mask = torch.ones(b, s, dtype=torch.int64, device=dev)
    mask[0, 10:80] = 0
    mask[2, :] = 0
    ctx = nv.attention_d32(qkv, mask, b, s, heads)
    check_attention_rows(ctx, ref_attention_d32(qkv, mask, b, s, heads), h16)


def test_attention_d32_many_items_and_rescale(dev, h16):
    """More CTAs than SMs over ragged rows, and key norms growing along S (online-softmax rescales)."""
    b, s, heads = 40, 300, 12
    g = torch.Generator(device=dev).manual_seed(77)
    qkv = torch.randn(b * s, 3 * heads * 32, device=dev, generator=g)
    qkv[:, heads * 32:2 * heads * 32] *= torch.linspace(0.2, 5.0, s, device=dev).repeat(b)[:, None]
    qkv = qkv.to(h16)
    lens = torch.randint(1, s + 1, (b,), generator=torch.Generator().manual_seed(5))
    mask = (torch.arange(s)[None] < lens[:, None]).long().to(dev)
    ctx = nv.attention_d32(qkv, mask, b, s, heads)
    check_attention_rows(ctx, ref_attention_d32(qkv, mask, b, s, heads), h16, mask.bool().view(-1))


# ---------------------------------------------------------------------------------- row kernels at 384 / 640
@pytest.mark.parametrize('h', [384, 640])
def test_layernorm_half_pass_widths(dev, h, h16):
    g = torch.Generator(device=dev).manual_seed(h)
    x = (torch.randn(1003, h, device=dev, generator=g) * 3 + 1).to(h16)
    gamma = torch.randn(h, device=dev, generator=g)
    beta = torch.randn(h, device=dev, generator=g)
    ref = torch.nn.functional.layer_norm(x.float(), (h,), gamma, beta, 1e-12)
    torch.testing.assert_close(nv.layernorm(x, gamma, beta, 1e-12, torch.float32), ref, rtol=1e-4, atol=1e-4)
    close(nv.layernorm(x, gamma, beta, 1e-12).float(), ref, h16, 2.0)


@pytest.mark.parametrize('h', [384, 640])
def test_pool_mean_half_pass_widths(dev, h):
    """Both pool kinds: the reference's cross-row quirk (mean.py:36) with its in-place mask edit, and per row."""
    g = torch.Generator().manual_seed(h)
    lens = [20, 5, 1, 2, 11, 11, 19, 0]
    s = 20
    emb = torch.randn(len(lens), s, h, generator=g)
    mask = (torch.arange(s)[None] < torch.tensor(lens)[:, None]).long()
    m_ref = mask.clone()
    ref = opool.average_pool(emb, m_ref)
    m = mask.to(dev)
    got = nv.pool_mean(emb.to(dev), m)
    torch.testing.assert_close(got.cpu(), ref, rtol=1e-5, atol=1e-6)
    assert torch.equal(m.cpu(), m_ref)
    lens2 = [20, 7, 12, 2]
    mask2 = (torch.arange(s)[None] < torch.tensor(lens2)[:, None]).long()
    ref2 = torch.stack([emb[i, 1:n - 1].mean(0) if n > 2 else torch.zeros(h) for i, n in enumerate(lens2)])
    m2 = mask2.to(dev)
    got2 = nv.pool_mean(emb[:4].contiguous().to(dev), m2, nv.POOL_MEAN_PER_ROW, mutate_mask=False)
    torch.testing.assert_close(got2.cpu(), ref2, rtol=1e-5, atol=1e-6)
    assert torch.equal(m2.cpu(), mask2)
    for dtype in (torch.bfloat16, torch.float16):
        e16 = emb.to(dtype)
        ref16 = opool.average_pool(e16.float(), mask.clone())
        torch.testing.assert_close(nv.pool_mean(e16.to(dev), mask.to(dev)).cpu(), ref16, rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize('h', [384, 640])
def test_pool_last_token_half_pass_widths(dev, h):
    g = torch.Generator().manual_seed(h + 1)
    emb = torch.randn(4, 10, h, generator=g)
    for mask in ((torch.arange(10)[None] < torch.tensor([10, 3, 7, 1])[:, None]).long(),
                 (torch.arange(10)[None] >= torch.tensor([0, 3, 7, 9])[:, None]).long()):
        got = nv.pool_last_token(emb.to(dev), mask.to(dev))
        np.testing.assert_array_equal(got.cpu().numpy(), opool.last_token_pool(emb, mask.clone()).numpy())


# ---------------------------------------------------------------------------------- reference parity (golden)
class TokenBatches(torch.utils.data.Dataset):
    """Pre-tokenised batches behind the DataLoader interface the embedders consume."""

    def __init__(self, batches):
        self.batches = batches
        self.data = [f'row{i}' for i in range(sum(len(b['input_ids']) for b in batches))]
        self.metadata = None

    def __len__(self):
        return len(self.data)

    def __getitem__(self, i):
        return BatchEncoding(self.batches[i])


def _loader(batches):
    return torch.utils.data.DataLoader(TokenBatches(batches), batch_size=None, sampler=range(len(batches)))


def test_bert_d32_matches_reference_vectors(storage):
    """MiniLM-width BERT (H = 384, 12 x 32) vs the reference's AutoEncoder + poolers + compute_embeddings."""
    from distllm_b200.embed import get_embedder
    from distllm_b200.embed import get_pooler
    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.native import NativeBertEncoder
    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    from oracle.make_golden import TINY_SEED
    from oracle.make_golden import weights_digest

    golden = np.load(GOLDEN / 'bert_d32_golden.npz')
    cfg = bert_d32_config()
    sd = random_bert_state_dict(cfg, seed=TINY_SEED, device='cpu')
    assert weights_digest(sd) == str(golden['weights_sha256'])
    batches = [{k: torch.from_numpy(golden[f'batch{i}/{k}']) for k in ('input_ids', 'attention_mask', 'token_type_ids')}
               for i in range(int(golden['n_batches']))]
    native = NativeBertEncoder(cfg, sd, storage=storage)
    try:
        b = batches[0]
        hidden = native.encode(b['input_ids'], b['attention_mask'], b['token_type_ids']).cpu().numpy()
        ref = golden['batch0/hidden']
        assert cosine_rows(hidden.reshape(-1, 384), ref.reshape(-1, 384)).min() > 1 - COS_TOL
        encoder = AutoEncoder.from_native(native)
        for kind, pooler, normalize in (('mean', 'mean', False), ('mean_normalized', 'mean', True),
                                        ('last_token', 'last_token', False)):
            result = get_embedder({'name': 'full_sequence', 'normalize_embeddings': normalize}).embed(
                _loader(batches), encoder, get_pooler({'name': pooler}))
            cos = cosine_rows(result.embeddings, golden[f'pooled/{kind}'])
            assert cos.min() > 1 - COS_TOL, (kind, cos)
    finally:
        native.close()


def test_esm_d32_matches_reference_vectors(storage):
    """ESM2-150M-width ESM-2 (H = 640, 20 x 32, rotary, token dropout) vs the reference's Esm2Encoder."""
    from distllm_b200.embed import get_embedder
    from distllm_b200.embed import get_pooler
    from distllm_b200.embed.encoders.esm2 import Esm2Encoder
    from distllm_b200.embed.encoders.native import NativeEsm2Encoder
    from distllm_b200.embed.encoders.weights import random_esm_state_dict
    from oracle.make_golden import TINY_ESM_SEED
    from oracle.make_golden import weights_digest

    golden = np.load(GOLDEN / 'esm_d32_golden.npz')
    cfg = esm_d32_config()
    sd = random_esm_state_dict(cfg, seed=TINY_ESM_SEED, device='cpu')
    assert weights_digest(sd) == str(golden['weights_sha256'])
    batches = [{k: torch.from_numpy(golden[f'batch{i}/{k}']) for k in ('input_ids', 'attention_mask')}
               for i in range(int(golden['n_batches']))]
    native = NativeEsm2Encoder(cfg, sd, storage=storage)
    try:
        encoder = Esm2Encoder.from_native(native)
        hidden = encoder.encode(BatchEncoding(batches[0])).cpu().numpy()
        valid = batches[0]['attention_mask'].bool().numpy()
        assert cosine_rows(hidden[valid], golden['batch0/hidden_attended']).min() > 1 - COS_TOL
        result = get_embedder({'name': 'full_sequence'}).embed(_loader(batches), encoder, get_pooler({'name': 'mean'}))
        cos = cosine_rows(result.embeddings, golden['pooled/mean'])
        assert cos.min() > 1 - COS_TOL, cos
    finally:
        native.close()


# ---------------------------------------------------------------------------------- packed == padded
@pytest.mark.parametrize('family', ['bert', 'esm'])
def test_packed_layout_equals_padded_d32(family):
    import ctypes

    from distllm_b200.embed.encoders.native import NativeBertEncoder
    from distllm_b200.embed.encoders.native import NativeEsm2Encoder
    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    from distllm_b200.embed.encoders.weights import random_esm_state_dict

    if family == 'bert':
        cfg = bert_d32_config(max_position_embeddings=512)
        enc = NativeBertEncoder(cfg, random_bert_state_dict(cfg, seed=1, device='cpu'))
    else:
        cfg = esm_d32_config(max_position_embeddings=1026)
        enc = NativeEsm2Encoder(cfg, random_esm_state_dict(cfg, seed=2, device='cpu'))
    lib = enc._lib
    lib.b2e_debug_set_packing.argtypes = [ctypes.c_int]
    g = torch.Generator().manual_seed(5)
    try:
        for b, s, lens in [(7, 50, [50, 3, 17, 50, 1, 33, 2]), (5, 300, [300, 129, 128, 64, 7]), (3, 40, [40] * 3)]:
            ids = torch.randint(4, 24 if family == 'esm' else cfg.vocab_size - 1, (b, s), generator=g)
            mask = (torch.arange(s)[None] < torch.tensor(lens)[:, None]).long()
            for kind in (nv.POOL_MEAN_REF, nv.POOL_MEAN_PER_ROW, nv.POOL_LAST_TOKEN):
                lib.b2e_debug_set_packing(1)
                packed = enc.encode_pooled(ids, mask, None, kind, True).clone()
                lib.b2e_debug_set_packing(0)
                padded = enc.encode_pooled(ids, mask, None, kind, True).clone()
                assert torch.isfinite(packed).all()
                live = padded.norm(dim=-1) > 0
                assert torch.equal(live, packed.norm(dim=-1) > 0)
                cos = torch.nn.functional.cosine_similarity(packed[live], padded[live])
                assert cos.min().item() > 1 - 1e-6, (family, b, s, kind, cos)
    finally:
        lib.b2e_debug_set_packing(1)
        enc.close()


# ---------------------------------------------------------------------------------- full size vs the oracle
def check_rows(got, ref, what):
    live = np.linalg.norm(ref, axis=-1) > 0
    assert np.isfinite(got).all(), what
    cos = cosine_rows(got[live], ref[live])
    assert cos.min() > 1 - COS_TOL, (what, float(cos.min()))


@pytest.mark.parametrize('weights', ['normal', 'outliers'])
@pytest.mark.parametrize('layers', [6, 12], ids=['minilm-l6', 'bge-small'])
def test_minilm_bge_full_depth_s512(layers, weights):
    from distllm_b200.embed.encoders.native import NativeBertEncoder
    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    from oracle import bert as obert

    cfg = bert_d32_config(layers, vocab_size=30522, max_position_embeddings=512, initializer_range=0.02)
    sd = random_bert_state_dict(cfg, seed=layers, device='cpu')
    if weights == 'outliers':
        add_outliers(sd, 'bert', seed=1)
    g = torch.Generator().manual_seed(31)
    b, s = 12, 512
    ids = torch.randint(7, cfg.vocab_size, (b, s), generator=g)
    lens = [512, 300, 64, 511, 129, 128, 2, 450, 17, 256, 257, 90]
    mask = (torch.arange(s)[None] < torch.tensor(lens)[:, None]).long()
    ref_hidden = obert.bert_forward(sd, cfg, ids, mask)
    enc = NativeBertEncoder(cfg, sd)
    try:
        for kind, pool in ((nv.POOL_MEAN_REF, opool.average_pool), (nv.POOL_LAST_TOKEN, opool.last_token_pool)):
            got = enc.encode_pooled(ids, mask, None, kind, False).cpu().numpy()
            check_rows(got, pool(ref_hidden, mask.clone()).numpy(), f'L{layers} {weights} pool {kind}')
    finally:
        enc.close()


@pytest.mark.parametrize('weights', ['normal', 'outliers'])
def test_esm2_150m_full_depth_s1026(weights):
    from distllm_b200.embed.encoders.native import NativeEsm2Encoder
    from distllm_b200.embed.encoders.weights import random_esm_state_dict
    from oracle import esm as oesm

    cfg = esm_d32_config(30, max_position_embeddings=1026, initializer_range=0.02)
    sd = random_esm_state_dict(cfg, seed=3, device='cpu')
    if weights == 'outliers':
        add_outliers(sd, 'esm', seed=2)
    g = torch.Generator().manual_seed(22)
    b, s = 3, 1026
    ids = torch.randint(4, 24, (b, s), generator=g)
    mask = (torch.arange(s)[None] < torch.tensor([1026, 700, 65])[:, None]).long()
    ids = ids.masked_fill(mask == 0, 1)
    ids[:, 0] = 0
    ids[0, 500:520] = 32      # <mask> tokens: token dropout
    ref = opool.average_pool(oesm.esm_forward(sd, cfg, ids, mask), mask.clone()).numpy()
    enc = NativeEsm2Encoder(cfg, sd)
    try:
        check_rows(enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_REF, False).cpu().numpy(), ref,
                   f'ESM2-150M {weights} mean')
    finally:
        enc.close()


# ---------------------------------------------------------------------------------- end to end at H = 384
def write_minilm_checkpoint(ckpt):
    from transformers import BertModel
    from transformers import BertTokenizerFast

    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    from oracle.make_golden import tiny_bert_vocab

    cfg = bert_d32_config(max_position_embeddings=128)
    model = BertModel(cfg)
    model.load_state_dict(random_bert_state_dict(cfg, seed=7, device='cpu'), strict=False)
    ckpt.mkdir(parents=True, exist_ok=True)
    (ckpt / 'vocab.txt').write_text('\n'.join(tiny_bert_vocab()) + '\n')
    tok = BertTokenizerFast(vocab=str(ckpt / 'vocab.txt'), do_lower_case=False)
    model.eval().save_pretrained(ckpt)
    tok.save_pretrained(ckpt)
    return cfg


def test_minilm_checkpoint_semantic_chunk_writer_and_search(tmp_path):
    """AutoEncoder from a checkpoint directory -> semantic_chunk embedder -> numpy writer, then Retriever.search
    over the written embeddings (float32 and ubinary) equal to a torch top-k over the same matrix."""
    import json

    from distllm_b200.embed import get_dataset
    from distllm_b200.embed import get_embedder
    from distllm_b200.embed import get_pooler
    from distllm_b200.embed import get_writer
    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig
    from distllm_b200.rag import ExactIndex
    from distllm_b200.rag import Retriever
    from distllm_b200.rag.search import ExactIndexConfig
    from oracle.make_golden import tiny_bert_vocab

    write_minilm_checkpoint(tmp_path / 'ckpt')
    encoder = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(tmp_path / 'ckpt'), quantization=False))
    assert encoder.embedding_size == 384
    words = tiny_bert_vocab()[5:]
    rng = np.random.default_rng(0)
    docs = [{'text': ''.join('S' + ' '.join(rng.choice(words, size=rng.integers(5, 9))) + '. ' for _ in range(12 + d)),
             'path': f'doc{d}'} for d in range(3)]
    f = tmp_path / 'docs.jsonl'
    f.write_text('\n'.join(json.dumps(d) for d in docs))
    dataset = get_dataset({'name': 'jsonl_chunk', 'buffer_size': 1, 'min_buffer_length': 20, 'batch_size': 5,
                           'num_data_workers': 0, 'pin_memory': False})
    embedder = get_embedder({'name': 'semantic_chunk', 'breakpoint_percentile_threshold': 80, 'chunk_batch_size': 4,
                             'min_chunk_length': 10})
    result = embedder.embed(dataset.get_dataloader(f, encoder), encoder, get_pooler({'name': 'mean'}))
    assert result.embeddings.shape[1] == 384 and np.isfinite(result.embeddings).all()
    (tmp_path / 'out').mkdir()
    get_writer({'name': 'numpy'}).write(tmp_path / 'out', result)
    emb = np.load(tmp_path / 'out' / 'embeddings.npy')
    np.testing.assert_array_equal(emb, result.embeddings)

    queries = [' '.join(rng.choice(words, size=n)) for n in (5, 30, 12)]
    k = min(5, len(emb))
    for precision in ('float32', 'ubinary'):
        # ubinary: every row a Hamming candidate (k * rescore_multiplier >= N), so the rescored top-k is the top-k of
        # q . bits over the whole matrix
        index = ExactIndex(emb, config=ExactIndexConfig(precision=precision, rescore_multiplier=len(emb) // k + 1))
        res, q_emb = Retriever(encoder, get_pooler({'name': 'mean'}), index, batch_size=4).search(queries, top_k=k)
        assert q_emb.shape == (3, 384)
        if precision == 'float32':
            scores = torch.from_numpy(q_emb).double() @ torch.from_numpy(emb).double().T
        else:   # packed bits -> {0, 1} per dimension, rescored with the float query (search.py's binary branch)
            scores = torch.from_numpy(q_emb).double() @ torch.from_numpy((emb > 0).astype(np.float64)).T
        ref_s, ref_i = torch.topk(scores, k, dim=1)
        np.testing.assert_allclose(np.array(res.total_scores), ref_s.numpy(), rtol=0, atol=2e-5)
        assert np.array(res.total_indices).tolist() == ref_i.tolist()
