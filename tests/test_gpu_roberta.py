"""-m gpu: RoBERTa / XLM-RoBERTa on the native path (B2E_ARCH_BERT with desc.reserved = padding_idx + 1).

(a) roberta_positions_kernel, through b2e_debug_roberta_positions, equals HF's rule bit for bit.
(b) The embedding row: a row-path model (oracle.rows.row_path_model, every weight matrix zero, Walsh rows in the
    position table) whose output is exact, b2e_encode and b2e_encode_pooled bit for bit, packed and padded.
(c) Two-layer models with random weights against the fp32 oracle (tools/oracle_roberta.py), both storage builds,
    right- and left-padded and pad-inside batches, and the BGE-M3 shape at S = 8192.
(d) The refusal of S + padding_idx >= max_position_embeddings, NF4 storage bit for bit against its 16-bit form, and
    the `auto` encoder on the tiny checkpoint against the reference's golden vectors."""

from __future__ import annotations

import math
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F  # noqa: N812

from distllm_b200 import _native as nv
from distllm_b200.embed.encoders import weights as W
from distllm_b200.embed.encoders.native import NativeRobertaEncoder
from oracle import pooling as opool
from oracle import rows as R
from tools import oracle_roberta as O

from conftest import cosine_rows

pytestmark = pytest.mark.gpu
PAD = 1
COS_TOL = 1e-3
GOLDEN = Path(__file__).parent / 'golden' / 'xlmr_tiny_golden.npz'


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


def set_packing(lib, on: bool) -> None:
    import ctypes as C
    import os

    lib.b2e_debug_set_packing.argtypes = [C.c_int]
    if on is None:
        on = os.environ.get('B2E_PACKED', '1')[:1] != '0'
    nv.check(lib.b2e_debug_set_packing(int(on)), lib)


def batch(lens: list[int], s: int, side: str, seed: int, vocab: int, inside: float = 0.0):
    """ids [B, S] (pad id where the mask is 0; with ``inside`` that share of attended ids is the pad id too), mask."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (len(lens), s), generator=g)
    cols = torch.arange(s)[None]
    n = torch.tensor(lens)[:, None]
    mask = (cols < n) if side == 'right' else (cols >= s - n)
    if inside:
        ids[(torch.rand(ids.shape, generator=g) < inside) & mask] = PAD
    ids[~mask] = PAD
    return ids, mask.long()


# ---------------------------------------------------------------------------------- (a) the position kernel
@pytest.mark.parametrize('s', [1, 31, 32, 33, 512, 513, 1025, 8194])
def test_position_kernel_exact(dev, s):
    b = 5
    lens = [s, max(s - 1, 1), s // 2 + 1, 1, max(s // 3, 1)]
    for side in ('right', 'left'):
        for inside in (0.0, 0.1):
            ids, _ = batch(lens, s, side, seed=s, vocab=50, inside=inside)
            for pad in (PAD, 0):
                got = nv.debug_roberta_positions(ids.to(dev), pad).cpu()
                exp = O.position_ids(ids, pad)
                assert got.dtype == torch.int32 and torch.equal(got.long(), exp), (s, side, inside, pad)
    # every id the pad id: every row reads row padding_idx
    ids = torch.full((2, s), 3, dtype=torch.int64)
    assert torch.equal(nv.debug_roberta_positions(ids.to(dev), 3).cpu().long(), torch.full((2, s), 3))


# ---------------------------------------------------------------------------------- (b) the embedding row, exact
def row_path_roberta(h: int, max_pos: int):
    """oracle.rows.row_path_model's BERT with the Walsh rows in its position table, read at RoBERTa's positions."""
    cfg, sd, _ = R.row_path_model('bert', h, 'pos', max_pos)
    cfg.pad_token_id = PAD
    eps = cfg.layer_norm_eps

    def vec(k):
        return sd[k].double().numpy()

    def reference(ids, dtype):
        x = vec('embeddings.position_embeddings.weight')[O.position_ids(ids, PAD).numpy()]   # word, type rows 0
        hdn = R.round16(R.layernorm(x, vec('embeddings.LayerNorm.weight'), vec('embeddings.LayerNorm.bias'), eps),
                        dtype)
        for layer in range(R.LAYERS):
            p = f'encoder.layer.{layer}.'
            for name, b in (('attention.output', 'attention.output.dense.bias'), ('output', 'output.dense.bias')):
                y = R.layernorm(R.round16(vec(p + b), dtype) + hdn, vec(p + name + '.LayerNorm.weight'),
                                vec(p + name + '.LayerNorm.bias'), eps)
                hdn = y if (layer == R.LAYERS - 1 and name == 'output') else R.round16(y, dtype)
        return hdn
    return cfg, sd, reference


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
@pytest.mark.parametrize('h', [384, 768, 1024])
def test_embedding_row_exact(dev, h, storage):
    cfg, sd, reference = row_path_roberta(h, max_pos=300)
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    enc = NativeRobertaEncoder(cfg, sd, device=dev, storage=storage)
    s = 129
    lens = [129, 128, 65, 2, 1]
    cases = {'right': batch(lens, s, 'right', 1, R.VOCAB), 'left': batch(lens, s, 'left', 2, R.VOCAB),
             'inside': batch(lens, s, 'right', 3, R.VOCAB, inside=0.2)}
    try:
        for name, (ids, mask) in cases.items():
            y = reference(ids, dtype)
            got = enc.encode(ids, mask, None, torch.float32).cpu().numpy()
            assert np.array_equal(got, y.astype(np.float32)), (h, storage, name, 'encode')
            refs = {nv.POOL_MEAN_REF: R.mean_pool(y, R.pool_weights(mask, 'ref')),
                    nv.POOL_MEAN_PER_ROW: R.mean_pool(y, R.pool_weights(mask, 'per_row')),
                    nv.POOL_LAST_TOKEN: R.last_token(y, mask)}
            for packed in (True, False):
                set_packing(enc._lib, packed)
                for code, exp in refs.items():
                    got = enc.encode_pooled(ids, mask, None, code, False).cpu().numpy()
                    assert np.array_equal(got, exp), (h, storage, name, code, packed)
                # the embedding step alone, in the layout the pooled pass uses
                out16, _ = nv.debug_embed(enc, ids.to(dev), mask.to(dev))
                first = R.round16(R.layernorm(
                    sd['embeddings.position_embeddings.weight'].double().numpy()[O.position_ids(ids, PAD).numpy()],
                    sd['embeddings.LayerNorm.weight'].double().numpy(), sd['embeddings.LayerNorm.bias'].double().numpy(),
                    cfg.layer_norm_eps), dtype)
                prefix = name != 'left'
                exp = first[mask.bool().numpy()] if packed and prefix else first.reshape(-1, h)
                assert np.array_equal(out16.float().cpu().numpy()[:len(exp)], exp), (h, storage, name, packed)
    finally:
        set_packing(enc._lib, None)
        enc.close()


# ---------------------------------------------------------------------------------- (c) against the fp32 oracle
def xlmr_config(h, heads, inter, layers=2, vocab=1000, max_pos=514):
    from transformers import XLMRobertaConfig

    return XLMRobertaConfig(vocab_size=vocab, hidden_size=h, num_hidden_layers=layers, num_attention_heads=heads,
                            intermediate_size=inter, max_position_embeddings=max_pos, type_vocab_size=1,
                            pad_token_id=PAD, layer_norm_eps=1e-5)


def assert_cos(got: np.ndarray, exp: np.ndarray, *what) -> None:
    """1 - cos <= COS_TOL per row; a row the reference pools to zero (the reference mean pooler's quirk clears every
    token of a two-token row) must be zero too."""
    zero = ~exp.any(-1)
    assert not got[zero].any(), (*what, 'rows pooled to zero by the reference', np.flatnonzero(zero))
    cos = cosine_rows(got[~zero], exp[~zero])
    assert (1 - cos).max() <= COS_TOL, (*what, cos)


def pooled_refs(y: np.ndarray, mask: torch.Tensor) -> dict[int, np.ndarray]:
    out = {nv.POOL_MEAN_REF: opool.average_pool(torch.from_numpy(y).double(), mask.clone()).numpy()}
    w = R.pool_weights(mask, 'per_row')
    out[nv.POOL_MEAN_PER_ROW] = np.einsum('bs,bsh->bh', w, y) / np.maximum(w.sum(1), 1e-9)[:, None]
    out[nv.POOL_LAST_TOKEN] = opool.last_token_pool(torch.from_numpy(y).double(), mask.clone()).numpy()
    return out


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
@pytest.mark.parametrize('h,heads,inter', [(384, 12, 1536), (768, 12, 3072), (1024, 16, 4096)])
def test_two_layer_vs_oracle(dev, h, heads, inter, storage):
    cfg = xlmr_config(h, heads, inter)
    sd = W.random_bert_state_dict(cfg, seed=h)
    enc = NativeRobertaEncoder(cfg, sd, device=dev, storage=storage)
    s = 300
    lens = [300, 257, 128, 64, 33, 2]
    cases = {'right': batch(lens, s, 'right', 4, 1000), 'left': batch(lens, s, 'left', 5, 1000),
             'inside': batch(lens, s, 'right', 6, 1000, inside=0.1)}
    try:
        for name, (ids, mask) in cases.items():
            y = O.roberta_forward(sd, cfg, ids, mask).double().numpy()
            for code, exp in pooled_refs(y, mask).items():
                got = enc.encode_pooled(ids, mask, None, code, False).cpu().numpy()
                assert_cos(got, exp, h, storage, name, code)
            hidden = enc.encode(ids, mask).cpu().numpy()
            m = mask.bool().numpy()
            cos = cosine_rows(hidden[m], y[m])
            assert (1 - cos).max() <= COS_TOL, (h, storage, name, 'tokens', cos.min())
    finally:
        enc.close()


@torch.no_grad()
def forward_fp32_device(sd, cfg, ids, mask):
    """oracle/bert.py's block, on the device in fp32 (TF32 off) at RoBERTa's positions: the S = 8192 score matrices
    do not fit a CPU restatement's time."""
    b, s = ids.shape
    h, heads = cfg.hidden_size, cfg.num_attention_heads
    d, eps = h // heads, cfg.layer_norm_eps
    x = (sd['embeddings.word_embeddings.weight'][ids] + sd['embeddings.token_type_embeddings.weight'][0]
         + sd['embeddings.position_embeddings.weight'][O.position_ids(ids, PAD)])
    x = F.layer_norm(x, (h,), sd['embeddings.LayerNorm.weight'], sd['embeddings.LayerNorm.bias'], eps)
    bias = torch.zeros(b, 1, 1, s, device=ids.device)
    bias.masked_fill_(mask.view(b, 1, 1, s) == 0, torch.finfo(torch.float32).min)
    for layer in range(cfg.num_hidden_layers):
        p = f'encoder.layer.{layer}.'

        def lin(t, name):
            return F.linear(t, sd[p + name + '.weight'], sd[p + name + '.bias'])

        q, k, v = (lin(x, f'attention.self.{n}').view(b, s, heads, d).transpose(1, 2)
                   for n in ('query', 'key', 'value'))
        ctx = torch.cat([torch.softmax(q[i:i + 1] @ k[i:i + 1].transpose(-1, -2) / math.sqrt(d) + bias[i:i + 1], -1)
                         @ v[i:i + 1] for i in range(b)]).transpose(1, 2).reshape(b, s, h)   # one sequence at a time
        x = F.layer_norm(lin(ctx, 'attention.output.dense') + x, (h,), sd[p + 'attention.output.LayerNorm.weight'],
                         sd[p + 'attention.output.LayerNorm.bias'], eps)
        x = F.layer_norm(lin(F.gelu(lin(x, 'intermediate.dense')), 'output.dense') + x, (h,),
                         sd[p + 'output.LayerNorm.weight'], sd[p + 'output.LayerNorm.bias'], eps)
    return x


def test_bge_m3_shape_at_8192(dev):
    cfg = xlmr_config(1024, 16, 4096, vocab=250002, max_pos=8194)
    sd = W.random_bert_state_dict(cfg, seed=3, device=dev)
    enc = NativeRobertaEncoder(cfg, sd, device=dev, storage='bf16')
    assert enc.max_positions == 8192
    ids, mask = batch([8192, 5001], 8192, 'right', 7, 250002, inside=0.01)
    ids, mask = ids.to(dev), mask.to(dev)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        y = forward_fp32_device(sd, cfg, ids, mask).double().cpu().numpy()
        for code, exp in pooled_refs(y, mask.cpu()).items():
            got = enc.encode_pooled(ids, mask, None, code, False).cpu().numpy()
            assert_cos(got, exp, code)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
        enc.close()


# ---------------------------------------------------------------------------------- (d) refusal, NF4, auto
def test_refuses_rows_past_the_position_table(dev):
    cfg, sd = O.tiny_xlmr_state_dict()                      # 66 position rows, padding_idx 1: S <= 64
    enc = NativeRobertaEncoder(cfg, sd, device=dev)
    try:
        ids, mask = batch([64, 10], 64, 'right', 8, 200)
        assert enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_REF, False).isfinite().all()
        ids, mask = batch([65, 10], 65, 'right', 8, 200)
        out = torch.full((2, cfg.hidden_size), 7.0, device=dev)
        with pytest.raises(nv.NativeError, match=r'S=65 .*66 rows'):
            enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_REF, False, out=out)
        assert (out == 7.0).all()
        with pytest.raises(nv.NativeError, match=r'S=65 .*66 rows'):
            enc.encode(ids, mask)
        with pytest.raises(nv.NativeError, match=r'S=65 .*66 rows'):
            enc.embed_host(ids.pin_memory(), mask.pin_memory(), None, 2, nv.POOL_MEAN_REF, False)
        torch.cuda.synchronize()
    finally:
        enc.close()


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
def test_nf4_equals_16bit_on_dequantised_weights(dev, storage):
    from distllm_b200.embed.encoders.nf4 import quantize_state_dict_nf4

    cfg = xlmr_config(768, 12, 3072)
    sd = W.random_bert_state_dict(cfg, seed=11)
    nf4 = NativeRobertaEncoder(cfg, sd, device=dev, storage=storage, nf4=True)
    b16 = NativeRobertaEncoder(cfg, quantize_state_dict_nf4(sd, device=dev), device=dev, storage=storage)
    try:
        for side, inside in (('right', 0.0), ('left', 0.0), ('right', 0.1)):
            ids, mask = batch([200, 150, 3], 200, side, 9, 1000, inside)
            for code in (nv.POOL_MEAN_REF, nv.POOL_MEAN_PER_ROW, nv.POOL_LAST_TOKEN):
                a = nf4.encode_pooled(ids, mask, None, code, False)
                b = b16.encode_pooled(ids, mask, None, code, False)
                assert torch.equal(a, b), (side, inside, code)
    finally:
        nf4.close()
        b16.close()


@pytest.fixture(scope='module')
def tiny_ckpt(tmp_path_factory):
    path = tmp_path_factory.mktemp('xlmr') / 'ckpt'
    O.write_tiny_xlmr_checkpoint(path)
    return path


def test_auto_encoder_matches_golden(dev, tiny_ckpt):
    from distllm_b200.embed import get_embedder
    from distllm_b200.embed import get_pooler
    from distllm_b200.embed.datasets.utils import DataCollator
    from distllm_b200.embed.datasets.utils import InMemoryDataset
    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig

    enc = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(tiny_ckpt), quantization=False))
    assert isinstance(enc.native, NativeRobertaEncoder)
    assert enc.tokenizer.model_max_length == 64
    texts = O.tiny_xlmr_texts()

    def loader():
        return torch.utils.data.DataLoader(InMemoryDataset(texts), batch_size=4, num_workers=0,
                                           collate_fn=DataCollator(enc.tokenizer))

    with np.load(GOLDEN) as z:
        for i, b in enumerate(loader()):
            assert np.array_equal(b['input_ids'].numpy(), z[f'batch{i}/input_ids'])
            if i == 0:
                hidden = enc.encode(b).cpu().numpy()
                m = z['batch0/attention_mask'].astype(bool)
                cos = cosine_rows(hidden[m], z['batch0/hidden'][m])
                assert (1 - cos).max() <= COS_TOL, cos.min()
        for kind, pooler, normalize in (('mean', 'mean', False), ('mean_normalized', 'mean', True),
                                        ('last_token', 'last_token', False)):
            embedder = get_embedder({'name': 'full_sequence', 'normalize_embeddings': normalize})
            got = embedder.embed(loader(), enc, get_pooler({'name': pooler})).embeddings
            assert_cos(got, z[f'pooled/{kind}'], kind)
    enc.native.close()


def test_auto_encoder_default_quantization(dev, tiny_ckpt):
    """quantization: true (the default) holds the BERT-slot matrices in NF4: the oracle on dequant(quant(W))."""
    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig
    from distllm_b200.embed.encoders.nf4 import quantize_state_dict_nf4

    enc = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(tiny_ckpt)))
    assert enc.native.nf4
    cfg, sd = O.tiny_xlmr_state_dict()
    ids, mask = batch([64, 40, 5], 64, 'right', 10, 200, inside=0.05)
    y = O.roberta_forward(quantize_state_dict_nf4(sd), cfg, ids, mask).double().numpy()
    for code, exp in pooled_refs(y, mask).items():
        got = enc.native.encode_pooled(ids, mask, None, code, False).cpu().numpy()
        assert_cos(got, exp, code)
    enc.native.close()
