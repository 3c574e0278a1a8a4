"""RoBERTa / XLM-RoBERTa on the host (no device): the oracle (tools/oracle_roberta.py) against the reference's golden
vectors and HF's position rule, the shapes b2e_check_model accepts through the RoBERTa description, what `validate`
refuses, the tokenizer length, and the collator's ids for a SentencePiece-style fast tokenizer."""

from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from distllm_b200 import _native
from distllm_b200.embed.encoders import weights as W
from tools import oracle_roberta as O

GOLDEN = Path(__file__).parent / 'golden' / 'xlmr_tiny_golden.npz'
ERR_INVALID = 1   # B2E_ERR_INVALID


def xlmr_config(**kw):
    from transformers import XLMRobertaConfig

    base = dict(vocab_size=250002, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                intermediate_size=3072, max_position_embeddings=514, type_vocab_size=1, pad_token_id=1,
                layer_norm_eps=1e-5)
    base.update(kw)
    return XLMRobertaConfig(**base)


def test_oracle_equals_golden():
    from oracle import make_golden as mg

    cfg, sd = O.tiny_xlmr_state_dict()
    with np.load(GOLDEN) as z:
        assert str(z['weights_sha256']) == mg.weights_digest(sd)
        ids, mask = torch.from_numpy(z['batch0/input_ids']), torch.from_numpy(z['batch0/attention_mask'])
        hidden = z['batch0/hidden']
        n = int(z['n_batches'])
        batches = [(torch.from_numpy(z[f'batch{i}/input_ids']), torch.from_numpy(z[f'batch{i}/attention_mask']))
                   for i in range(n)]
        last = z['pooled/last_token']
    assert (ids == 1).logical_and(mask == 1).any(), 'the first batch holds a <pad> id inside the attended text'
    got = O.roberta_forward(sd, cfg, ids, mask).numpy()
    m = mask.numpy().astype(bool)
    np.testing.assert_allclose(got[m], hidden[m], rtol=0, atol=2e-5)
    # last-token pooling of every batch: the row's last attended token (right padding)
    rows = []
    for bids, bmask in batches:
        y = O.roberta_forward(sd, cfg, bids, bmask)
        rows.append(y[torch.arange(len(bids)), bmask.sum(1) - 1].numpy())
    np.testing.assert_allclose(np.concatenate(rows), last, rtol=0, atol=2e-5)


def test_golden_ids_are_the_collators():
    from distllm_b200.embed.datasets.utils import DataCollator

    tok = O.tiny_xlmr_tokenizer()
    tok.model_max_length = W.roberta_max_length(O.tiny_xlmr_state_dict()[0])
    texts = O.tiny_xlmr_texts()
    with np.load(GOLDEN) as z:
        for i in range(int(z['n_batches'])):
            batch = DataCollator(tok)(texts[4 * i: 4 * i + 4])
            assert np.array_equal(batch['input_ids'].numpy(), z[f'batch{i}/input_ids'])
            assert np.array_equal(batch['attention_mask'].numpy(), z[f'batch{i}/attention_mask'])


@pytest.mark.parametrize('side', ['right', 'left'])
def test_position_rule_equals_hf(side):
    from transformers.models.xlm_roberta.modeling_xlm_roberta import XLMRobertaEmbeddings

    g = torch.Generator().manual_seed(3)
    for pad in (1, 0, 5):
        ids = torch.randint(0, 8, (16, 77), generator=g)       # pad ids inside rows
        lens = torch.randint(0, 78, (16,), generator=g)
        cols = torch.arange(77)[None]
        padded = cols >= lens[:, None] if side == 'right' else cols < (77 - lens)[:, None]
        ids[padded] = pad
        exp = XLMRobertaEmbeddings.create_position_ids_from_input_ids(ids, pad)
        assert torch.equal(O.position_ids(ids, pad), exp)
    # the three consequences, spelled out
    pos = O.position_ids(torch.tensor([[0, 7, 1, 7, 2, 1, 1], [1, 1, 0, 7, 7, 7, 2]]), 1)
    assert pos.tolist() == [[2, 3, 1, 4, 5, 1, 1], [1, 1, 2, 3, 4, 5, 6]]


# multilingual-e5-small / paraphrase-multilingual-MiniLM-L12-v2, xlm-roberta-base / e5-base, BGE-M3 / e5-large,
# all-distilroberta-v1
PUBLISHED = {
    'e5-small': dict(hidden_size=384, num_attention_heads=12, intermediate_size=1536, num_hidden_layers=12),
    'base': dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12),
    'bge-m3': dict(hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
                   max_position_embeddings=8194),
    'distilroberta': dict(vocab_size=50265, hidden_size=768, num_attention_heads=12, intermediate_size=3072,
                          num_hidden_layers=6),
}


@pytest.mark.parametrize('name', list(PUBLISHED))
def test_check_model_accepts_published_shapes(name):
    from distllm_b200.embed.encoders.native import NativeRobertaEncoder

    cfg = xlmr_config(**PUBLISHED[name])
    desc = W.roberta_desc(cfg)
    assert desc.arch == _native.ARCH_BERT and desc.reserved == cfg.pad_token_id + 1
    lib = _native.load()
    assert lib.b2e_check_model(C.byref(desc)) == 0, lib.b2e_last_error()
    assert lib.b2e_num_weights(C.byref(desc)) == 5 + 12 * cfg.num_hidden_layers
    NativeRobertaEncoder.validate(cfg)


@pytest.mark.parametrize('shape', [dict(hidden_size=320, num_attention_heads=20),     # head_dim 16
                                   dict(hidden_size=896, num_attention_heads=14),     # 896 not built
                                   dict(hidden_size=768, num_attention_heads=6)])     # head_dim 128
def test_check_model_rejects_unbuilt_shapes_with_berts_messages(shape):
    from transformers import BertConfig

    lib = _native.load()
    rob = W.roberta_desc(xlmr_config(**shape))
    rc = lib.b2e_check_model(C.byref(rob))
    msg = lib.b2e_last_error()
    bert = W.bert_desc(BertConfig(**{**shape, 'intermediate_size': 3072}))
    assert rc != 0 and rc == lib.b2e_check_model(C.byref(bert)) and msg == lib.b2e_last_error()


def test_check_model_rejects_negative_reserved():
    lib = _native.load()
    desc = W.roberta_desc(xlmr_config())
    desc.reserved = -1
    assert lib.b2e_check_model(C.byref(desc)) == ERR_INVALID
    assert b'padding_idx' in lib.b2e_last_error()


def test_validate_refuses_by_name():
    from distllm_b200.embed.encoders.native import NativeRobertaEncoder

    with pytest.raises(NotImplementedError, match='relative_key'):
        NativeRobertaEncoder.validate(xlmr_config(position_embedding_type='relative_key'))
    with pytest.raises(NotImplementedError, match='relative_key_query'):
        NativeRobertaEncoder.validate(xlmr_config(position_embedding_type='relative_key_query'))
    with pytest.raises(NotImplementedError, match='gelu_new'):
        NativeRobertaEncoder.validate(xlmr_config(hidden_act='gelu_new'))
    with pytest.raises(NotImplementedError, match='pad_token_id'):
        NativeRobertaEncoder.validate(xlmr_config(pad_token_id=None))


def test_model_max_length():
    assert W.roberta_max_length(xlmr_config()) == 512
    assert W.roberta_max_length(xlmr_config(max_position_embeddings=8194)) == 8192
    assert W.roberta_max_length(xlmr_config(max_position_embeddings=66)) == 64


def test_auto_maps_both_model_types():
    from distllm_b200.embed.encoders import auto
    from distllm_b200.embed.encoders.native import NativeRobertaEncoder

    assert auto._NATIVE_BY_MODEL_TYPE['roberta'] is NativeRobertaEncoder
    assert auto._NATIVE_BY_MODEL_TYPE['xlm-roberta'] is NativeRobertaEncoder
    assert xlmr_config().model_type == 'xlm-roberta'


@pytest.mark.parametrize('side', ['right', 'left'])
def test_collator_equals_tokenizer(side):
    from distllm_b200.embed.datasets.utils import DataCollator
    from distllm_b200.embed.datasets.utils import SentenceTokenCache

    tok = O.tiny_xlmr_tokenizer()
    tok.model_max_length = 64
    tok.padding_side = side
    assert not SentenceTokenCache.supported(tok)      # the sentence cache stays off for SentencePiece tokenizers
    rng = np.random.default_rng(1)
    words = O.tiny_xlmr_words()
    texts = [' '.join(rng.choice(words, size=n)) for n in (1, 5, 80, 30, 62, 63)] + O.tiny_xlmr_texts()
    collator = DataCollator(tok)
    assert collator._fast
    for lo in range(0, len(texts), 5):
        batch = texts[lo:lo + 5]
        got = collator(batch)
        exp = tok(batch, padding=True, truncation=True, return_tensors='pt')
        assert set(got.keys()) == set(exp.keys()) == {'input_ids', 'attention_mask'}
        for k in exp:
            assert torch.equal(got[k], exp[k]), (side, lo, k)
