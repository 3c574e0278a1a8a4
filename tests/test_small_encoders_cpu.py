"""The small encoders without a device: which shapes b2e_check_model accepts, AutoEncoder's validation of a
MiniLM-shaped checkpoint directory, and the CPU oracle against the reference's head_dim-32 golden vectors."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from distllm_b200 import _native
from oracle import pooling as opool
from oracle.make_golden import weights_digest

from conftest import GOLDEN


def desc(arch, hidden, heads, head_dim, intermediate, layers=2, kv_heads=None):
    return _native.ModelDesc(arch=arch, num_layers=layers, hidden=hidden, heads=heads, kv_heads=kv_heads or heads,
                             head_dim=head_dim, intermediate=intermediate, vocab=100, max_pos=512,
                             sliding_window=64, global_every=3)


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
def test_check_model_accepts_the_small_encoders(storage):
    lib = _native.load(storage)
    for d in (desc(_native.ARCH_BERT, 384, 12, 32, 1536, 6),      # all-MiniLM-L6-v2
              desc(_native.ARCH_BERT, 384, 12, 32, 1536, 12),     # bge-small-en-v1.5, e5-small-v2
              desc(_native.ARCH_ESM2, 640, 20, 32, 2560, 30)):    # esm2_t30_150M
        assert lib.b2e_check_model(C.byref(d)) == 0, lib.b2e_last_error()


def test_check_model_still_rejects_other_shapes():
    lib = _native.load()
    cases = [
        (desc(_native.ARCH_ESM2, 320, 20, 16, 1280), b'head_dim 64'),       # esm2_t6_8M
        (desc(_native.ARCH_ESM2, 480, 20, 24, 1920), b'head_dim 64'),       # esm2_t12_35M
        (desc(_native.ARCH_BERT, 1792, 28, 64, 4096), b'hidden size 1792'),
        (desc(_native.ARCH_BERT, 320, 10, 32, 1280), b'hidden size 320'),
        (desc(_native.ARCH_BERT, 480, 15, 32, 1920), b'hidden size 480'),
        (desc(_native.ARCH_BERT, 384, 6, 32, 1536), b'head_dim 64'),        # heads x head_dim != H
        (desc(_native.ARCH_MISTRAL, 4096, 32, 32, 14336, kv_heads=8), b'head_dim 128'),
        (desc(_native.ARCH_MISTRAL, 384, 3, 128, 1536), b'multiple of 256'),
        (desc(_native.ARCH_MODERNBERT, 768, 24, 32, 1152), b'head_dim 64'),
        (desc(_native.ARCH_MODERNBERT, 384, 6, 64, 1536), b'multiple of 256'),
        (desc(_native.ARCH_MODERNBERT, 640, 10, 64, 1280), b'multiple of 256'),
    ]
    for d, msg in cases:
        assert lib.b2e_check_model(C.byref(d)) in (1, 3), (d.arch, d.hidden, d.head_dim)
        assert msg in lib.b2e_last_error(), (d.arch, d.hidden, lib.b2e_last_error())


def test_num_weights_does_not_depend_on_head_dim():
    lib = _native.load()
    assert lib.b2e_num_weights(C.byref(desc(_native.ARCH_BERT, 384, 12, 32, 1536, 6))) == 5 + 12 * 6
    assert lib.b2e_num_weights(C.byref(desc(_native.ARCH_ESM2, 640, 20, 32, 2560, 30))) == 3 + 12 * 30


def test_auto_encoder_validates_a_minilm_checkpoint(tmp_path):
    """AutoEncoder checks the shape before any weight is loaded: a MiniLM-shaped directory passes validation; on a
    box without a GPU the construction then fails for want of a device, not for the shape."""
    from transformers import AutoConfig
    from transformers import BertConfig
    from transformers import BertModel

    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig
    from distllm_b200.embed.encoders.native import NativeBertEncoder

    cfg = BertConfig(vocab_size=120, hidden_size=384, num_hidden_layers=1, num_attention_heads=12,
                     intermediate_size=1536, max_position_embeddings=64)
    ckpt = tmp_path / 'minilm'
    BertModel(cfg).save_pretrained(ckpt)
    (ckpt / 'vocab.txt').write_text('\n'.join(['[PAD]', '[UNK]', '[CLS]', '[SEP]', '[MASK]'] +
                                              [f'w{i}' for i in range(115)]) + '\n')
    NativeBertEncoder.validate(AutoConfig.from_pretrained(ckpt))
    if torch.cuda.is_available():
        enc = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(ckpt), quantization=False))
        assert enc.embedding_size == 384
    else:
        with pytest.raises(_native.NativeError):
            AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(ckpt), quantization=False))
    cfg.num_attention_heads = 24      # head_dim 16: rejected before the weights are read
    bad = tmp_path / 'bad'
    cfg.save_pretrained(bad)
    with pytest.raises(_native.NativeError, match='head_dim 64'):
        AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(bad), quantization=False))


def test_oracle_matches_bert_d32_golden():
    from transformers import BertConfig

    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    from oracle import bert as obert
    from oracle.make_golden import TINY_SEED
    from tools.make_golden_small import BERT_D32

    golden = np.load(GOLDEN / 'bert_d32_golden.npz')
    cfg = BertConfig(**BERT_D32)
    sd = random_bert_state_dict(cfg, seed=TINY_SEED, device='cpu')
    assert weights_digest(sd) == str(golden['weights_sha256'])
    batches = [{k: torch.from_numpy(golden[f'batch{i}/{k}']) for k in ('input_ids', 'attention_mask', 'token_type_ids')}
               for i in range(int(golden['n_batches']))]

    def encode(b):
        return obert.bert_forward(sd, cfg, b['input_ids'], b['attention_mask'], b['token_type_ids'])

    np.testing.assert_allclose(encode(batches[0]).numpy(), golden['batch0/hidden'], rtol=1e-4, atol=5e-5)
    for kind in ('mean', 'mean_normalized', 'last_token'):
        pool = opool.last_token_pool if kind == 'last_token' else opool.average_pool
        got = opool.compute_embeddings([{k: v.clone() for k, v in b.items()} for b in batches], encode, pool,
                                       do_normalize=(kind == 'mean_normalized'))
        np.testing.assert_allclose(got, golden[f'pooled/{kind}'], rtol=1e-4, atol=5e-5)


def test_oracle_matches_esm_d32_golden():
    from transformers import EsmConfig

    from distllm_b200.embed.encoders.weights import random_esm_state_dict
    from oracle import esm as oesm
    from oracle.make_golden import TINY_ESM_SEED
    from tools.make_golden_small import ESM_D32

    golden = np.load(GOLDEN / 'esm_d32_golden.npz')
    cfg = EsmConfig(**ESM_D32)
    sd = random_esm_state_dict(cfg, seed=TINY_ESM_SEED, device='cpu')
    assert weights_digest(sd) == str(golden['weights_sha256'])
    batches = [{k: torch.from_numpy(golden[f'batch{i}/{k}']) for k in ('input_ids', 'attention_mask')}
               for i in range(int(golden['n_batches']))]
    assert (batches[0]['input_ids'] == cfg.mask_token_id).any(), 'fixture must exercise token dropout'

    def encode(b):
        return oesm.esm_forward(sd, cfg, b['input_ids'], b['attention_mask'])

    valid = batches[0]['attention_mask'].bool()
    np.testing.assert_allclose(encode(batches[0])[valid].numpy(), golden['batch0/hidden_attended'], rtol=1e-4,
                               atol=5e-5)
    got = opool.compute_embeddings(batches, encode, opool.average_pool)
    np.testing.assert_allclose(got, golden['pooled/mean'], rtol=1e-4, atol=5e-5)
