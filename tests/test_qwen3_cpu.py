"""Qwen3 without a device: the fp32 oracle against the reference's golden vectors and against HF Qwen3Model layer by
layer, the shapes b2e_check_model accepts and rejects, the weight count, the config translation and AutoEncoder's
validation of a Qwen3 config.json before any weight is read."""

from __future__ import annotations

import ctypes as C
import json

import numpy as np
import pytest
import torch

from distllm_b200 import _native
from oracle import pooling as opool
from oracle.make_golden import weights_digest
from tools import make_golden_qwen3 as mq
from tools.oracle_qwen3 import qwen3_forward

from conftest import GOLDEN

# the published Qwen3-Embedding shapes: (layers, H, heads, kv_heads, I)
QWEN3_EMBEDDING = {'0.6B': (28, 1024, 16, 8, 3072), '4B': (36, 2560, 32, 8, 9728), '8B': (36, 4096, 32, 8, 12288)}


def qdesc(layers, hidden, heads, kv_heads, intermediate, head_dim=128, window=0):
    return _native.ModelDesc(arch=_native.ARCH_QWEN3, num_layers=layers, hidden=hidden, heads=heads,
                             kv_heads=kv_heads, head_dim=head_dim, intermediate=intermediate, vocab=151669,
                             max_pos=32768, eps=1e-6, rope_theta=1e6, sliding_window=window)


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN / 'qwen3_tiny_golden.npz')


@pytest.fixture(scope='module')
def tiny():
    from distllm_b200.embed.encoders.weights import random_qwen3_state_dict

    cfg = mq.tiny_qwen3_config()
    return cfg, random_qwen3_state_dict(cfg, seed=mq.TINY_QWEN3_SEED, device='cpu')


def _batches(golden, side):
    return [(torch.from_numpy(golden[f'{side}/batch{i}/input_ids']),
             torch.from_numpy(golden[f'{side}/batch{i}/attention_mask'])) for i in range(int(golden['n_batches']))]


def test_fixture_weights_are_the_seeded_ones(golden, tiny):
    assert str(golden['weights_sha256']) == weights_digest(tiny[1])
    assert int(golden['n_texts']) == len(mq.tiny_qwen3_texts())


@pytest.mark.parametrize('side', ['right', 'left'])
def test_oracle_matches_reference_golden(golden, tiny, side):
    cfg, sd = tiny
    last, mean = [], []
    for i, (ids, mask) in enumerate(_batches(golden, side)):
        hidden = qwen3_forward(sd, cfg, ids, mask)
        if i == 0 and side == 'right':
            np.testing.assert_allclose(hidden[mask.bool()].numpy(), golden['right/batch0/hidden_attended'],
                                       atol=5e-5, rtol=0)
        last.append(opool.last_token_pool(hidden, mask))
        mean.append(torch.nn.functional.normalize(opool.average_pool(hidden, mask.clone()), dim=-1))
    np.testing.assert_allclose(torch.cat(last).numpy(), golden[f'{side}/pooled/last_token'], atol=5e-5, rtol=0)
    if side == 'right':
        np.testing.assert_allclose(torch.cat(mean).numpy(), golden['right/pooled/mean_normalized'], atol=5e-5,
                                   rtol=0)
    assert max(ids.shape[1] for ids, _ in _batches(golden, side)) == 512   # the truncated row


def test_oracle_matches_hf_layer_by_layer(golden, tiny):
    """Every depth against HF Qwen3Model: hidden_states[l] is the residual stream after l layers (the last one
    after the final norm); the oracle's return_all states are final_norm of the same streams."""
    from transformers import Qwen3Model

    from oracle.mistral import _rms

    cfg, sd = tiny
    model = Qwen3Model(cfg).eval()
    model.load_state_dict(sd, strict=False)
    ids, mask = _batches(golden, 'left')[1]
    with torch.no_grad():
        hf = model(input_ids=ids, attention_mask=mask, output_hidden_states=True).hidden_states
    states = qwen3_forward(sd, cfg, ids, mask, return_all=True)
    assert len(states) == cfg.num_hidden_layers
    valid = mask.bool()
    for layer, got in enumerate(states, start=1):
        want = hf[layer] if layer == cfg.num_hidden_layers else _rms(hf[layer], sd['norm.weight'], cfg.rms_norm_eps)
        np.testing.assert_allclose(got[valid].numpy(), want[valid].numpy(), atol=5e-5, rtol=0)


def test_oracle_norm_then_rotate_is_observable(golden, tiny):
    """The fixture tells the reference's order (head norm, then rotary) from the swapped one, and a missing k gain
    from the right one: each changes the pooled rows far beyond the 5e-5 tolerance."""
    from oracle import mistral as omis

    cfg, sd = tiny
    ids, mask = _batches(golden, 'right')[1]
    want = torch.from_numpy(golden['right/pooled/last_token'][4:8])
    no_k_gain = {k: (torch.ones_like(v) if k.endswith('k_norm.weight') else v) for k, v in sd.items()}
    assert (opool.last_token_pool(qwen3_forward(no_k_gain, cfg, ids, mask), mask) - want).abs().max() > 1e-3
    rotate = omis._rotate
    eps, heads, kv, d = cfg.rms_norm_eps, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    b, s = ids.shape
    y = omis._rms(sd['embed_tokens.weight'][ids], sd['layers.0.input_layernorm.weight'], eps)
    q = torch.nn.functional.linear(y, sd['layers.0.self_attn.q_proj.weight']).view(b, s, heads, d).transpose(1, 2)
    g = sd['layers.0.self_attn.q_norm.weight']
    norm_first = rotate(omis._rms(q, g, eps), cfg.rope_parameters['rope_theta'])
    rot_first = omis._rms(rotate(q, cfg.rope_parameters['rope_theta']), g, eps)
    assert (norm_first - rot_first).abs().max() > 1e-3
    assert kv < heads


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
@pytest.mark.parametrize('name', sorted(QWEN3_EMBEDDING))
def test_check_model_accepts_qwen3_embedding(storage, name):
    lib = _native.load(storage)
    layers, h, heads, kv, i = QWEN3_EMBEDDING[name]
    d = qdesc(layers, h, heads, kv, i)
    assert lib.b2e_check_model(C.byref(d)) == 0, lib.b2e_last_error()
    assert lib.b2e_num_weights(C.byref(d)) == 2 + 8 * layers


def test_check_model_rejects_what_is_not_built():
    lib = _native.load()
    cases = [
        (qdesc(28, 1024, 16, 8, 3072, window=4096), b'Qwen3: sliding-window layers are not built'),
        (qdesc(28, 1024, 16, 8, 3072, head_dim=64), b'Qwen3: need head_dim 128'),
        (qdesc(28, 1024, 16, 6, 3072), b'heads % kv_heads == 0'),
        (qdesc(28, 1536, 12, 2, 8960), b'hidden size 1536'),      # gte-Qwen2-1.5B's width
        (qdesc(28, 1024, 16, 8, 3000), b'multiple of 128'),
    ]
    for d, msg in cases:
        assert lib.b2e_check_model(C.byref(d)) in (1, 3), (d.hidden, d.head_dim, d.kv_heads, d.sliding_window)
        assert msg in lib.b2e_last_error(), lib.b2e_last_error()


def test_num_weights_counts_the_head_norms():
    lib = _native.load()
    for layers in (1, 4, 36):
        assert lib.b2e_num_weights(C.byref(qdesc(layers, 1024, 16, 8, 3072))) == 2 + 8 * layers
    mistral = qdesc(4, 1024, 16, 8, 3072)
    mistral.arch = _native.ARCH_MISTRAL
    assert lib.b2e_num_weights(C.byref(mistral)) == 2 + 6 * 4


def test_qwen3_desc_translates_and_rejects():
    from transformers import Qwen3Config

    from distllm_b200.embed.encoders.weights import qwen3_desc

    d = qwen3_desc(mq.tiny_qwen3_config())
    assert (d.arch, d.hidden, d.heads, d.kv_heads, d.head_dim, d.intermediate) == (_native.ARCH_QWEN3, 256, 4, 2,
                                                                                   128, 384)
    assert (d.rope_theta, d.sliding_window, d.max_pos) == (1e6, 0, 512)
    assert d.eps == pytest.approx(1e-6)
    base = dict(mq.TINY_QWEN3)
    for change, msg in (({'attention_bias': True}, 'attention_bias'),
                        ({'use_sliding_window': True, 'sliding_window': 64, 'max_window_layers': 2},
                         'sliding_attention'),
                        ({'rope_parameters': {'rope_type': 'yarn', 'rope_theta': 1e6, 'factor': 4.0,
                                              'original_max_position_embeddings': 512}}, "'yarn'"),
                        ({'hidden_act': 'gelu'}, 'hidden_act')):
        with pytest.raises(NotImplementedError, match=msg):
            qwen3_desc(Qwen3Config(**{**base, **change}))


def test_qwen3_weight_list_order_with_and_without_prefix(tiny):
    from distllm_b200.embed.encoders.weights import qwen3_weight_list

    cfg, sd = tiny
    for state in (sd, {'model.' + k: v for k, v in sd.items()}):
        w = qwen3_weight_list(state, cfg.num_hidden_layers, torch.device('cpu'), torch.float16)
        assert len(w) == 2 + 8 * cfg.num_hidden_layers
        for layer in range(cfg.num_hidden_layers):
            base = 2 + 8 * layer
            assert w[base + 1].shape == (512 + 2 * 256, 256) and w[base + 1].dtype == torch.float16   # Wqkv
            assert w[base + 2].shape == (256, 512)                                                    # Wo: H x ctx
            for k, n in ((6, 'q_norm'), (7, 'k_norm')):
                assert w[base + k].dtype == torch.float32
                assert torch.equal(w[base + k], sd[f'layers.{layer}.self_attn.{n}.weight'])
        assert not torch.equal(w[8], w[9])   # the random gains differ (HF's all-ones would hide a swap)


@pytest.mark.parametrize('change, error', [
    ({'use_sliding_window': True, 'sliding_window': 64, 'max_window_layers': 1}, NotImplementedError),
    ({'attention_bias': True}, NotImplementedError),
    ({'head_dim': 64}, _native.NativeError),
    ({'hidden_size': 1536, 'num_attention_heads': 12, 'num_key_value_heads': 2}, _native.NativeError),
])
def test_auto_encoder_rejects_before_reading_weights(tmp_path, change, error):
    """Only config.json exists: a loader that read weights first would fail with a missing-file error instead."""
    from transformers import Qwen3Config

    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig

    ckpt = tmp_path / 'qwen3'
    ckpt.mkdir()
    Qwen3Config(**{**mq.TINY_QWEN3, **change}).save_pretrained(ckpt)
    assert json.loads((ckpt / 'config.json').read_text())['model_type'] == 'qwen3'
    with pytest.raises(error):
        AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(ckpt), quantization=False))


def test_auto_encoder_maps_qwen3():
    from distllm_b200.embed.encoders import auto
    from distllm_b200.embed.encoders.native import NativeQwen3Encoder

    assert auto._NATIVE_BY_MODEL_TYPE['qwen3'] is NativeQwen3Encoder
    NativeQwen3Encoder.validate(mq.tiny_qwen3_config())


def test_storage_for_qwen3(monkeypatch):
    monkeypatch.delenv('B2E_STORAGE', raising=False)
    assert _native.storage_for_arch('qwen3') == 'f16'
    monkeypatch.setenv('B2E_STORAGE', 'bf16')
    assert _native.storage_for_arch('qwen3') == 'bf16'


def test_outliers_leave_other_families_unchanged_and_bound_head_gains(tiny):
    """The 'qwen3' entry draws the head-norm gains from a generator of its own: the Mistral names of a Qwen3 state
    dict get exactly the gains a Mistral state dict gets, and the [128] gains stay in the moderate range."""
    from tools.workloads import add_outliers

    cfg, sd = tiny
    qwen = add_outliers({k: v.clone() for k, v in sd.items()}, 'qwen3', seed=4)
    mis = add_outliers({k: v.clone() for k, v in sd.items() if not k.endswith(('q_norm.weight', 'k_norm.weight'))},
                       'mistral', seed=4)
    for k, v in mis.items():
        assert torch.equal(qwen[k], v), k
    for k, v in qwen.items():
        if k.endswith(('q_norm.weight', 'k_norm.weight')):
            assert v.shape == (128,) and 0.5 <= v.min() and v.max() <= 2.0
            assert not torch.equal(v, sd[k])
