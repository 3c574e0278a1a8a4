"""-m gpu: Qwen3 (Qwen3-Embedding) on the H100, from the fused q/k RMSNorm + rotary kernel up to files on disk.

  * b2e_qk_norm_rope against fp32 torch on the same 16-bit inputs: T in {1, 1000, 16 897}, both builds, positions up
    to 32 767 at theta 1e6 through a packed tok_src, a device row count below T; V columns and rows past the row
    count must come back bit-unchanged;
  * the reference's own outputs (tests/golden/qwen3_tiny_golden.npz, tools/make_golden_qwen3.py): right and left
    padding, last-token and normalised mean rows, one batch's hidden state, both storage builds;
  * packed layout == padded layout, b2e_embed_host's graph replay == the eager call;
  * two layers at each Qwen3-Embedding width (0.6B / 4B / 8B layer shapes) and the full 28-layer 0.6B shape at
    S = 1024, normal and outlier weights, against the fp32 oracle (tools/oracle_qwen3.py);
  * a checkpoint directory through get_encoder({'name': 'auto'}) -> embedding_worker -> numpy writer.

Each tolerance is about ten times the worst 1 - cos measured for that comparison on an H100 80GB HBM3 (700 W power
limit); the measured values are in the comments beside them.
"""

from __future__ import annotations

import ctypes
import json

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from oracle import pooling as opool
from tools import make_golden_qwen3 as mq
from tools.oracle_qwen3 import qwen3_forward
from tools.workloads import add_outliers

from conftest import GOLDEN
from conftest import cosine_rows

pytestmark = pytest.mark.gpu
STORAGE_DTYPE = {'f16': torch.float16, 'bf16': torch.bfloat16}
# 1 - cos tolerances (see the module docstring)
TOL_GOLDEN = {'f16': 1e-5, 'bf16': 7e-4}   # measured worst: 1.1e-6 (f16 hidden), 7.3e-5 (bf16 hidden)
TOL_TWO_LAYERS = 3e-5                       # measured worst: 2.9e-6 (4B outlier weights, token states)
TOL_FULL_DEPTH = 5e-5                       # measured worst: 5.1e-6 (outlier weights, token states)


def check_rows(got, ref, tol, what):
    got, ref = np.asarray(got), np.asarray(ref)
    assert np.isfinite(got).all(), what
    live = np.linalg.norm(ref, axis=-1) > 0
    assert not got[~live].any(), what
    worst = float(1 - cosine_rows(got[live], ref[live]).min())
    print(f'QWEN3-COS {what} {worst:.3e}')
    assert worst < tol, (what, worst, tol)
    return worst


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN / 'qwen3_tiny_golden.npz')


@pytest.fixture(scope='module')
def tiny():
    from distllm_b200.embed.encoders.weights import random_qwen3_state_dict

    cfg = mq.tiny_qwen3_config()
    return cfg, random_qwen3_state_dict(cfg, seed=mq.TINY_QWEN3_SEED, device='cpu')


def rope_tables(s, theta, device):
    inv = 1.0 / (theta ** (torch.arange(0, 128, 2, dtype=torch.float64) / 128))
    ang = torch.outer(torch.arange(s, dtype=torch.float64), inv)
    return ang.cos().float().to(device).contiguous(), ang.sin().float().to(device).contiguous()


# ------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize('storage', ['f16', 'bf16'])
@pytest.mark.parametrize('t, packed', [(1, False), (1000, False), (1000, True), (16897, True)])
def test_qk_norm_rope_matches_fp32(storage, t, packed):
    heads, kv, s, eps, theta = 16, 8, 32768, 1e-6, 1e6
    dev = torch.device('cuda:0')
    dt = STORAGE_DTYPE[storage]
    g = torch.Generator().manual_seed(t + packed)
    cols = (heads + 2 * kv) * 128
    # rows of very different magnitudes: the statistic is per head, not per row
    qkv = (torch.randn(t, cols, generator=g) * torch.exp(torch.randn(t, 1, generator=g) * 2)).to(dt)
    # gains in [0.5, 2) that differ between the two halves of a head and between q and k: a swapped, missing or
    # rotated gain changes the result
    q_gamma = 0.5 + 1.5 * torch.rand(128, generator=g)
    k_gamma = 0.5 + 1.5 * torch.rand(128, generator=g)
    cos, sin = rope_tables(s, theta, dev)
    if packed:
        tok_src = torch.randint(0, 2 * s, (t,), generator=g, dtype=torch.int32)
        tok_src[0], tok_src[-1] = s - 1, 2 * s - 1            # position 32 767 in both "sequences"
        t_real = max(1, t - 37)
        pos = tok_src.long() % s
    else:
        tok_src, t_real = None, t
        pos = torch.arange(t) % s
    x = qkv.float()
    out = qkv.to(dev)
    nv.qk_norm_rope_(out, q_gamma.to(dev), k_gamma.to(dev), cos, sin, heads, kv, eps,
                     t_real=torch.tensor([t_real, 1], dtype=torch.int32, device=dev) if packed else None,
                     tok_src=tok_src.to(dev) if packed else None)
    out = out.cpu()

    # fp32 reference: per-head RMSNorm with its gain, THEN the halves rotation
    hk = x[:, :(heads + kv) * 128].view(t, heads + kv, 128)
    y = hk * torch.rsqrt(hk.pow(2).mean(-1, keepdim=True) + eps)
    y = y * torch.cat([q_gamma.expand(heads, 128), k_gamma.expand(kv, 128)])[None]
    c, sn = cos.cpu()[pos][:, None], sin.cpu()[pos][:, None]   # the tables the kernel is given
    y1, y2 = y[..., :64], y[..., 64:]
    ref = torch.cat([y1 * c - y2 * sn, y2 * c + y1 * sn], -1).view(t, -1)

    got = out[:t_real, :(heads + kv) * 128].float()
    scale = {'f16': 2.0 ** -10, 'bf16': 2.0 ** -7}[storage]
    # one rounding of |value| <= |y1| + |y2| at the store, plus fp32 differences in the statistic
    bound = scale * (y1.abs() + y2.abs()).repeat(1, 1, 2).view(t, -1)[:t_real] + 1e-6
    err = (got - ref[:t_real]).abs()
    assert (err <= bound).all(), (storage, t, packed, float((err / bound).max()))
    assert torch.equal(out[:, (heads + kv) * 128:], qkv[:, (heads + kv) * 128:])   # V heads untouched
    assert torch.equal(out[t_real:], qkv[t_real:])                                  # rows past the row count


# -------------------------------------------------------------------------------- reference fixture
def _batches(golden, side):
    return [(torch.from_numpy(golden[f'{side}/batch{i}/input_ids']),
             torch.from_numpy(golden[f'{side}/batch{i}/attention_mask'])) for i in range(int(golden['n_batches']))]


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
@pytest.mark.parametrize('side', ['right', 'left'])
def test_matches_reference_vectors(golden, tiny, storage, side):
    from distllm_b200.embed.encoders.native import NativeQwen3Encoder

    cfg, sd = tiny
    enc = NativeQwen3Encoder(cfg, sd, storage=storage)
    tol = TOL_GOLDEN[storage]
    try:
        batches = _batches(golden, side)
        if side == 'right':
            ids, mask = batches[0]
            hidden = enc.encode(ids, mask).cpu().numpy()
            check_rows(hidden[mask.bool().numpy()], golden['right/batch0/hidden_attended'], tol,
                       f'golden {storage} hidden')
        last = torch.cat([enc.encode_pooled(ids, mask, None, nv.POOL_LAST_TOKEN, False).cpu()
                          for ids, mask in batches])
        check_rows(last.numpy(), golden[f'{side}/pooled/last_token'], tol, f'golden {storage} {side} last_token')
        if side == 'right':
            mean = torch.cat([enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_REF, True).cpu()
                              for ids, mask in batches])
            check_rows(mean.numpy(), golden['right/pooled/mean_normalized'], tol, f'golden {storage} mean')
    finally:
        enc.close()


def _pooled_packed_and_padded(enc, ids, mask, kind):
    lib = enc._lib
    lib.b2e_debug_set_packing.argtypes = [ctypes.c_int]
    try:
        lib.b2e_debug_set_packing(1)
        packed = enc.encode_pooled(ids, mask, None, kind, True).cpu()
        lib.b2e_debug_set_packing(0)
        padded = enc.encode_pooled(ids, mask, None, kind, True).cpu()
    finally:
        lib.b2e_debug_set_packing(1)
    return packed, padded


def test_packed_layout_equals_padded(tiny):
    from distllm_b200.embed.encoders.native import NativeQwen3Encoder

    cfg, sd = tiny
    enc = NativeQwen3Encoder(cfg, sd)
    g = torch.Generator().manual_seed(7)
    try:
        for b, s, lens in [(7, 50, [50, 3, 17, 50, 1, 33, 2]), (5, 512, [512, 129, 128, 64, 7])]:
            ids = torch.randint(4, cfg.vocab_size, (b, s), generator=g)
            mask = (torch.arange(s)[None] < torch.tensor(lens)[:, None]).long()
            for kind in (nv.POOL_MEAN_REF, nv.POOL_MEAN_PER_ROW, nv.POOL_LAST_TOKEN):
                packed, padded = _pooled_packed_and_padded(enc, ids, mask, kind)
                live = padded.norm(dim=-1) > 0
                assert torch.isfinite(packed).all() and torch.equal(live, packed.norm(dim=-1) > 0)
                cos = torch.nn.functional.cosine_similarity(packed[live], padded[live])
                assert cos.min().item() > 1 - 1e-6, (b, s, kind, cos)
    finally:
        enc.close()


def test_embed_host_graph_replay_equals_eager(tiny):
    from distllm_b200.embed.encoders.native import NativeQwen3Encoder

    cfg, sd = tiny
    enc = NativeQwen3Encoder(cfg, sd)
    g = torch.Generator().manual_seed(31)
    try:
        for n, s, batch, pool in [(27, 40, 4, nv.POOL_MEAN_REF), (16, 200, 8, nv.POOL_LAST_TOKEN)]:
            ids = torch.randint(4, cfg.vocab_size, (n, s), generator=g)
            lens = torch.randint(1, s + 1, (n,), generator=g)
            mask = (torch.arange(s)[None] < lens[:, None]).long()
            ids, mask = ids.pin_memory(), mask.pin_memory()
            host = enc.embed_host(ids, mask, None, batch=batch, pool_kind=pool, normalize=True)
            for r0 in range(0, n, batch):
                sl = slice(r0, min(n, r0 + batch))
                assert torch.equal(host[sl], enc.encode_pooled(ids[sl], mask[sl], None, pool, True).cpu()), (n, r0)
    finally:
        enc.close()


# ------------------------------------------------------------------------ real shapes vs the oracle
# (H, heads, kv_heads, I) of Qwen3-Embedding-0.6B / 4B / 8B
SHAPES = {'0.6B': (1024, 16, 8, 3072), '4B': (2560, 32, 8, 9728), '8B': (4096, 32, 8, 12288)}


def qwen3_config(name, layers, vocab=2000, max_pos=2048):
    from transformers import Qwen3Config

    h, heads, kv, i = SHAPES[name]
    return Qwen3Config(vocab_size=vocab, hidden_size=h, num_hidden_layers=layers, num_attention_heads=heads,
                       num_key_value_heads=kv, head_dim=128, intermediate_size=i, max_position_embeddings=max_pos,
                       rms_norm_eps=1e-6, rope_parameters={'rope_type': 'default', 'rope_theta': 1e6},
                       initializer_range=0.02, tie_word_embeddings=False)


def _seeded_weights(cfg, weights, seed):
    from distllm_b200.embed.encoders.weights import random_qwen3_state_dict

    sd = random_qwen3_state_dict(cfg, seed=seed, device=torch.device('cuda:0'), dtype=torch.float16)
    if weights == 'outliers':
        add_outliers(sd, 'qwen3', seed=seed + 1)
    return sd


@pytest.mark.parametrize('weights', ['normal', 'outliers'])
@pytest.mark.parametrize('name', sorted(SHAPES))
def test_two_layers_at_each_width_vs_oracle(name, weights):
    from distllm_b200.embed.encoders.native import NativeQwen3Encoder

    cfg = qwen3_config(name, 2)
    sd = _seeded_weights(cfg, weights, 11)
    g = torch.Generator().manual_seed(12)
    b, s = 3, 300
    ids = torch.randint(3, cfg.vocab_size, (b, s), generator=g)
    mask = (torch.arange(s)[None] < torch.tensor([300, 129, 5])[:, None]).long()
    ref = qwen3_forward(sd, cfg, ids, mask)
    enc = NativeQwen3Encoder(cfg, sd)
    try:
        what = f'2L {name} {weights}'
        hidden = enc.encode(ids, mask).cpu().numpy()
        valid = mask.bool().numpy()
        check_rows(hidden[valid], ref.numpy()[valid], TOL_TWO_LAYERS, f'{what} tokens')
        check_rows(enc.encode_pooled(ids, mask, None, nv.POOL_LAST_TOKEN, False).cpu().numpy(),
                   opool.last_token_pool(ref, mask).numpy(), TOL_TWO_LAYERS, f'{what} last_token')
        check_rows(enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_REF, False).cpu().numpy(),
                   opool.average_pool(ref, mask.clone()).numpy(), TOL_TWO_LAYERS, f'{what} mean')
        packed, padded = _pooled_packed_and_padded(enc, ids, mask, nv.POOL_LAST_TOKEN)
        assert torch.nn.functional.cosine_similarity(packed, padded).min().item() > 1 - 1e-6
    finally:
        enc.close()
        del sd
        torch.cuda.empty_cache()


@pytest.mark.parametrize('weights', ['normal', 'outliers'])
def test_qwen3_embedding_0p6b_full_depth_s1024(weights):
    """All 28 layers of the 0.6B shape, S = 1024, rows of 1024 and 700 tokens (as the C3 Mistral test)."""
    from distllm_b200.embed.encoders.native import NativeQwen3Encoder

    cfg = qwen3_config('0.6B', 28, vocab=32000, max_pos=32768)
    sd = _seeded_weights(cfg, weights, 21)
    g = torch.Generator().manual_seed(23)
    b, s = 2, 1024
    ids = torch.randint(3, cfg.vocab_size, (b, s), generator=g)
    mask = (torch.arange(s)[None] < torch.tensor([1024, 700])[:, None]).long()
    ref = qwen3_forward(sd, cfg, ids, mask)
    enc = NativeQwen3Encoder(cfg, sd)
    try:
        what = f'0.6B 28L {weights}'
        check_rows(enc.encode_pooled(ids, mask, None, nv.POOL_LAST_TOKEN, False).cpu().numpy(),
                   opool.last_token_pool(ref, mask).numpy(), TOL_FULL_DEPTH, f'{what} last_token')
        hidden = enc.encode(ids, mask).cpu().numpy()
        valid = mask.bool().numpy()
        check_rows(hidden[valid], ref.numpy()[valid], TOL_FULL_DEPTH, f'{what} tokens')
    finally:
        enc.close()
        del sd
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------- files on disk
def test_embedding_worker_qwen3_checkpoint_dir_matches_reference(tmp_path, golden):
    """A Qwen3 checkpoint directory through the plugin API: get_encoder({'name': 'auto'}) maps model_type 'qwen3' to
    the native encoder, embedding_worker writes the last-token rows with the numpy writer."""
    from distllm_b200.distributed_embedding import embedding_worker
    from distllm_b200.embed import get_encoder
    from distllm_b200.embed.encoders.native import NativeQwen3Encoder
    from distllm_b200.registry import registry

    mq.write_tiny_qwen3_checkpoint(tmp_path / 'ckpt')
    texts = mq.tiny_qwen3_texts()
    (tmp_path / 't.jsonl').write_text('\n'.join(json.dumps({'text': t}) for t in texts) + '\n')
    enc_kw = {'name': 'auto', 'pretrained_model_name_or_path': str(tmp_path / 'ckpt'), 'half_precision': False,
              'quantization': False}
    try:
        assert isinstance(get_encoder(enc_kw).native, NativeQwen3Encoder)
        embedding_worker(tmp_path / 't.jsonl', tmp_path / 'out',
                         dataset_kwargs={'name': 'jsonl', 'batch_size': 4, 'num_data_workers': 0,
                                         'pin_memory': True},
                         encoder_kwargs=enc_kw, pooler_kwargs={'name': 'last_token'},
                         embedder_kwargs={'name': 'full_sequence'}, writer_kwargs={'name': 'numpy'})
        out = [p for p in (tmp_path / 'out').iterdir() if p.is_dir()]
        assert len(out) == 1, out
        emb = np.load(out[0] / 'embeddings.npy')
        check_rows(emb, golden['right/pooled/last_token'], TOL_GOLDEN['f16'], 'worker last_token')
    finally:
        registry.clear()
