"""-m gpu: weight matrices held in 4-bit NF4 on the H100, from the dequantising GEMM up to files on disk.

Every comparison is bitwise: the NF4 GEMM writes, byte for byte, the W tile the 16-bit GEMM loads for the matrix
dequantised on the host (embed/encoders/nf4.py), so the NF4 encoder must reproduce the 16-bit encoder built from
quantize_state_dict_nf4(state_dict) -- the load-time path -- exactly:
  * b2e_gemm_nf4 against b2e_gemm_h16 on to_storage(nf4_dequantize(codes, absmax)): all five epilogues, K from 64 to
    14 336, N up to 28 672, M across the tile edges, every code value, zero and negative scales, both builds;
  * encode / encode_pooled / b2e_embed_host of BERT, ModernBERT, Mistral (sliding window) and Qwen3, tiny and at one
    realistic width each, right-padded (packed layout) and left-padded (padded layout) batches;
  * a device row count far below the M the grid is sized for (CTAs without a tile);
  * the device weight bytes and the load's peak memory of a 2-layer H = 4096 encoder;
  * one embedding_worker run, file to file, with quantization: true.
"""

from __future__ import annotations

import json

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from distllm_b200.embed.encoders import nf4
from distllm_b200.embed.encoders import weights as W

pytestmark = pytest.mark.gpu
STORAGE_DTYPE = {'f16': torch.float16, 'bf16': torch.bfloat16}
DEV = torch.device('cuda:0')


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view({4: torch.int32, 2: torch.int16}[t.element_size()])


def assert_bitwise(got: torch.Tensor, ref: torch.Tensor, what: str) -> None:
    assert got.shape == ref.shape and got.dtype == ref.dtype, what
    if not torch.equal(bits(got), bits(ref)):
        bad = (bits(got) != bits(ref)).nonzero()
        pytest.fail(f'{what}: {bad.shape[0]} elements differ, first at {bad[0].tolist()}')


# -------------------------------------------------------------------------------------------- the GEMM
def random_nf4(n: int, k: int, seed: int) -> tuple[torch.Tensor, torch.Tensor]:
    """Codes over all 16 values, scales with zeros and negative values (no checkpoint has negative scales; the
    kernel must not care)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    codes = torch.randint(0, 256, (n, k // 2), generator=g, device=DEV, dtype=torch.uint8)
    absmax = torch.rand((k // 64, n), generator=g, device=DEV) * 0.08 + 0.005
    absmax[torch.rand(absmax.shape, generator=g, device=DEV) < 0.05] = 0.0
    absmax[torch.rand(absmax.shape, generator=g, device=DEV) < 0.05] *= -1.0
    return codes, absmax.contiguous()


GEMM_CASES = [
    # (M, N, K, epilogue)
    *[(m, 256, 768, epi) for epi in range(5) for m in (1, 129, 1000)],
    (127, 768, 64, nv.EPI_BIAS),
    (128, 3072, 768, nv.EPI_BIAS_GELU),
    (4099, 3072, 768, nv.EPI_BIAS_GELU),
    (1000, 768, 3072, nv.EPI_BIAS_RESID),
    (128, 6144, 4096, nv.EPI_BIAS),
    (129, 4096, 14336, nv.EPI_BIAS),
    (4099, 28672, 4096, nv.EPI_SWIGLU),
    (1000, 5376, 768, nv.EPI_GEGLU),
]


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
@pytest.mark.parametrize('m, n, k, epi', GEMM_CASES)
def test_gemm_nf4_equals_gemm_h16_on_the_dequantised_matrix(storage, m, n, k, epi):
    dt = STORAGE_DTYPE[storage]
    g = torch.Generator(device=DEV).manual_seed(m * 7 + n + k + epi)
    codes, absmax = random_nf4(n, k, m + n + k)
    w16 = W.to_storage(nf4.nf4_dequantize(codes, absmax), DEV, dt)
    a = (torch.randn((m, k), generator=g, device=DEV) * 0.5).to(dt)
    glu = epi in (nv.EPI_SWIGLU, nv.EPI_GEGLU)
    bias = None if glu else torch.randn(n, generator=g, device=DEV) * 0.1
    resid = (torch.randn((m, n), generator=g, device=DEV)).to(dt) if epi == nv.EPI_BIAS_RESID else None
    ref = nv.gemm_h16(a, w16, bias, resid, epi)
    got = nv.gemm_nf4(a, codes, absmax, bias, resid, epi)
    assert torch.isfinite(ref.float()).all()
    assert_bitwise(got, ref, f'{storage} M{m} N{n} K{k} epi{epi}')


def test_gemm_nf4_rejects_bad_operands():
    a = torch.zeros((128, 96), dtype=torch.float16, device=DEV)
    with pytest.raises(nv.NativeError, match='K=96'):
        nv.gemm_nf4(a, torch.zeros((128, 48), dtype=torch.uint8, device=DEV),
                    torch.zeros((1, 128), device=DEV), None)
    a = torch.zeros((128, 128), dtype=torch.float16, device=DEV)
    with pytest.raises(nv.NativeError, match='expected codes'):
        nv.gemm_nf4(a, torch.zeros((128, 128), dtype=torch.uint8, device=DEV), torch.zeros((2, 128), device=DEV),
                    None)


# ------------------------------------------------------------------------------------------- encoders
def _configs():
    from transformers import BertConfig
    from transformers import MistralConfig
    from transformers import ModernBertConfig
    from transformers import Qwen3Config

    def bert(h, i, heads):
        return BertConfig(vocab_size=300, hidden_size=h, num_hidden_layers=2, num_attention_heads=heads,
                          intermediate_size=i, max_position_embeddings=512, initializer_range=0.05)

    def modernbert(h, i, heads):
        return ModernBertConfig(vocab_size=300, hidden_size=h, num_hidden_layers=2, num_attention_heads=heads,
                                intermediate_size=i, max_position_embeddings=512, local_attention=64,
                                pad_token_id=0, bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2)

    def mistral(h, i, heads, kv, window):
        return MistralConfig(vocab_size=300, hidden_size=h, num_hidden_layers=2, num_attention_heads=heads,
                             num_key_value_heads=kv, head_dim=128, intermediate_size=i, max_position_embeddings=512,
                             sliding_window=window, initializer_range=0.02)

    def qwen3(h, i, heads, kv):
        return Qwen3Config(vocab_size=300, hidden_size=h, num_hidden_layers=2, num_attention_heads=heads,
                           num_key_value_heads=kv, head_dim=128, intermediate_size=i, max_position_embeddings=512,
                           initializer_range=0.02)

    return {
        'bert-tiny': ('bert', bert(256, 512, 4)),
        'bert-768': ('bert', bert(768, 3072, 12)),
        'modernbert-tiny': ('modernbert', modernbert(256, 192, 4)),     # intermediate padded 192 -> 256
        'modernbert-base': ('modernbert', modernbert(768, 1152, 12)),
        'mistral-tiny': ('mistral', mistral(256, 384, 4, 2, 48)),
        'mistral-7b-layers': ('mistral', mistral(4096, 14336, 32, 8, 96)),
        'qwen3-tiny': ('qwen3', qwen3(256, 384, 4, 2)),
        'qwen3-0.6b-layers': ('qwen3', qwen3(1024, 3072, 16, 8)),
    }


def _encoder_class(family):
    from distllm_b200.embed.encoders import native

    return {'bert': native.NativeBertEncoder, 'modernbert': native.NativeModernBertEncoder,
            'mistral': native.NativeMistralEncoder, 'qwen3': native.NativeQwen3Encoder}[family]


def _state_dict(family, cfg, seed):
    make = {'bert': W.random_bert_state_dict, 'modernbert': W.random_modernbert_state_dict,
            'mistral': W.random_mistral_state_dict, 'qwen3': W.random_qwen3_state_dict}[family]
    return make(cfg, seed=seed, device='cpu')


def _batch(b, s, lengths, left, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, 300, (b, s), generator=g)
    pos = torch.arange(s)[None]
    lens = torch.tensor(lengths)[:, None]
    mask = (pos >= s - lens) if left else (pos < lens)
    return ids, mask.long()


def _storages(family):
    # Mistral and Qwen3 ship on the half build only (the bfloat16 drift at depth, _native.storage_for_arch)
    return ['f16', 'bf16'] if family in ('bert', 'modernbert') else ['f16']


ENCODER_CASES = [(name, st) for name, (fam, _) in _configs().items() for st in _storages(fam)]


@pytest.mark.parametrize('name, storage', ENCODER_CASES)
def test_nf4_encoder_equals_the_load_time_16bit_encoder(name, storage):
    family, cfg = _configs()[name]
    cls = _encoder_class(family)
    sd = _state_dict(family, cfg, seed=5)
    ref_enc = cls(cfg, nf4.quantize_state_dict_nf4(sd, device=DEV), device=DEV, storage=storage)
    enc = cls(cfg, sd, device=DEV, storage=storage, nf4=True)
    try:
        wb, rb = enc.weight_bytes(), ref_enc.weight_bytes()
        assert wb['other'] == rb['other'] and wb['matrix'] <= 0.2813 * rb['matrix']
        decoder = family in ('mistral', 'qwen3')
        s = 200
        batches = {'right-padded': _batch(5, s, [200, 1, 77, 150, 128], left=False, seed=1)}
        if decoder:
            batches['left-padded'] = _batch(4, s, [200, 3, 120, 64], left=True, seed=2)
        for layout, (ids, mask) in batches.items():
            what = f'{name} {storage} {layout}'
            assert_bitwise(enc.encode(ids, mask), ref_enc.encode(ids, mask), f'{what} encode')
            kinds = [(nv.POOL_MEAN_REF, False), (nv.POOL_MEAN_REF, True)]
            if decoder:
                kinds.append((nv.POOL_LAST_TOKEN, False))
            for kind, norm in kinds:
                assert_bitwise(enc.encode_pooled(ids, mask, None, kind, norm),
                               ref_enc.encode_pooled(ids, mask, None, kind, norm), f'{what} pooled {kind} {norm}')
            kind = nv.POOL_LAST_TOKEN if decoder else nv.POOL_MEAN_REF
            for _ in range(2):   # the second call replays the captured graphs
                got = enc.embed_host(ids.contiguous(), mask.contiguous(), None, 2, kind, True)
                ref = ref_enc.embed_host(ids.contiguous(), mask.contiguous(), None, 2, kind, True)
                assert_bitwise(got, ref, f'{what} embed_host')
    finally:
        enc.close()
        ref_enc.close()
        del sd
        torch.cuda.empty_cache()


@pytest.mark.parametrize('name', ['bert-tiny', 'mistral-tiny'])
def test_nf4_gemm_with_a_device_row_count_far_below_m(name):
    """The packed layout hands every GEMM a device row count (t_real) below the M its grid is sized for: 64 rows of 256
    tokens with 2-6 attended each give M = 16 384 but 256 rows, so most of the 132 CTAs find no tile at all and
    their NF4 producers must load and dequantise nothing (b2e_gemm_nf4, like b2e_gemm_h16, takes no row count: this
    path is reached through the encoder)."""
    family, cfg = _configs()[name]
    cls = _encoder_class(family)
    sd = _state_dict(family, cfg, seed=8)
    ref_enc = cls(cfg, nf4.quantize_state_dict_nf4(sd, device=DEV), device=DEV)
    enc = cls(cfg, sd, device=DEV, nf4=True)
    try:
        lengths = [2 + 2 * (i % 3) for i in range(64)]
        ids, mask = _batch(64, 256, lengths, left=False, seed=4)
        # (the reference mean drops every row's first and last token, and with the cross-row quirk these short rows
        # would pool to zeros: the per-row mean keeps their middle tokens)
        kind = nv.POOL_LAST_TOKEN if family == 'mistral' else nv.POOL_MEAN_PER_ROW
        got = enc.encode_pooled(ids, mask, None, kind, False)
        assert_bitwise(got, ref_enc.encode_pooled(ids, mask, None, kind, False), f'{name} sparse rows')
        assert torch.isfinite(got).all() and got.abs().sum() > 0
    finally:
        enc.close()
        ref_enc.close()


def test_nf4_load_peak_memory_and_matrix_bytes_at_h4096():
    """2-layer Mistral-7B-shaped encoder: matrices at <= 0.2813x their 16-bit bytes, and the load never holds more
    than the NF4 weights, the fp32 non-matrix tensors and two fp32 copies of the largest checkpoint matrix."""
    from distllm_b200.embed.encoders.native import NativeMistralEncoder

    family, cfg = _configs()['mistral-7b-layers']
    sd = _state_dict(family, cfg, seed=9)
    largest = max(t.numel() for k, t in sd.items() if nf4.is_quantized_linear(k, t)) * 4
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    enc = NativeMistralEncoder(cfg, sd, device=DEV, nf4=True)
    try:
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated(DEV) - base
        wb = enc.weight_bytes()
        h, i, q, kv = 4096, 14336, 32 * 128, 8 * 128
        b16 = 2 * 2 * ((q + 2 * kv) * h + h * q + 2 * i * h + h * i)
        print(f'NF4-MEMORY matrix {wb["matrix"]} (16-bit {b16}) other {wb["other"]} peak {peak} largest {largest}')
        assert wb['matrix'] <= 0.2813 * b16
        assert peak <= wb['matrix'] + wb['other'] + 2 * largest, (peak, wb, largest)
    finally:
        enc.close()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- files on disk
def test_embedding_worker_quantization_true_equals_the_load_time_path(tmp_path):
    """A tiny Mistral checkpoint through embedding_worker (jsonl_chunk + semantic_chunk + last_token + numpy writer)
    with quantization: true, against quantization: false on the checkpoint quantize_state_dict_nf4 round-tripped."""
    from transformers import MistralModel

    from distllm_b200.distributed_embedding import embedding_worker
    from distllm_b200.embed import get_encoder
    from distllm_b200.registry import registry
    from oracle.make_golden import TINY_MISTRAL
    from oracle.make_golden import TINY_MISTRAL_WINDOW
    from oracle.make_golden import write_tiny_mistral_checkpoint

    write_tiny_mistral_checkpoint(tmp_path / 'ckpt', window=TINY_MISTRAL_WINDOW)
    model = MistralModel.from_pretrained(tmp_path / 'ckpt')
    q = nf4.quantize_state_dict_nf4(model.state_dict(), device=DEV)
    model.load_state_dict({k: v.cpu() for k, v in q.items()})
    model.save_pretrained(tmp_path / 'ckpt_rt')
    from transformers import AutoTokenizer

    AutoTokenizer.from_pretrained(tmp_path / 'ckpt').save_pretrained(tmp_path / 'ckpt_rt')

    words = [f'w{i:03d}' for i in range(TINY_MISTRAL['vocab_size'] - 4)]
    rng = np.random.default_rng(4)
    # sentences open with a capital (the regex splitter's boundary), as oracle.make_golden.worker_docs
    docs = [{'text': ''.join('S' + ' '.join(rng.choice(words, size=rng.integers(4, 30))) + '. '
                             for _ in range(10 + d)), 'path': f'doc{d}'} for d in range(3)]
    (tmp_path / 'docs.jsonl').write_text('\n'.join(json.dumps(d) for d in docs))
    outs = {}
    try:
        for tag, ckpt, quant in (('nf4', 'ckpt', True), ('load-time', 'ckpt_rt', False)):
            enc_kw = {'name': 'auto', 'pretrained_model_name_or_path': str(tmp_path / ckpt), 'quantization': quant}
            if quant:
                assert get_encoder(enc_kw).native.nf4
            embedding_worker(
                tmp_path / 'docs.jsonl', tmp_path / tag,
                dataset_kwargs={'name': 'jsonl_chunk', 'buffer_size': 1, 'min_buffer_length': 20, 'batch_size': 4,
                                'num_data_workers': 0, 'pin_memory': False, 'sentence_splitter': 'regex'},
                encoder_kwargs=enc_kw, pooler_kwargs={'name': 'last_token'},
                embedder_kwargs={'name': 'semantic_chunk', 'breakpoint_percentile_threshold': 70,
                                 'chunk_batch_size': 4, 'min_chunk_length': 10},
                writer_kwargs={'name': 'numpy'})
            out = [p for p in (tmp_path / tag).iterdir() if p.is_dir()]
            assert len(out) == 1, out
            outs[tag] = (np.load(out[0] / 'embeddings.npy'), np.load(out[0] / 'text.npy').tolist())
            registry.clear()
    finally:
        registry.clear()
    (emb_q, text_q), (emb_r, text_r) = outs['nf4'], outs['load-time']
    assert text_q == text_r and emb_q.shape == emb_r.shape and emb_q.shape[0] > 3
    assert np.array_equal(emb_q.view(np.int32), emb_r.view(np.int32))
