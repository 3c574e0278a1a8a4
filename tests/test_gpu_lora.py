"""-m gpu: PEFT adapter checkpoints on the H100, from the NF4 GEMM's low-rank tail up to files on disk.

  * b2e_gemm_nf4_lora equals b2e_gemm_h16 on the K-concatenated operands [A | U[:, :R]] and
    [to_storage(nf4_roundtrip(W)) | B_cat] bit for bit: the tail k-blocks are the same sums in the same order.  Every
    epilogue, R from 64 to 640 (tails of up to ten k-blocks, more than the NF4 ring's four stages), K in {64, 768,
    4096}, M off the tile grid, N across tile edges, both builds; and the encoder slot's launch sequence (U's GEMM,
    then the tail) under a device row count far below M;
  * the encoders of every family against the oracle on the adapted state dict (oracle/adapters.py), 1 - cos <= 1e-3
    per row, for the three weight paths (16-bit, quantization with nf4_storage: false, NF4 storage with the LoRA term
    unmerged), LoRA and IA3, packed and padded layouts and a left-padded Mistral batch, plus a batch whose device row
    count is far below M.  The base model must FAIL that tolerance, so a dropped or mis-laid adapter cannot pass;
  * IA3 under NF4 storage equals the nf4_storage: false encoder bit for bit (it takes that path);
  * a Mistral LoRA adapter directory shaped like the SFR scirun configs, through embedding_worker and the embed CLI.
"""

from __future__ import annotations

import json

import numpy as np
import pytest
import torch
from safetensors.torch import save_file

from distllm_b200 import _native as nv
from distllm_b200.embed.encoders import adapters as ad
from distllm_b200.embed.encoders import nf4
from distllm_b200.embed.encoders import weights as W
from oracle import adapters as oad

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


def trained_like(shape, g, device='cpu') -> torch.Tensor:
    """Entries of magnitude 1e-4 .. 1e-2, random sign: where trained lora_B entries live."""
    mag = 10.0 ** (torch.rand(shape, generator=g, device=device) * 2.0 - 4.0)
    sign = torch.randint(0, 2, shape, generator=g, device=device) * 2 - 1
    return mag * sign


# -------------------------------------------------------------------------------------------- the GEMM
GEMM_CASES = [
    # (M, N, K, R, epilogue)
    *[(m, 256, 768, 64, epi) for epi in range(5) for m in (1, 129, 1000)],
    (1000, 384, 64, 128, nv.EPI_BIAS),
    (127, 768, 768, 192, nv.EPI_BIAS_GELU),
    (4099, 3072, 768, 64, nv.EPI_BIAS_GELU),
    (1000, 768, 3072, 192, nv.EPI_BIAS_RESID),
    (129, 6144, 4096, 128, nv.EPI_BIAS),
    (257, 4096, 4096, 192, nv.EPI_BIAS_RESID),
    (1000, 28672, 4096, 64, nv.EPI_SWIGLU),
    (300, 5376, 768, 128, nv.EPI_GEGLU),
    # R / 64 at and beyond the NF4 ring's four stages: the tail of one tile spans the whole ring
    (300, 768, 768, 256, nv.EPI_BIAS_GELU),
    (1000, 6144, 4096, 384, nv.EPI_BIAS),      # Mistral-7B QKV with rank 128 on q, k and v
    (129, 4096, 4096, 512, nv.EPI_BIAS_RESID),
    (700, 2048, 768, 640, nv.EPI_SWIGLU),
]


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
@pytest.mark.parametrize('m, n, k, r, epi', GEMM_CASES)
def test_gemm_nf4_lora_equals_gemm_h16_on_the_concatenated_operands(storage, m, n, k, r, epi):
    dt = STORAGE_DTYPE[storage]
    g = torch.Generator(device=DEV).manual_seed(m + 3 * n + 5 * k + 7 * r + epi)
    w = torch.randn((n, k), generator=g, device=DEV) * 0.05
    codes, absmax = nf4.nf4_quantize(w)
    w16 = W.to_storage(nf4.nf4_dequantize(codes, absmax), DEV, dt)
    a = (torch.randn((m, k), generator=g, device=DEV) * 0.5).to(dt)
    ldu = (r + 127) // 128 * 128          # the encoder's U workspace is R rounded up to 128 wide
    u = (torch.randn((m, ldu), generator=g, device=DEV) * 0.5).to(dt)
    b_cat = (trained_like((n, r), g, device=DEV) * 4.0).to(dt)
    glu = epi in (nv.EPI_SWIGLU, nv.EPI_GEGLU)
    bias = None if glu else torch.randn(n, generator=g, device=DEV) * 0.1
    resid = torch.randn((m, n), generator=g, device=DEV).to(dt) if epi == nv.EPI_BIAS_RESID else None
    ref = nv.gemm_h16(torch.cat([a, u[:, :r]], dim=1).contiguous(), torch.cat([w16, b_cat], dim=1).contiguous(),
                      bias, resid, epi)
    got = nv.gemm_nf4_lora(a, codes, absmax, u, b_cat, bias, resid, epi)
    assert torch.isfinite(ref.float()).all()
    assert_bitwise(got, ref, f'{storage} M{m} N{n} K{k} R{r} epi{epi}')
    if epi == nv.EPI_BIAS:   # the tail is not a no-op
        assert not torch.equal(bits(got), bits(nv.gemm_nf4(a, codes, absmax, bias, None, epi)))


ROWS_CASES = [
    # (M, device rows, N, K, R, epilogue)
    (16384, 256, 768, 768, 64, nv.EPI_BIAS),
    (4096, 1000, 6144, 4096, 384, nv.EPI_BIAS),
    (2048, 300, 2048, 768, 512, nv.EPI_SWIGLU),
    (2000, 129, 768, 3072, 256, nv.EPI_BIAS_RESID),
    (640, 0, 768, 768, 128, nv.EPI_BIAS_GELU),
]


@pytest.mark.parametrize('m, m_dev, n, k, r, epi', ROWS_CASES)
def test_gemm_nf4_lora_with_a_device_row_count_equals_the_concatenated_gemm(m, m_dev, n, k, r, epi):
    """The launch sequence of an NF4 + LoRA encoder slot (U's 16-bit GEMM into a workspace, then the NF4 GEMM with
    its tail) under a device row count far below M: rows below it equal bit for bit the 16-bit GEMM over
    [A | A . A_cat^T] and [dequant(W) | B_cat], rows at or beyond it are not written."""
    import ctypes as C

    lib = nv.load('f16')
    dt = torch.float16
    g = torch.Generator(device=DEV).manual_seed(m + n + k + r + epi)
    codes, absmax = nf4.nf4_quantize(torch.randn((n, k), generator=g, device=DEV) * 0.05)
    w16 = W.to_storage(nf4.nf4_dequantize(codes, absmax), DEV, dt)
    r128 = (r + 127) // 128 * 128
    a = (torch.randn((m, k), generator=g, device=DEV) * 0.5).to(dt)
    a_cat = torch.zeros((r128, k), device=DEV)
    a_cat[:r] = torch.randn((r, k), generator=g, device=DEV) / k ** 0.5
    a_cat = a_cat.to(dt)
    b_cat = (trained_like((n, r), g, device=DEV) * 4.0).to(dt)
    glu = epi in (nv.EPI_SWIGLU, nv.EPI_GEGLU)
    bias = None if glu else torch.randn(n, generator=g, device=DEV) * 0.1
    resid = torch.randn((m, n), generator=g, device=DEV).to(dt) if epi == nv.EPI_BIAS_RESID else None
    n_out = n // 2 if glu else n
    sentinel = -12345
    out = torch.full((m, n_out), sentinel, dtype=torch.int16, device=DEV).view(dt)
    u_ws = torch.full((m, r128), sentinel, dtype=torch.int16, device=DEV).view(dt)
    md = torch.tensor([m_dev], dtype=torch.int32, device=DEV)
    lib.b2e_debug_gemm_nf4_lora_rows.restype = C.c_int
    lib.b2e_debug_gemm_nf4_lora_rows.argtypes = ([C.c_void_p] * 5 + [C.c_int] + [C.c_void_p] * 4 + [C.c_int] * 4
                                                 + [C.c_void_p] * 2)
    nv.check(lib.b2e_debug_gemm_nf4_lora_rows(
        a.data_ptr(), codes.data_ptr(), absmax.data_ptr(), a_cat.data_ptr(), b_cat.data_ptr(), r, u_ws.data_ptr(),
        nv._ptr(bias), nv._ptr(resid), out.data_ptr(), m, n, k, epi, md.data_ptr(), nv.stream_ptr(DEV)), lib)
    torch.cuda.synchronize(DEV)
    assert (out[m_dev:].view(torch.int16) == sentinel).all(), 'rows at or beyond the device row count were written'
    if m_dev == 0:
        return
    a_rows = a[:m_dev].contiguous()
    u = nv.gemm_h16(a_rows, a_cat, None)
    ref = nv.gemm_h16(torch.cat([a_rows, u[:, :r]], dim=1).contiguous(), torch.cat([w16, b_cat], dim=1).contiguous(),
                      bias, None if resid is None else resid[:m_dev].contiguous(), epi)
    assert_bitwise(out[:m_dev], ref, f'M{m} rows {m_dev} N{n} K{k} R{r} epi{epi}')


def test_gemm_nf4_lora_rejects_bad_operands():
    a = torch.zeros((128, 128), dtype=torch.float16, device=DEV)
    codes = torch.zeros((128, 64), dtype=torch.uint8, device=DEV)
    absmax = torch.zeros((2, 128), device=DEV)
    u = torch.zeros((128, 128), dtype=torch.float16, device=DEV)
    with pytest.raises(nv.NativeError, match='multiple of 64'):
        nv.gemm_nf4_lora(a, codes, absmax, u, torch.zeros((128, 96), dtype=torch.float16, device=DEV), None)
    with pytest.raises(nv.NativeError, match='ldu >= R'):
        nv.gemm_nf4_lora(a, codes, absmax, u[:, :64].contiguous(),
                         torch.zeros((128, 128), dtype=torch.float16, device=DEV), None)


# ------------------------------------------------------------------------------------------- encoders
def _configs():
    from transformers import BertConfig
    from transformers import EsmConfig
    from transformers import MistralConfig
    from transformers import ModernBertConfig
    from transformers import Qwen3Config

    return {
        'bert': BertConfig(vocab_size=300, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                           intermediate_size=512, max_position_embeddings=512, initializer_range=0.05),
        'modernbert': ModernBertConfig(vocab_size=300, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                       intermediate_size=192, max_position_embeddings=512, local_attention=64,
                                       pad_token_id=0, bos_token_id=1, eos_token_id=2, cls_token_id=1,
                                       sep_token_id=2),
        'mistral': MistralConfig(vocab_size=300, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                 num_key_value_heads=2, head_dim=128, intermediate_size=384,
                                 max_position_embeddings=512, sliding_window=48, initializer_range=0.02),
        'qwen3': Qwen3Config(vocab_size=300, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                             num_key_value_heads=2, head_dim=128, intermediate_size=384, max_position_embeddings=512,
                             initializer_range=0.02),
        'esm': EsmConfig(vocab_size=33, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                         intermediate_size=512, max_position_embeddings=1026, position_embedding_type='rotary',
                         token_dropout=False, pad_token_id=1, mask_token_id=32, initializer_range=0.05),
    }


def _oracle(family):
    from oracle import bert, esm, mistral, modernbert
    from tools import oracle_qwen3

    return {'bert': bert.bert_forward, 'esm': esm.esm_forward, 'mistral': mistral.mistral_forward,
            'modernbert': modernbert.modernbert_forward, 'qwen3': oracle_qwen3.qwen3_forward}[family]


_MODULES = {
    'bert': ('encoder.layer.{}.', {'qv': ['attention.self.query', 'attention.self.value'],
                                   'ia3': ['attention.self.key', 'attention.self.value', 'attention.output.dense',
                                           'output.dense']}),
    'esm': ('esm.encoder.layer.{}.', {'qv': ['attention.self.query', 'attention.self.value'],
                                      'ia3': ['attention.self.key', 'attention.self.value',
                                              'attention.output.dense', 'output.dense']}),
    'modernbert': ('layers.{}.', {'all': ['attn.Wqkv', 'attn.Wo', 'mlp.Wi', 'mlp.Wo']}),
    'mistral': ('layers.{}.', {'qv': ['self_attn.q_proj', 'self_attn.v_proj'],
                               'all': ['self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj', 'self_attn.o_proj',
                                       'mlp.gate_proj', 'mlp.up_proj', 'mlp.down_proj']}),
    'qwen3': ('layers.{}.', {'all': ['self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj',
                                     'self_attn.o_proj', 'mlp.gate_proj', 'mlp.up_proj', 'mlp.down_proj']}),
}


def _checkpoint(family, root):
    """A seeded base checkpoint on disk (tokenizer from the tiny BERT / ESM checkpoints) -> (path, config, sd)."""
    from transformers import AutoModel
    from transformers import EsmForMaskedLM

    from oracle.make_golden import write_tiny_bert_checkpoint
    from oracle.make_golden import write_tiny_esm_checkpoint

    cfg = _configs()[family]
    path = root / family
    torch.manual_seed(17)
    model = EsmForMaskedLM(cfg) if family == 'esm' else AutoModel.from_config(cfg)
    sd = model.state_dict()
    g = torch.Generator().manual_seed(5)
    std = 0.05 if family in ('bert', 'esm') else 0.02
    for k, v in sd.items():
        if v.dim() == 2 and 'embed' not in k:
            sd[k] = torch.randn(v.shape, generator=g) * std
        elif k.endswith('.bias'):
            sd[k] = torch.randn(v.shape, generator=g) * 0.05
    model.load_state_dict(sd)
    model.save_pretrained(path)
    tok = root / f'{family}_tok'
    (write_tiny_esm_checkpoint if family == 'esm' else write_tiny_bert_checkpoint)(tok)
    return path, cfg, model.state_dict(), tok


def _adapter(family, kind, sd, base, root, seed):
    prefix, groups = _MODULES[family]
    names = groups[kind]
    mods = [prefix.format(layer) + n for layer in (0, 1) for n in names]
    g = torch.Generator().manual_seed(seed)
    tensors = {}
    if kind == 'ia3':
        config = {'peft_type': 'IA3', 'base_model_name_or_path': str(base), 'target_modules': ['key', 'value',
                  'output.dense'], 'feedforward_modules': ['output.dense'], 'modules_to_save': None}
        for m in mods:
            o, i = sd[m + '.weight'].shape
            shape = (1, i) if m.endswith('.output.dense') and 'attention' not in m else (o, 1)
            tensors[f'base_model.model.{m}.ia3_l'] = 1.0 + 0.5 * torch.randn(*shape, generator=g)
    else:
        r = 8
        # ModernBERT's pre-LN blocks damp a rank-8 change most: a larger scaling keeps B in the trained range
        config = {'peft_type': 'LORA', 'base_model_name_or_path': str(base), 'r': r,
                  'lora_alpha': 256 if family == 'modernbert' else 32,
                  'bias': 'none', 'modules_to_save': None, 'use_dora': False, 'fan_in_fan_out': False}
        for m in mods:
            o, i = sd[m + '.weight'].shape
            tensors[f'base_model.model.{m}.lora_A.weight'] = torch.randn(r, i, generator=g) / i ** 0.5
            tensors[f'base_model.model.{m}.lora_B.weight'] = trained_like((o, r), g) * 3.0
    d = root / f'{family}_{kind}_{seed}'
    d.mkdir()
    (d / ad.ADAPTER_CONFIG).write_text(json.dumps(config))
    save_file(tensors, str(d / 'adapter_model.safetensors'))
    return d, tensors, config


def _batches(family):
    g = torch.Generator().manual_seed(9)
    vocab = 33 if family == 'esm' else 300
    s = 160
    ids = torch.randint(4, vocab - 1, (5, s), generator=g)
    lens = torch.tensor([160, 1, 77, 130, 64])[:, None]
    out = {'right-padded': (ids, (torch.arange(s)[None] < lens).long())}
    if family in ('mistral', 'qwen3'):
        out['left-padded'] = (ids[:4], (torch.arange(s)[None] >= s - lens[:4]).long())
    return out


def _rows_1mcos(got: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    got, ref = got.double(), ref.double()
    return 1.0 - (got * ref).sum(-1) / (got.norm(dim=-1) * ref.norm(dim=-1)).clamp_min(1e-30)


def _pooled_ref(family, hidden, mask):
    from oracle import pooling

    if family in ('mistral', 'qwen3'):
        return pooling.last_token_pool(hidden, mask)
    return pooling.average_pool(hidden, mask.clone())


def _check_encoder(enc, family, sd_base, tensors, config, what):
    fwd = _oracle(family)
    adapted = oad.adapted_state_dict(sd_base, tensors, config)
    decoder = family in ('mistral', 'qwen3')
    kind = nv.POOL_LAST_TOKEN if decoder else nv.POOL_MEAN_REF
    for layout, (ids, mask) in _batches(family).items():
        ref = fwd(adapted, enc.native.hf_config, ids, mask)
        base = fwd(sd_base, enc.native.hf_config, ids, mask)
        live = mask.bool()
        hid = enc.encode({'input_ids': ids, 'attention_mask': mask}).cpu()
        err = _rows_1mcos(hid[live], ref[live])
        assert err.max() <= 1e-3, f'{what} {layout} encode: 1-cos {err.max():.3g}'
        assert _rows_1mcos(base[live], ref[live]).max() > 1e-3, f'{what}: the adapter is too weak to be seen'
        pooled = enc.encode_pooled({'input_ids': ids, 'attention_mask': mask}, kind, False).cpu()
        pref = _pooled_ref(family, ref, mask)
        nz = pref.norm(dim=-1) > 0
        err = _rows_1mcos(pooled[nz], pref[nz])
        assert err.max() <= 1e-3, f'{what} {layout} pooled: 1-cos {err.max():.3g}'


ENCODER_CASES = [
    ('bert', 'qv'), ('bert', 'ia3'), ('modernbert', 'all'), ('mistral', 'qv'), ('mistral', 'all'), ('qwen3', 'all'),
]
PATHS = {'16-bit': dict(quantization=False), 'nf4-load-time': dict(quantization=True, nf4_storage=False),
         'nf4-storage': dict(quantization=True, nf4_storage=True)}


@pytest.fixture(scope='module')
def ckpts(tmp_path_factory):
    root = tmp_path_factory.mktemp('lora')
    return root, {f: _checkpoint(f, root) for f in ('bert', 'modernbert', 'mistral', 'qwen3', 'esm')}


@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('family, kind', ENCODER_CASES)
def test_auto_encoder_with_an_adapter_matches_the_oracle(ckpts, family, kind, path):
    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig

    root, table = ckpts
    base, cfg, sd, tok = table[family]
    d, tensors, config = _adapter(family, kind, sd, base, root, seed=len(path) + 31 * len(kind))
    enc = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(d), tokenizer_name=str(tok), **PATHS[path]))
    try:
        unmerged = path == 'nf4-storage' and kind != 'ia3'
        assert enc.native.nf4 == unmerged and bool(enc.native._lora) == unmerged
        sd_base = nf4.quantize_state_dict_nf4(sd) if path != '16-bit' else sd
        _check_encoder(enc, family, sd_base, tensors, config, f'{family} {kind} {path}')
    finally:
        enc.native.close()
        torch.cuda.empty_cache()


@pytest.mark.parametrize('kind', ['qv', 'ia3'])
def test_esm2_encoder_with_an_adapter_matches_the_oracle(ckpts, kind):
    from distllm_b200.embed.encoders.esm2 import Esm2Encoder
    from distllm_b200.embed.encoders.esm2 import Esm2EncoderConfig

    root, table = ckpts
    base, cfg, sd, tok = table['esm']
    d, tensors, config = _adapter('esm', kind, sd, base, root, seed=40 + len(kind))
    enc = Esm2Encoder(Esm2EncoderConfig(pretrained_model_name_or_path=str(d), tokenizer_path=str(tok),
                                        half_precision=False))
    try:
        _check_encoder(enc, 'esm', sd, tensors, config, f'esm {kind}')
    finally:
        enc.native.close()


@pytest.mark.parametrize('family', ['bert', 'mistral'])
def test_nf4_lora_encoder_with_a_device_row_count_far_below_m(ckpts, family):
    """64 rows of 256 tokens with 2-6 attended: the packed layout hands U's GEMM and the tail-carrying GEMM 256 device
    rows out of M = 16 384, so most CTAs have no tile; rows past the device count of U are never read into an output."""
    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig

    root, table = ckpts
    base, cfg, sd, tok = table[family]
    kind = 'qv'
    d, tensors, config = _adapter(family, kind, sd, base, root, seed=77)
    enc = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(d), tokenizer_name=str(tok)))
    try:
        assert enc.native.nf4 and enc.native._lora
        g = torch.Generator().manual_seed(4)
        ids = torch.randint(4, 299, (64, 256), generator=g)
        lens = torch.tensor([2 + 2 * (i % 3) for i in range(64)])[:, None]
        mask = (torch.arange(256)[None] < lens).long()
        pk = nv.POOL_LAST_TOKEN if family == 'mistral' else nv.POOL_MEAN_PER_ROW
        got = enc.encode_pooled({'input_ids': ids, 'attention_mask': mask}, pk, False).cpu()
        ref = _oracle(family)(oad.adapted_state_dict(nf4.quantize_state_dict_nf4(sd), tensors, config), cfg, ids, mask)
        if family == 'mistral':
            pref = ref[torch.arange(64), lens[:, 0] - 1]
        else:   # per-row mean without the row's own first and last token
            keep = mask.clone()
            keep[:, 0] = 0
            keep[torch.arange(64), lens[:, 0] - 1] = 0
            pref = (ref * keep[..., None]).sum(1) / keep.sum(1, keepdim=True).clamp_min(1)
        nz = pref.norm(dim=-1) > 0
        assert torch.isfinite(got).all() and nz.sum() > 32
        assert _rows_1mcos(got[nz], pref[nz]).max() <= 1e-3
    finally:
        enc.native.close()


def test_ia3_under_nf4_storage_equals_the_nf4_storage_false_encoder_bit_for_bit(ckpts):
    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig

    root, table = ckpts
    base, cfg, sd, tok = table['bert']
    d, _, _ = _adapter('bert', 'ia3', sd, base, root, seed=91)
    a = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(d), tokenizer_name=str(tok)))
    b = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(d), tokenizer_name=str(tok),
                                      nf4_storage=False))
    try:
        assert not a.native.nf4
        for ids, mask in _batches('bert').values():
            batch = {'input_ids': ids, 'attention_mask': mask}
            assert_bitwise(a.encode(batch), b.encode(batch), 'ia3 encode')
            assert_bitwise(a.encode_pooled(batch, nv.POOL_MEAN_REF, True), b.encode_pooled(batch, nv.POOL_MEAN_REF,
                                                                                           True), 'ia3 pooled')
    finally:
        a.native.close()
        b.native.close()


# ------------------------------------------------------------------------------------------- files on disk
def test_mistral_scirun_shaped_lora_adapter_end_to_end(tmp_path):
    """A local Mistral base, an adapter-only directory pointing at it, tokenizer_name, the last_token pooler and
    normalize_embeddings: true, quantization: true (NF4 storage, LoRA unmerged), through embedding_worker and the
    embed CLI: rows equal to the oracle, and b2e_embed_host equal to encode_pooled bit for bit."""
    import subprocess
    import sys

    from transformers import AutoModel

    from distllm_b200.distributed_embedding import embedding_worker
    from distllm_b200.embed import get_encoder
    from distllm_b200.registry import registry
    from oracle import mistral as omistral
    from oracle import pooling
    from oracle.make_golden import TINY_MISTRAL
    from oracle.make_golden import write_tiny_mistral_checkpoint

    write_tiny_mistral_checkpoint(tmp_path / 'base')
    sd = AutoModel.from_pretrained(tmp_path / 'base').state_dict()
    adir = tmp_path / 'checkpoint-100'
    adir.mkdir()
    g = torch.Generator().manual_seed(3)
    mods = [f'layers.{l}.{n}' for l in range(TINY_MISTRAL['num_hidden_layers'])
            for n in ('self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj', 'self_attn.o_proj',
                      'mlp.gate_proj', 'mlp.up_proj', 'mlp.down_proj')]
    tensors = {}
    for m in mods:
        o, i = sd[m + '.weight'].shape
        tensors[f'base_model.model.{m}.lora_A.weight'] = torch.randn(16, i, generator=g) / i ** 0.5
        tensors[f'base_model.model.{m}.lora_B.weight'] = trained_like((o, 16), g) * 3.0
    config = {'peft_type': 'LORA', 'base_model_name_or_path': str(tmp_path / 'base'), 'r': 16, 'lora_alpha': 32,
              'bias': 'none', 'task_type': 'FEATURE_EXTRACTION'}
    (adir / ad.ADAPTER_CONFIG).write_text(json.dumps(config))
    save_file(tensors, str(adir / 'adapter_model.safetensors'))

    texts = [f'S{" ".join(f"w{(7 * d + j) % 300:03d}" for j in range(5 + 3 * d))}.' for d in range(9)]
    (tmp_path / 'data').mkdir()
    (tmp_path / 'data' / 'in.jsonl').write_text('\n'.join(json.dumps({'text': t}) for t in texts) + '\n')
    enc_kw = {'name': 'auto', 'pretrained_model_name_or_path': str(adir), 'tokenizer_name': str(tmp_path / 'base'),
              'quantization': True}
    try:
        enc = get_encoder(enc_kw)
        assert enc.native.nf4 and enc.native._lora
        tok = enc.tokenizer
        batch = tok(texts, padding=True, truncation=True, return_tensors='pt')
        ids, mask = batch['input_ids'], batch['attention_mask']
        ref = omistral.mistral_forward(oad.adapted_state_dict(nf4.quantize_state_dict_nf4(sd), tensors, config),
                                       enc.native.hf_config, ids, mask)
        ref = pooling.normalize(pooling.last_token_pool(ref, mask))
        pooled = enc.encode_pooled(batch, nv.POOL_LAST_TOKEN, True)
        assert _rows_1mcos(pooled.cpu(), ref).max() <= 1e-3
        host = enc.native.embed_host(ids.contiguous(), mask.contiguous(), None, len(texts), nv.POOL_LAST_TOKEN, True)
        assert_bitwise(host, pooled.cpu(), 'embed_host vs encode_pooled')
        registry.clear()
        embedding_worker(
            tmp_path / 'data' / 'in.jsonl', tmp_path / 'worker',
            dataset_kwargs={'name': 'jsonl', 'batch_size': 4, 'num_data_workers': 0, 'pin_memory': False},
            encoder_kwargs=enc_kw, pooler_kwargs={'name': 'last_token'},
            embedder_kwargs={'name': 'full_sequence', 'normalize_embeddings': True}, writer_kwargs={'name': 'numpy'})
        out = [p for p in (tmp_path / 'worker').iterdir() if p.is_dir()]
        assert len(out) == 1
        emb = torch.from_numpy(np.load(out[0] / 'embeddings.npy'))
        order = [texts.index(t) for t in np.load(out[0] / 'text.npy').tolist()]
        assert _rows_1mcos(emb.float(), ref[order]).max() <= 1e-3
    finally:
        registry.clear()
    # the embed CLI (reference flag spellings): no tokenizer flag, so the adapter directory's base tokenizer
    import os

    from conftest import REPO

    cmd = [sys.executable, '-m', 'distllm_b200.cli', 'embed', '--encoder_name', 'auto', '-m', str(adir),
           '-d', str(tmp_path / 'data'), '-de', 'jsonl', '-o', str(tmp_path / 'cli'), '--dataset_name', 'jsonl',
           '-b', '4', '--pooler_name', 'last_token', '--embedder_name', 'full_sequence', '--writer_name', 'numpy',
           '--quantization']
    run = subprocess.run(cmd, env={**os.environ, 'PYTHONPATH': str(REPO)}, capture_output=True, text=True,
                         timeout=900, check=False)
    assert run.returncode == 0, run.stderr[-3000:]
    files = list((tmp_path / 'cli').rglob('embeddings.npy'))
    assert len(files) == 1
    emb = torch.from_numpy(np.load(files[0]))
    texts_cli = np.load(files[0].parent / 'text.npy').tolist()
    assert _rows_1mcos(emb.float(), ref[[texts.index(t) for t in texts_cli]]).max() <= 1e-3
