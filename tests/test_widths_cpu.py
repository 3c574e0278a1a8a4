"""Hidden widths without a device: which (family, width) pairs b2e_check_model accepts in both builds, AutoEncoder /
Esm2Encoder validation of bge-large- and esm2_t36_3B-shaped checkpoint directories, and the shapes that stay rejected
with the errors they give.  tests/test_gpu_widths.py runs every accepted pair against the oracle."""

from __future__ import annotations

import ctypes as C

import pytest
import torch

from distllm_b200 import _native

# The row kernels are instantiated per width (DISPATCH_H in csrc/b2e_api.cu).
BUILT_WIDTHS = (256, 384, 512, 640, 768, 1024, 1280, 2048, 2560, 4096)
MULTIPLES_OF_256 = tuple(h for h in BUILT_WIDTHS if h % 256 == 0)


def desc(arch, hidden, heads, head_dim, intermediate, layers=2, kv_heads=None):
    return _native.ModelDesc(arch=arch, num_layers=layers, hidden=hidden, heads=heads, kv_heads=kv_heads or heads,
                             head_dim=head_dim, intermediate=intermediate, vocab=100, max_pos=512,
                             sliding_window=64, global_every=3)


def accepted(storage):
    """Every (family, width, head_dim) b2e_check_model accepts."""
    out = []
    for h in BUILT_WIDTHS:
        out.append(desc(_native.ARCH_BERT, h, h // 64, 64, 4 * h))
        out.append(desc(_native.ARCH_BERT, h, h // 32, 32, 4 * h))
        out.append(desc(_native.ARCH_ESM2, h, h // 64, 64, 4 * h))
        out.append(desc(_native.ARCH_ESM2, h, h // 32, 32, 4 * h))
    for h in MULTIPLES_OF_256:
        out.append(desc(_native.ARCH_MODERNBERT, h, h // 64, 64, 3 * h // 2))
        heads = h // 128
        out.append(desc(_native.ARCH_MISTRAL, h, heads, 128, 2 * h, kv_heads=max(1, heads // 4)))
    return out


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
def test_check_model_accepts_every_built_width(storage):
    lib = _native.load(storage)
    for d in accepted(storage):
        assert lib.b2e_check_model(C.byref(d)) == 0, (d.arch, d.hidden, d.head_dim, lib.b2e_last_error())
    # the published shapes among them
    for d in (desc(_native.ARCH_BERT, 1024, 16, 64, 4096, 24),          # bge-large-en-v1.5, e5-large-v2
              desc(_native.ARCH_ESM2, 2560, 40, 64, 10240, 36),         # esm2_t36_3B
              desc(_native.ARCH_ESM2, 1280, 20, 64, 5120, 33),          # esm2_t33_650M
              desc(_native.ARCH_MODERNBERT, 1024, 16, 64, 2688, 28),    # ModernBERT-large, I zero-padded 2624 -> 2688
              desc(_native.ARCH_MISTRAL, 4096, 32, 128, 14336, 32, kv_heads=8)):   # Mistral-7B
        assert lib.b2e_check_model(C.byref(d)) == 0, (d.arch, d.hidden, lib.b2e_last_error())


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
def test_check_model_rejects_unbuilt_widths_with_their_errors(storage):
    lib = _native.load(storage)
    cases = []
    for h in (320, 480):
        msg = f'hidden size {h} must be a multiple of 256, or 384 or 640'.encode()
        cases += [(desc(_native.ARCH_BERT, h, h // 32, 32, 4 * h), msg),
                  (desc(_native.ARCH_ESM2, h, h // 32, 32, 4 * h), msg)]
    cases.append((desc(_native.ARCH_MODERNBERT, 320, 5, 64, 512), b'ModernBERT: hidden size 320 must be a multiple of 256'))
    for h in (1536, 1792, 3072):
        msg = f'hidden size {h} not supported (built: 256 x {{1,2,3,4,5,8,10,16}}, 384, 640)'.encode()
        cases += [(desc(_native.ARCH_BERT, h, h // 64, 64, 4 * h), msg),
                  (desc(_native.ARCH_BERT, h, h // 32, 32, 4 * h), msg),
                  (desc(_native.ARCH_ESM2, h, h // 64, 64, 4 * h), msg),
                  (desc(_native.ARCH_MODERNBERT, h, h // 64, 64, 2 * h), msg),
                  (desc(_native.ARCH_MISTRAL, h, h // 128, 128, 2 * h, kv_heads=1), msg)]
    for h in (384, 640):
        cases += [(desc(_native.ARCH_MISTRAL, h, 2, 128, 1024), f'Mistral: hidden size {h} must be a multiple of 256'.encode()),
                  (desc(_native.ARCH_MODERNBERT, h, h // 64, 64, 2 * h),
                   f'ModernBERT: hidden size {h} must be a multiple of 256'.encode())]
    # ModernBERT-large's published intermediate size: the gated epilogue needs 2I % 256 == 0.  (The Python
    # description, weights.modernbert_desc, zero-pads it to 2688 first; see the validation test below.)
    cases.append((desc(_native.ARCH_MODERNBERT, 1024, 16, 64, 2624, 28),
                  b'ModernBERT: 2 * intermediate_size = 5248 must be a multiple of 256'))
    for d, msg in cases:
        assert lib.b2e_check_model(C.byref(d)) in (1, 3), (d.arch, d.hidden, d.head_dim)
        assert msg in lib.b2e_last_error(), (d.arch, d.hidden, lib.b2e_last_error())


def test_num_weights_does_not_depend_on_width():
    lib = _native.load()
    for h in BUILT_WIDTHS:
        assert lib.b2e_num_weights(C.byref(desc(_native.ARCH_BERT, h, h // 64, 64, 4 * h, 3))) == 5 + 12 * 3
        assert lib.b2e_num_weights(C.byref(desc(_native.ARCH_ESM2, h, h // 64, 64, 4 * h, 3))) == 3 + 12 * 3


def _no_device_or_built(ctor, embedding_size):
    """With a GPU the encoder builds; on a box without one the construction fails for want of a device (the shape
    has passed validation by then)."""
    if torch.cuda.is_available():
        assert ctor().embedding_size == embedding_size
    else:
        with pytest.raises(_native.NativeError, match='no CUDA device'):
            ctor()


def test_auto_encoder_validates_a_bge_large_checkpoint(tmp_path):
    """bge-large-en-v1.5 / e5-large-v2 layer shape: BERT, H = 1024, 16 heads x 64, I = 4096."""
    from transformers import AutoConfig
    from transformers import BertConfig
    from transformers import BertModel

    from distllm_b200.embed.encoders.auto import AutoEncoder
    from distllm_b200.embed.encoders.auto import AutoEncoderConfig
    from distllm_b200.embed.encoders.native import NativeBertEncoder

    cfg = BertConfig(vocab_size=120, hidden_size=1024, num_hidden_layers=1, num_attention_heads=16,
                     intermediate_size=4096, max_position_embeddings=64)
    ckpt = tmp_path / 'bge-large'
    BertModel(cfg).save_pretrained(ckpt)
    (ckpt / 'vocab.txt').write_text('\n'.join(['[PAD]', '[UNK]', '[CLS]', '[SEP]', '[MASK]'] +
                                              [f'w{i}' for i in range(115)]) + '\n')
    NativeBertEncoder.validate(AutoConfig.from_pretrained(ckpt))
    _no_device_or_built(lambda: AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(ckpt),
                                                              quantization=False)), 1024)
    cfg.hidden_size = 1536       # 24 x 64: not a built width, rejected before the weights are read
    cfg.num_attention_heads = 24
    bad = tmp_path / 'bad'
    cfg.save_pretrained(bad)
    with pytest.raises(_native.NativeError, match='hidden size 1536 not supported'):
        AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(bad), quantization=False))


def test_esm2_encoder_validates_an_esm2_3b_checkpoint(tmp_path):
    """esm2_t36_3B layer shape: ESM-2, H = 2560, 40 heads x 64, I = 10240."""
    from transformers import AutoConfig
    from transformers import EsmConfig

    from distllm_b200.embed.encoders.esm2 import Esm2Encoder
    from distllm_b200.embed.encoders.esm2 import Esm2EncoderConfig
    from distllm_b200.embed.encoders.native import NativeEsm2Encoder

    cfg = EsmConfig(vocab_size=33, hidden_size=2560, num_hidden_layers=36, num_attention_heads=40,
                    intermediate_size=10240, max_position_embeddings=1026, position_embedding_type='rotary',
                    token_dropout=True, mask_token_id=32, pad_token_id=1, layer_norm_eps=1e-5,
                    emb_layer_norm_before=False)
    ckpt = tmp_path / 'esm2_t36_3B'
    cfg.save_pretrained(ckpt)
    NativeEsm2Encoder.validate(AutoConfig.from_pretrained(ckpt))
    # the encoder validates config.json before it reads a weight (this directory has none)
    cfg.hidden_size, cfg.num_attention_heads, cfg.intermediate_size = 3072, 48, 12288
    bad = tmp_path / 'bad'
    cfg.save_pretrained(bad)
    with pytest.raises(_native.NativeError, match='hidden size 3072 not supported'):
        Esm2Encoder(Esm2EncoderConfig(pretrained_model_name_or_path=str(bad)))


def test_modernbert_large_config_validates_through_its_padded_intermediate():
    """The published ModernBERT-large configuration (H = 1024, 16 x 64, I = 2624): b2e_check_model rejects I = 2624
    (previous test), and the Python description zero-pads it to the next multiple of 128, which passes."""
    from transformers import ModernBertConfig

    from distllm_b200.embed.encoders import weights as W
    from distllm_b200.embed.encoders.native import NativeModernBertEncoder

    cfg = ModernBertConfig(hidden_size=1024, num_hidden_layers=28, num_attention_heads=16, intermediate_size=2624)
    assert W.modernbert_desc(cfg).intermediate == 2688
    NativeModernBertEncoder.validate(cfg)
    for h in (384, 640, 1536):
        bad = ModernBertConfig(hidden_size=h, num_hidden_layers=2, num_attention_heads=h // 64, intermediate_size=h)
        with pytest.raises(_native.NativeError, match=f'hidden size {h}'):
            NativeModernBertEncoder.validate(bad)
