"""NF4 weight storage on the CPU: the device format of embed/encoders/nf4.py and the assembled weight slots.

The NF4 GEMM computes round16(code[q] * absmax') from (codes, absmax') in front of the tensor cores.  These tests pin,
without a GPU, every step of the argument that this equals the 16-bit matrix the load-time path hands the 16-bit GEMM,
to_storage(nf4_roundtrip(W)), bit for bit:
  * nf4_dequantize(*nf4_quantize(W)) == the round trip as it stood before the device format existed;
  * an independent numpy emulation of the kernel's arithmetic (fp32 product, bfloat16 round-to-nearest-even or the
    half clamp + round-to-nearest) == to_storage(nf4_roundtrip(W));
  * the assembled NF4 slots of every family dequantise to exactly today's 16-bit slots, padding included;
  * the nibble order, the [K/64, N] scale layout and the kernel's code table.
"""

from __future__ import annotations

import re

import numpy as np
import pytest
import torch

from conftest import REPO
from distllm_b200.embed.encoders import nf4
from distllm_b200.embed.encoders import weights as W


def parent_roundtrip(weight: torch.Tensor, blocksize: int = 64, double_quant: bool = True) -> torch.Tensor:
    """nf4_roundtrip as it was before the device format (one full-size pass, int64 codes)."""
    w = weight.detach().to(torch.float32)
    flat = w.flatten()
    n = flat.numel()
    pad = (-n) % blocksize
    if pad:
        flat = torch.cat([flat, flat.new_zeros(pad)])
    blocks = flat.view(-1, blocksize)
    absmax = blocks.abs().amax(dim=1)
    code = torch.tensor(nf4.NF4_CODE, dtype=torch.float32, device=w.device)
    safe = torch.where(absmax > 0, absmax, torch.ones_like(absmax))
    q4 = nf4._nearest(blocks / safe[:, None], code)
    if double_quant:
        code8 = nf4.dynamic_map_8bit().to(w.device)
        offset = absmax.mean()
        centred = absmax - offset
        pad2 = (-centred.numel()) % 256
        c = torch.cat([centred, centred.new_zeros(pad2)]) if pad2 else centred
        c = c.view(-1, 256)
        absmax2 = c.abs().amax(dim=1)
        safe2 = torch.where(absmax2 > 0, absmax2, torch.ones_like(absmax2))
        q8 = nf4._nearest(c / safe2[:, None], code8)
        absmax = (code8[q8] * absmax2[:, None]).flatten()[: absmax.numel()] + offset
    out = (code[q4] * absmax[:, None]).flatten()[:n]
    return out.view_as(w)


def bits(t: torch.Tensor) -> torch.Tensor:
    """Bit pattern (so that -0.0 != +0.0)."""
    return t.contiguous().view({4: torch.int32, 2: torch.int16}[t.element_size()])


def matrices() -> dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(7)
    out = {
        'random 96x256 (384 blocks)': torch.randn(96, 256, generator=g) * 0.02,
        'random 128x512 (1024 blocks = 4 x 256)': torch.randn(128, 512, generator=g) * 0.02,
        'random 3x64 (3 blocks)': torch.randn(3, 64, generator=g),
        'random 256x4096 (2^14 blocks)': torch.randn(256, 4096, generator=g) * 0.03,
    }
    z = torch.randn(64, 256, generator=g) * 0.02
    z[5] = 0.0                       # all-zero blocks (a whole row)
    z[9, 64:128] = 0.0
    z[10, :64] = 0.25                # constant blocks
    z[11, 128:192] = -0.125
    z[12, 3] = 40.0                  # outlier blocks
    z[40, 200] = -1e3
    out['zero / constant / outlier blocks'] = z
    out['bfloat16 checkpoint'] = (torch.randn(128, 192, generator=g) * 0.05).to(torch.bfloat16)
    return out


@pytest.mark.parametrize('double_quant', [True, False])
def test_quantize_dequantize_is_the_parent_roundtrip_bitwise(double_quant):
    for name, w in matrices().items():
        codes, absmax = nf4.nf4_quantize(w, double_quant=double_quant)
        n, k = w.shape
        assert codes.dtype == torch.uint8 and tuple(codes.shape) == (n, k // 2), name
        assert absmax.dtype == torch.float32 and tuple(absmax.shape) == (k // 64, n) and absmax.is_contiguous(), name
        ref = parent_roundtrip(w, double_quant=double_quant)
        assert torch.equal(bits(nf4.nf4_dequantize(codes, absmax)), bits(ref)), name
        assert torch.equal(bits(nf4.nf4_roundtrip(w, double_quant=double_quant)), bits(ref)), name


def test_roundtrip_of_shapes_outside_the_device_format_is_unchanged():
    g = torch.Generator().manual_seed(3)
    for shape in [(96, 200), (7, 9), (1000,), (4, 5, 32)]:
        w = torch.randn(*shape, generator=g) * 0.02
        assert not nf4.nf4_storable(w)
        for dq in (True, False):
            assert torch.equal(bits(nf4.nf4_roundtrip(w, double_quant=dq)), bits(parent_roundtrip(w, double_quant=dq)))
    with pytest.raises(ValueError, match='K % 64'):
        nf4.nf4_quantize(torch.zeros(4, 96))


def test_quantize_in_chunks_equals_one_pass(monkeypatch):
    """The code search runs in chunks of blocks to bound its temporaries; the chunk size cannot change a bit."""
    w = torch.randn(300, 640, generator=torch.Generator().manual_seed(1)) * 0.02
    whole = nf4.nf4_quantize(w)
    monkeypatch.setattr(nf4, '_CHUNK_BLOCKS', 7)
    chunked = nf4.nf4_quantize(w)
    assert torch.equal(whole[0], chunked[0]) and torch.equal(bits(whole[1]), bits(chunked[1]))


def _round_bf16(x: np.ndarray) -> np.ndarray:
    """fp32 -> bfloat16 bit patterns, round to nearest even (cvt.rn.bf16x2.f32 for finite values)."""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return u.astype(np.uint16)


def _device_formula(codes: torch.Tensor, absmax: torch.Tensor, dtype: torch.dtype) -> np.ndarray:
    """The kernel's producer, restated in numpy: nibbles high-first, code table lookup, one fp32 product, then the
    storage rounding (half: clamp to +-65504, round to nearest even)."""
    c = codes.numpy()
    q = np.empty((c.shape[0], c.shape[1] * 2), dtype=np.int64)
    q[:, 0::2], q[:, 1::2] = c >> 4, c & 15
    table = np.array(nf4.NF4_CODE, dtype=np.float32)
    scale = np.repeat(absmax.numpy().T, 64, axis=1).astype(np.float32)
    prod = np.multiply(table[q], scale, dtype=np.float32)
    if dtype == torch.float16:
        return np.clip(prod, -65504.0, 65504.0).astype(np.float16).view(np.int16)
    return _round_bf16(prod).view(np.int16)


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_device_formula_equals_the_16bit_matrix_of_the_load_time_path(dtype):
    ms = matrices()
    # beyond half's range: the clamp (the half build's saturation) must agree too
    ms['large scale'] = torch.randn(64, 128, generator=torch.Generator().manual_seed(5)) * 4e4
    for name, w in ms.items():
        ref = W.to_storage(nf4.nf4_roundtrip(w), torch.device('cpu'), dtype)
        got = _device_formula(*nf4.nf4_quantize(w), dtype)
        assert np.array_equal(got, bits(ref).numpy()), name
    assert (W.to_storage(nf4.nf4_roundtrip(ms['large scale']), torch.device('cpu'), torch.float16).abs()
            == 65504).any()


def test_nibble_order_and_scale_layout():
    """Byte j of a row: column 2j in the high nibble, 2j+1 in the low one; absmax[kb, n] = scale of row n's k-block kb."""
    n, k = 3, 192
    q = torch.randint(0, 16, (n, k), generator=torch.Generator().manual_seed(0))
    q[:, 0] = 15                                  # every block holds +1.0 x its scale: absmax = scale exactly
    q[:, 64] = q[:, 128] = 15
    scale = torch.tensor([[1.0, 2.0, 4.0], [0.5, 8.0, 0.25], [16.0, 1.0, 2.0]])   # [row, k-block]
    w = torch.tensor(nf4.NF4_CODE)[q] * scale.repeat_interleave(64, dim=1)
    codes, absmax = nf4.nf4_quantize(w, double_quant=False)
    assert torch.equal(codes.long(), q[:, 0::2] * 16 + q[:, 1::2])
    assert torch.equal(absmax, scale.t())
    assert torch.equal(nf4.nf4_dequantize(codes, absmax), w)


def test_kernel_code_table_is_nf4_code():
    src = (REPO / 'distllm_b200' / 'csrc' / 'gemm.cuh').read_text()
    body = re.search(r'kNf4CodeBits\[16\] = \{([^}]*)\}', src).group(1)
    got = [int(x, 16) for x in re.findall(r'0x([0-9a-f]{8})u', body)]
    want = torch.tensor(nf4.NF4_CODE, dtype=torch.float32).view(torch.int32).tolist()
    assert got == [v & 0xFFFFFFFF for v in want]


# ------------------------------------------------------------------------------------------ assembled slots
def family_cases():
    from transformers import BertConfig
    from transformers import MistralConfig
    from transformers import ModernBertConfig
    from transformers import Qwen3Config

    return {
        'bert': (BertConfig(vocab_size=50, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                            intermediate_size=512, max_position_embeddings=32),
                 W.random_bert_state_dict, W.bert_weight_list),
        # intermediate 192 is padded to 256: zero rows of Wi, one zero k-block of mlp.Wo
        'modernbert': (ModernBertConfig(vocab_size=50, hidden_size=256, num_hidden_layers=3, num_attention_heads=4,
                                        intermediate_size=192, max_position_embeddings=64, local_attention=16,
                                        pad_token_id=0, bos_token_id=1, eos_token_id=2, cls_token_id=1,
                                        sep_token_id=2),
                       W.random_modernbert_state_dict, W.modernbert_weight_list),
        'mistral': (MistralConfig(vocab_size=50, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                                  num_key_value_heads=2, head_dim=128, intermediate_size=384,
                                  max_position_embeddings=64),
                    W.random_mistral_state_dict, W.mistral_weight_list),
        'qwen3': (Qwen3Config(vocab_size=50, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                              num_key_value_heads=2, head_dim=128, intermediate_size=384, max_position_embeddings=64),
                  W.random_qwen3_state_dict, W.qwen3_weight_list),
    }


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
@pytest.mark.parametrize('family', ['bert', 'modernbert', 'mistral', 'qwen3'])
def test_nf4_slots_dequantise_to_the_load_time_16bit_slots(family, dtype):
    cfg, make, build = family_cases()[family]
    cpu = torch.device('cpu')
    sd = make(cfg, seed=11, device='cpu')
    layers = cfg.num_hidden_layers
    ref = build(nf4.quantize_state_dict_nf4(sd), layers, cpu, dtype)
    got = build(sd, layers, cpu, dtype, matrix=W.nf4_matrix(cpu))
    assert len(got) == len(ref)
    slots = [i for i, t in enumerate(got) if isinstance(t, W.Nf4Matrix)]
    assert len(slots) == 4 * layers
    for i, (g, r) in enumerate(zip(got, ref)):
        if isinstance(g, W.Nf4Matrix):
            n, k = r.shape
            assert g.codes.shape == (n, k // 2) and g.absmax.shape == (k // 64, n), (family, i)
            assert g.codes.is_contiguous() and g.absmax.is_contiguous(), (family, i)
            assert torch.equal(bits(W.to_storage(nf4.nf4_dequantize(*g), cpu, dtype)), bits(r)), (family, i)
        else:
            assert g.dtype == r.dtype == torch.float32 and torch.equal(bits(g), bits(r)), (family, i)
    if family == 'modernbert':
        wi, wo = got[5 + 6], got[5 + 7]
        assert wi.codes.shape == (512, 128) and wo.codes.shape == (256, 128)
        assert (wo.codes[:, 96:] == W.NF4_ZERO).all() and not wo.absmax[3:].any()
        # input rows [192, 256) and gate rows [192, 256) are padding: the fourth 64-row block of each, interleaved
        # to rows [384, 448) and [448, 512)
        assert (wi.codes[384:] == W.NF4_ZERO).all() and not wi.absmax[:, 384:].any()
        assert (wi.codes[:384] != W.NF4_ZERO).any(dim=1).all()


def test_matrix_bytes_shrink_3_56x():
    cfg, make, build = family_cases()['mistral']
    sd = make(cfg, seed=1, device='cpu')
    cpu = torch.device('cpu')
    b16 = W.device_weight_bytes(build(sd, 2, cpu, torch.float16))
    q = W.device_weight_bytes(build(sd, 2, cpu, torch.float16, matrix=W.nf4_matrix(cpu)))
    assert q['other'] == b16['other']
    assert q['matrix'] <= 0.2813 * b16['matrix'] and q['matrix'] * 64 == b16['matrix'] * 18   # 0.5625 / 2 bytes


class _RecordingEncoder:
    """Stands in for the native encoder class (no GPU here): records what AutoEncoder hands it."""

    calls: list = []

    def __init__(self, hf_config, state_dict, nf4=False):
        type(self).calls.append((dict(state_dict), nf4))

    @classmethod
    def validate(cls, hf_config):
        pass


def _tiny_mistral_dir(tmp_path, intermediate):
    from transformers import MistralConfig
    from transformers import MistralModel

    from oracle.make_golden import TINY_MISTRAL
    from oracle.make_golden import write_tiny_mistral_checkpoint

    write_tiny_mistral_checkpoint(tmp_path / 'tok')
    cfg = MistralConfig(**{**TINY_MISTRAL, 'intermediate_size': intermediate})
    model = MistralModel(cfg)
    model.load_state_dict(W.random_mistral_state_dict(cfg, seed=3), strict=False)
    ckpt = tmp_path / f'ckpt{intermediate}'
    model.save_pretrained(ckpt)
    from transformers import AutoTokenizer

    AutoTokenizer.from_pretrained(tmp_path / 'tok').save_pretrained(ckpt)
    return ckpt


@pytest.mark.parametrize('intermediate, nf4_storage, want_nf4', [(768, True, True), (768, False, False),
                                                                 (704, True, True), (200, True, False)])
def test_auto_encoder_chooses_the_weight_storage(tmp_path, monkeypatch, intermediate, nf4_storage, want_nf4):
    """quantization=True: NF4 storage (the checkpoint's own matrices handed over, quantised by the encoder) when every
    quantised matrix is in 64-column blocks and nf4_storage is on; else the load-time round trip in 16 bits
    (down_proj with 200 input columns, or nf4_storage: False)."""
    from distllm_b200.embed.encoders import auto

    _RecordingEncoder.calls = []
    monkeypatch.setitem(auto._NATIVE_BY_MODEL_TYPE, 'mistral', _RecordingEncoder)
    ckpt = _tiny_mistral_dir(tmp_path, intermediate)
    auto.AutoEncoder(auto.AutoEncoderConfig(pretrained_model_name_or_path=str(ckpt), quantization=True,
                                            nf4_storage=nf4_storage))
    (sd, got_nf4), = _RecordingEncoder.calls
    assert got_nf4 is want_nf4
    key = 'layers.0.mlp.down_proj.weight'
    from transformers import MistralModel

    original = MistralModel.from_pretrained(ckpt).state_dict()[key]
    if want_nf4:
        assert torch.equal(sd[key], original)
    else:
        assert torch.equal(bits(sd[key].cpu()), bits(nf4.nf4_roundtrip(original)))
    auto.AutoEncoder(auto.AutoEncoderConfig(pretrained_model_name_or_path=str(ckpt), quantization=False))
    sd_off, nf4_off = _RecordingEncoder.calls[1]
    assert nf4_off is False and torch.equal(sd_off[key], original)
