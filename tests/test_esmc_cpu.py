"""ESM C without a device: the config and tokenizer against the reference's behaviour, shape inference and the
checkpoint rejections, b2e_check_model / b2e_num_weights for the published shapes in both builds, the weight order and
the residual-scale fold, and the fp32 restatement (tools/oracle_esmc.py) against an nn.Module transcription of the
checkpoint's key table loaded with ``strict=True``."""

from __future__ import annotations

import ctypes as C
import math

import pytest
import torch
from torch import nn

from distllm_b200 import _native
from distllm_b200.embed.encoders import weights as W
from tools import oracle_esmc as O

ESM2_VOCAB = ['<cls>', '<pad>', '<eos>', '<unk>', 'L', 'A', 'G', 'V', 'S', 'E', 'R', 'T', 'I', 'D', 'P', 'K', 'Q',
              'N', 'F', 'Y', 'M', 'H', 'W', 'C', 'X', 'B', 'U', 'Z', 'O', '.', '-', '<null_1>', '<mask>']


def test_config_matches_the_reference():
    from distllm_b200.embed.encoders.esmc import EsmCambrianEncoderConfig

    assert EsmCambrianEncoderConfig().embedding_size == 960
    assert EsmCambrianEncoderConfig(
        pretrained_model_name_or_path='EvolutionaryScale/esmc-600m-2024-12').embedding_size == 1152
    assert EsmCambrianEncoderConfig(pretrained_model_name_or_path='/some/dir', embedding_size=960).embedding_size == 960
    with pytest.raises(ValueError, match='Invalid model name for ESMC: /some/dir Valid model names are: '
                                         'EvolutionaryScale/esmc-300m-2024-12, EvolutionaryScale/esmc-600m-2024-12'):
        EsmCambrianEncoderConfig(pretrained_model_name_or_path='/some/dir')


def test_yaml_name_esmc_validates_through_the_worker_config(tmp_path):
    from distllm_b200.distributed_embedding import Config
    from distllm_b200.embed.encoders import STRATEGIES
    from distllm_b200.embed.encoders.esmc import EsmCambrianEncoderConfig

    assert STRATEGIES['esmc'][0] is EsmCambrianEncoderConfig
    (tmp_path / 'in').mkdir()
    (tmp_path / 'cfg.yaml').write_text(f"""
input_dir: {tmp_path / 'in'}
output_dir: {tmp_path / 'out'}
glob_patterns: ['*.fasta']
dataset_config:
  name: fasta
  batch_size: 8
encoder_config:
  name: esmc
  pretrained_model_name_or_path: EvolutionaryScale/esmc-600m-2024-12
pooler_config:
  name: mean
embedder_config:
  name: full_sequence
writer_config:
  name: numpy
""")
    cfg = Config.from_yaml(tmp_path / 'cfg.yaml')
    assert isinstance(cfg.encoder_config, EsmCambrianEncoderConfig)
    assert cfg.encoder_config.embedding_size == 1152


def test_tokenizer_matches_esm2_ids(tmp_path):
    from transformers import EsmTokenizer

    from distllm_b200.embed.encoders.esmc import esmc_tokenizer

    (tmp_path / 'vocab.txt').write_text('\n'.join(ESM2_VOCAB) + '\n')
    esm2 = EsmTokenizer(str(tmp_path / 'vocab.txt'))
    tok = esmc_tokenizer()
    seqs = ['MKTAYIAKQRQISFVKSHFSRQ', 'XBUZO.-', 'A', 'LAGVSERTIDPKQNFYMHWCXBUZO.-']
    for s in seqs:
        assert tok(s)['input_ids'] == esm2(s)['input_ids'], s
    assert tok('A|G')['input_ids'] == [0, 5, 31, 6, 2]
    assert tok('A<mask>G')['input_ids'] == [0, 5, 32, 6, 2]
    assert tok('AJ')['input_ids'] == [0, 5, 3, 2]          # unknown character -> <unk>
    batch = tok(seqs, padding=True, return_tensors='pt')
    assert batch['input_ids'][2].tolist() == [0, 5, 2] + [1] * (batch['input_ids'].shape[1] - 3)
    assert torch.equal(batch['attention_mask'], (batch['input_ids'] != 1).long())
    assert tok.model_max_length == 2048
    long = tok(['A' * 3000], truncation=True)['input_ids'][0]
    assert len(long) == 2048 and long[0] == 0 and long[-1] == 2


def tiny_sd(h=960, layers=2, inter=256, seed=0):
    return W.random_esmc_state_dict(h, layers, inter, seed=seed)


def test_shape_inference_and_rejections():
    sd = tiny_sd()
    cfg = W.esmc_config(sd)
    assert cfg == W.EsmcConfig(hidden_size=960, num_hidden_layers=2, intermediate_size=256, vocab_size=64)
    d = W.esmc_desc(cfg)
    assert (d.arch, d.heads, d.head_dim, d.max_pos, d.eps) == (_native.ARCH_ESMC, 15, 64, 2048, pytest.approx(1e-5))
    bad = dict(sd, **{'transformer.blocks.0.attn.out_proj.bias': torch.zeros(960)})
    with pytest.raises(ValueError, match=r"unexpected keys \['transformer.blocks.0.attn.out_proj.bias'\]"):
        W.esmc_config(bad)
    bad = dict(sd, **{'transformer.blocks.1.attn.q_ln.weight': torch.ones(64)})
    with pytest.raises(ValueError, match=r'transformer.blocks.1.attn.q_ln.weight has shape \[64\], expected \[960\]'):
        W.esmc_config(bad)
    lib = _native.load()
    d = W.esmc_desc(W.esmc_config(tiny_sd(h=1024)))
    assert lib.b2e_check_model(C.byref(d)) == 3
    assert b'ESMC: hidden size 1024 not built (built: 960, 1152)' in lib.b2e_last_error()


def test_embedding_size_mismatch_is_an_error(tmp_path):
    from distllm_b200.embed.encoders.esmc import EsmCambrianEncoder
    from distllm_b200.embed.encoders.esmc import EsmCambrianEncoderConfig

    path = tmp_path / 'data' / 'weights' / 'esmc_300m_2024_12_v0.pth'
    path.parent.mkdir(parents=True)
    torch.save(tiny_sd(), path)
    with pytest.raises(ValueError, match='embedding_size 1152 disagrees'):
        EsmCambrianEncoder(EsmCambrianEncoderConfig(pretrained_model_name_or_path=str(tmp_path), embedding_size=1152))


def esmc_desc(h, layers, inter):
    return W.esmc_desc(W.EsmcConfig(hidden_size=h, num_hidden_layers=layers, intermediate_size=inter, vocab_size=64))


@pytest.mark.parametrize('storage', ['f16', 'bf16'])
def test_check_model_accepts_the_published_shapes(storage):
    lib = _native.load(storage)
    for h, layers, inter in ((960, 30, 2560), (1152, 36, 3072)):
        d = esmc_desc(h, layers, inter)
        assert lib.b2e_check_model(C.byref(d)) == 0, lib.b2e_last_error()
        assert lib.b2e_num_weights(C.byref(d)) == 3 + 10 * layers
    # NF4 weights are refused when the handle is created (before any device is touched)
    d = esmc_desc(960, 2, 2560)
    n = lib.b2e_num_weights(C.byref(d))
    ptrs, scales = (C.c_void_p * n)(*([16] * n)), (C.c_void_p * 8)(*([16] * 8))
    lib.b2e_encoder_create_nf4.argtypes = [C.POINTER(_native.ModelDesc), C.POINTER(C.c_void_p), C.c_int,
                                           C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    handle = C.c_void_p()
    assert lib.b2e_encoder_create_nf4(C.byref(d), ptrs, n, scales, 8, 0, C.byref(handle)) == 3
    assert b'ESMC: NF4 weights are not built' in lib.b2e_last_error() and not handle.value
    d = esmc_desc(960, 2, 2560 + 64)
    assert lib.b2e_check_model(C.byref(d)) == 3 and b'ESMC: intermediate size 2624' in lib.b2e_last_error()
    d.intermediate, d.heads = 2560, 16
    assert lib.b2e_check_model(C.byref(d)) == 3 and b'ESMC: need head_dim 64' in lib.b2e_last_error()


def test_weight_order_and_residual_scale_fold():
    layers = 2
    sd = tiny_sd(layers=layers, seed=3)
    w = W.esmc_weight_list(sd, layers, torch.device('cpu'), torch.float16)
    s = math.sqrt(layers / 36)
    assert len(w) == 3 + 10 * layers
    assert torch.equal(w[0], sd['embed.weight']) and torch.equal(w[1], sd['transformer.norm.weight'])
    assert not w[2].any()
    p = 'transformer.blocks.1.'
    base = 3 + 10
    assert torch.equal(w[base + 0], sd[p + 'attn.layernorm_qkv.0.weight'])
    assert torch.equal(w[base + 1], sd[p + 'attn.layernorm_qkv.0.bias'])
    assert torch.equal(w[base + 2], sd[p + 'attn.layernorm_qkv.1.weight'].half())
    assert torch.equal(w[base + 3], sd[p + 'attn.q_ln.weight'])
    assert torch.equal(w[base + 4], sd[p + 'attn.k_ln.weight'])
    assert torch.equal(w[base + 5], (sd[p + 'attn.out_proj.weight'] / s).half())     # folded in fp32, rounded once
    assert torch.equal(w[base + 6], sd[p + 'ffn.0.weight']) and torch.equal(w[base + 7], sd[p + 'ffn.0.bias'])
    w1 = sd[p + 'ffn.1.weight'].half()
    assert torch.equal(w[base + 8], W.interleave_gate_up(w1[:256], w1[256:]))
    assert torch.equal(w[base + 9], (sd[p + 'ffn.3.weight'] / s).half())
    # s = 1 at 36 layers: the weights go through untouched
    assert W.esmc_residual_scale(36) == 1.0


# ------------------------------------------------------------------------------ nn.Module transcription
class Attn(nn.Module):
    def __init__(self, h):
        super().__init__()
        self.layernorm_qkv = nn.Sequential(nn.LayerNorm(h), nn.Linear(h, 3 * h, bias=False))
        self.q_ln = nn.LayerNorm(h, bias=False)
        self.k_ln = nn.LayerNorm(h, bias=False)
        self.out_proj = nn.Linear(h, h, bias=False)


class SwiGLU(nn.Module):
    def forward(self, x):
        a, b = x.chunk(2, dim=-1)
        return nn.functional.silu(a) * b


class Block(nn.Module):
    def __init__(self, h, i):
        super().__init__()
        self.attn = Attn(h)
        self.ffn = nn.Sequential(nn.LayerNorm(h), nn.Linear(h, 2 * i, bias=False), SwiGLU(),
                                 nn.Linear(i, h, bias=False))


class Stack(nn.Module):
    def __init__(self, h, i, layers):
        super().__init__()
        self.blocks = nn.ModuleList([Block(h, i) for _ in range(layers)])
        self.norm = nn.LayerNorm(h, bias=False)


class Esmc(nn.Module):
    """The checkpoint's key table as modules (sequence_head left out: the forward pass never reads it)."""

    def __init__(self, h, i, layers, vocab=64):
        super().__init__()
        self.embed = nn.Embedding(vocab, h)
        self.transformer = Stack(h, i, layers)
        self.h, self.layers = h, layers

    def forward(self, ids):
        pad = ids != 1      # ESMC.forward: sequence_id = input_ids != <pad>
        x = self.embed(ids)
        b, s, h = x.shape
        # rotary written out here, independently of the oracle: halves convention, base 10000, positions 0..s-1
        inv = 1.0 / 10000 ** (torch.arange(0, 64, 2, dtype=torch.float32) / 64)
        ang = torch.arange(s, dtype=torch.float32)[:, None] * inv[None]
        cos, sin = ang.cos()[None, :, None, :], ang.sin()[None, :, None, :]

        def rot(t):
            t1, t2 = t[..., :32], t[..., 32:]
            return torch.cat([t1 * cos - t2 * sin, t2 * cos + t1 * sin], dim=-1)

        scale = math.sqrt(self.layers / 36)
        for blk in self.transformer.blocks:
            q, k, v = blk.attn.layernorm_qkv(x).chunk(3, dim=-1)
            q, k = blk.attn.q_ln(q), blk.attn.k_ln(k)
            q = rot(q.reshape(b, s, -1, 64)).transpose(1, 2)
            k = rot(k.reshape(b, s, -1, 64)).transpose(1, 2)
            v = v.reshape(b, s, -1, 64).transpose(1, 2)
            ctx = nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=pad[:, None, None, :])
            x = x + blk.attn.out_proj(ctx.transpose(1, 2).reshape(b, s, h)) / scale
            x = x + blk.ffn(x) / scale
        return self.transformer.norm(x)


@torch.no_grad()
def test_oracle_matches_module_transcription():
    h, i, layers = 960, 256, 2
    sd = tiny_sd(h, layers, i, seed=5)
    model = Esmc(h, i, layers)
    model.load_state_dict({k: v for k, v in sd.items() if not k.startswith('sequence_head.')}, strict=True)
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(4, 29, (3, 40), generator=g)
    ids[:, 0] = 0
    lens = torch.tensor([40, 17, 5])
    ids[torch.arange(3), lens - 1] = 2
    mask = (torch.arange(40)[None] < lens[:, None]).long()
    ids[mask == 0] = 1
    got = O.esmc_forward(sd, ids, mask)
    exp = model(ids)
    live = mask.bool()
    assert (got[live] - exp[live]).abs().max() <= 5e-5
