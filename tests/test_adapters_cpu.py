"""PEFT adapter checkpoints on the CPU: resolution, key matching, refusals, scaling, the NF4 slot layout of the LoRA
factors, and the adapter oracle pinned against forward hooks on HF's own modules.

The encoders' wiring is checked with the native forward pass replaced by a recorder (the CPU has no device): what
reaches it -- the base config, the merged or unmerged weights, nf4 -- is what the GPU encoder would be built from.
"""

from __future__ import annotations

import json
import math

import pytest
import torch
from safetensors.torch import save_file

from distllm_b200.embed.encoders import adapters as ad
from distllm_b200.embed.encoders import nf4
from distllm_b200.embed.encoders import weights as W
from oracle import adapters as oad

BERT_Q = 'encoder.layer.{}.attention.self.query'
BERT_V = 'encoder.layer.{}.attention.self.value'


def lora_tensors(sd, modules, r, seed, scale_b=0.01, prefix='base_model.model.'):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for m in modules:
        o, i = sd[m + '.weight'].shape
        out[f'{prefix}{m}.lora_A.weight'] = torch.randn(r, i, generator=g) * 0.1
        out[f'{prefix}{m}.lora_B.weight'] = torch.randn(o, r, generator=g) * scale_b
    return out


def ia3_tensors(sd, modules, ff, seed):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for m in modules:
        o, i = sd[m + '.weight'].shape
        shape = (1, i) if m in ff else (o, 1)
        out[f'base_model.model.{m}.ia3_l'] = 1.0 + 0.3 * torch.randn(*shape, generator=g)
    return out


def lora_config(base, targets=('query', 'value'), **kw):
    cfg = {'peft_type': 'LORA', 'base_model_name_or_path': str(base), 'r': 8, 'lora_alpha': 16,
           'target_modules': list(targets), 'bias': 'none', 'modules_to_save': None, 'use_rslora': False,
           'use_dora': False, 'fan_in_fan_out': False, 'alpha_pattern': {}, 'rank_pattern': {}}
    cfg.update(kw)
    return cfg


def write_adapter(d, config, tensors, fmt='safetensors'):
    d.mkdir(parents=True, exist_ok=True)
    (d / ad.ADAPTER_CONFIG).write_text(json.dumps(config))
    if fmt == 'safetensors':
        save_file({k: v.contiguous() for k, v in tensors.items()}, str(d / 'adapter_model.safetensors'))
    else:
        torch.save(tensors, d / 'adapter_model.bin')
    return d


@pytest.fixture(scope='module')
def bert_ckpt(tmp_path_factory):
    from oracle.make_golden import write_tiny_bert_checkpoint

    d = tmp_path_factory.mktemp('bert') / 'ckpt'
    write_tiny_bert_checkpoint(d)
    return d


def bert_sd(path):
    from transformers import AutoModel

    return AutoModel.from_pretrained(path).state_dict()


# ------------------------------------------------------------------------------------------- resolution
def test_adapter_only_directory_resolves_to_its_base_and_the_base_tokenizer(bert_ckpt, tmp_path):
    sd = bert_sd(bert_ckpt)
    d = write_adapter(tmp_path / 'lora', lora_config(bert_ckpt), lora_tensors(sd, [BERT_Q.format(0)], 8, 1))
    assert ad.resolve(d) == (str(bert_ckpt), d)
    assert ad.tokenizer_source(None, d, str(bert_ckpt)) == str(bert_ckpt)
    assert ad.tokenizer_source('tok-name', d, str(bert_ckpt)) == 'tok-name'
    (d / 'tokenizer_config.json').write_text('{}')
    assert ad.tokenizer_source(None, d, str(bert_ckpt)) == str(d)


def test_a_directory_with_config_json_is_a_full_checkpoint(bert_ckpt, tmp_path):
    d = write_adapter(tmp_path / 'both', lora_config(bert_ckpt), {})
    (d / 'config.json').write_text((bert_ckpt / 'config.json').read_text())
    assert ad.resolve(d) == (str(d), None)
    assert ad.resolve(bert_ckpt) == (str(bert_ckpt), None)
    assert ad.tokenizer_source(None, d, str(d)) == str(d)


def test_missing_base_model_name_is_an_error(tmp_path):
    d = write_adapter(tmp_path / 'nobase', {'peft_type': 'LORA'}, {})
    with pytest.raises(ad.AdapterError, match='base_model_name_or_path'):
        ad.resolve(d)


def test_bin_and_safetensors_forms_load_the_same_adapter(bert_ckpt, tmp_path):
    sd = bert_sd(bert_ckpt)
    t = lora_tensors(sd, [BERT_Q.format(0), BERT_V.format(1)], 8, 2)
    a = ad.load_adapter(write_adapter(tmp_path / 'st', lora_config(bert_ckpt), t), sd)
    b = ad.load_adapter(write_adapter(tmp_path / 'bin', lora_config(bert_ckpt), t, fmt='bin'), sd)
    assert sorted(a.lora) == sorted(b.lora) == [BERT_Q.format(0), BERT_V.format(1)]
    for m in a.lora:
        assert torch.equal(a.lora[m][0], b.lora[m][0]) and torch.equal(a.lora[m][1], b.lora[m][1])
        assert a.lora[m][2] == b.lora[m][2] == 2.0


# ------------------------------------------------------------------------------------------- keys and refusals
def test_keys_strip_the_peft_prefix_and_pooler_tensors_are_ignored(bert_ckpt):
    sd = bert_sd(bert_ckpt)
    t = lora_tensors(sd, [BERT_Q.format(0), 'pooler.dense'], 4, 3)
    a = ad.match_adapter(lora_config(bert_ckpt), t, sd)
    assert list(a.lora) == [BERT_Q.format(0)] and a.ignored == ['pooler.dense']


def test_keys_of_another_model_class_are_an_error_naming_them(bert_ckpt):
    sd = bert_sd(bert_ckpt)
    t = lora_tensors(sd, [BERT_Q.format(0)], 4, 3, prefix='base_model.model.bert.')
    with pytest.raises(ad.AdapterError, match=r'match no transformer-block linear layer.*bert\.encoder\.layer\.0'):
        ad.match_adapter(lora_config(bert_ckpt), t, sd)
    with pytest.raises(ad.AdapterError, match='embeddings.LayerNorm.lora_A'):
        ad.match_adapter(lora_config(bert_ckpt), {'base_model.model.embeddings.LayerNorm.lora_A.weight':
                                                  torch.zeros(4, 64)}, sd)


@pytest.mark.parametrize('field, value, message', [
    ('peft_type', 'PREFIX_TUNING', 'peft_type'),
    ('use_dora', True, 'use_dora'),
    ('alpha_pattern', {'query': 32}, 'alpha_pattern'),
    ('modules_to_save', ['classifier'], 'modules_to_save'),
    ('bias', 'all', 'bias'),
    ('lora_bias', True, 'lora_bias'),
    ('fan_in_fan_out', True, 'fan_in_fan_out'),
])
def test_refused_config_fields_are_named(bert_ckpt, field, value, message):
    sd = bert_sd(bert_ckpt)
    cfg = lora_config(bert_ckpt, **{field: value})
    with pytest.raises(ad.AdapterError, match=message):
        ad.match_adapter(cfg, lora_tensors(sd, [BERT_Q.format(0)], 4, 3), sd)


def test_embedding_lora_and_lora_bias_tensors_are_refused(bert_ckpt):
    sd = bert_sd(bert_ckpt)
    t = {'base_model.model.embeddings.word_embeddings.lora_embedding_A': torch.zeros(4, 10)}
    with pytest.raises(ad.AdapterError, match='LoRA on embeddings'):
        ad.match_adapter(lora_config(bert_ckpt), t, sd)
    t = lora_tensors(sd, [BERT_Q.format(0)], 4, 3)
    t[f'base_model.model.{BERT_Q.format(0)}.lora_B.bias'] = torch.zeros(sd[BERT_Q.format(0) + '.weight'].shape[0])
    with pytest.raises(ad.AdapterError, match='lora_bias'):
        ad.match_adapter(lora_config(bert_ckpt), t, sd)


def test_ia3_feedforward_detection_by_shape_on_berts_two_output_dense(bert_ckpt):
    """peft's default BERT targets (key, value, output.dense) with feedforward_modules output.dense: the attention
    output's output.dense is (out, 1), the FFN down projection's (1, in) -- the name matches both."""
    sd = bert_sd(bert_ckpt)
    mods = ['encoder.layer.0.attention.output.dense', 'encoder.layer.0.output.dense']
    t = ia3_tensors(sd, mods, ff={'encoder.layer.0.output.dense'}, seed=4)
    cfg = {'peft_type': 'IA3', 'base_model_name_or_path': str(bert_ckpt), 'target_modules': ['key', 'value',
           'output.dense'], 'feedforward_modules': ['output.dense'], 'modules_to_save': None, 'fan_in_fan_out': False}
    a = ad.match_adapter(cfg, t, sd)
    assert a.ia3[mods[0]][1] is False and a.ia3[mods[1]][1] is True
    merged = ad.merge_adapter(sd, a)
    l0, l1 = a.ia3[mods[0]][0], a.ia3[mods[1]][0]
    assert torch.equal(merged[mods[0] + '.weight'], sd[mods[0] + '.weight'] * l0[:, None])
    assert torch.equal(merged[mods[0] + '.bias'], sd[mods[0] + '.bias'] * l0)
    assert torch.equal(merged[mods[1] + '.weight'], sd[mods[1] + '.weight'] * l1[None, :])
    assert torch.equal(merged[mods[1] + '.bias'], sd[mods[1] + '.bias'])
    bad = {f'base_model.model.{mods[0]}.ia3_l': torch.ones(3, 1)}
    with pytest.raises(ad.AdapterError, match='neither'):
        ad.match_adapter(cfg, bad, sd)


def test_rslora_scaling_and_rank_from_the_shapes(bert_ckpt):
    sd = bert_sd(bert_ckpt)
    t = {**lora_tensors(sd, [BERT_Q.format(0)], 16, 5), **lora_tensors(sd, [BERT_V.format(0)], 4, 6)}
    a = ad.match_adapter(lora_config(bert_ckpt, lora_alpha=32, use_rslora=True), t, sd)
    assert a.lora[BERT_Q.format(0)][2] == 32 / math.sqrt(16) and a.lora[BERT_V.format(0)][2] == 32 / math.sqrt(4)
    a = ad.match_adapter(lora_config(bert_ckpt, lora_alpha=32), t, sd)
    assert a.lora[BERT_Q.format(0)][2] == 2.0 and a.lora[BERT_V.format(0)][2] == 8.0
    merged = ad.merge_adapter(sd, a)
    ref = oad.adapted_state_dict(sd, t, lora_config(bert_ckpt, lora_alpha=32))
    for m in a.lora:
        torch.testing.assert_close(merged[m + '.weight'], ref[m + '.weight'], rtol=0, atol=1e-7)


# ------------------------------------------------------------------------------------------- encoder wiring
class _Recorder:
    built: list = []

    def __init__(self, hf_config, state_dict, nf4=False, lora=None):
        self.hf_config, self.state_dict, self.nf4, self.lora = hf_config, state_dict, nf4, lora
        self.hidden_size = hf_config.hidden_size
        _Recorder.built.append(self)

    @classmethod
    def validate(cls, hf_config):
        pass


@pytest.mark.parametrize('quantization, nf4_storage, kind', [
    (False, True, 'LORA'), (True, False, 'LORA'), (True, True, 'LORA'), (False, True, 'IA3'), (True, True, 'IA3')])
def test_auto_encoder_builds_the_adapted_model_of_each_weight_path(bert_ckpt, tmp_path, monkeypatch, quantization,
                                                                  nf4_storage, kind):
    from distllm_b200.embed.encoders import auto

    monkeypatch.setitem(auto._NATIVE_BY_MODEL_TYPE, 'bert', _Recorder)
    sd = bert_sd(bert_ckpt)
    if kind == 'LORA':
        cfg, t = lora_config(bert_ckpt), lora_tensors(sd, [BERT_Q.format(0), BERT_V.format(1), 'pooler.dense'], 8, 7)
    else:
        mods = ['encoder.layer.1.attention.self.key', 'encoder.layer.1.output.dense']
        cfg = {'peft_type': 'IA3', 'base_model_name_or_path': str(bert_ckpt)}
        t = ia3_tensors(sd, mods, ff={mods[1]}, seed=8)
    d = write_adapter(tmp_path / 'adapter', cfg, t)
    _Recorder.built.clear()
    enc = auto.AutoEncoder(auto.AutoEncoderConfig(pretrained_model_name_or_path=str(d), quantization=quantization,
                                                  nf4_storage=nf4_storage))
    rec = _Recorder.built[-1]
    assert enc.tokenizer.name_or_path == str(bert_ckpt)
    assert enc.adapter_ignored == (['pooler.dense'] if kind == 'LORA' else [])
    base = nf4.quantize_state_dict_nf4(sd) if quantization and not rec.nf4 else sd
    ref = oad.adapted_state_dict(base, t, cfg)
    if quantization and nf4_storage and kind == 'LORA':
        assert rec.nf4 and sorted(rec.lora) == [BERT_Q.format(0), BERT_V.format(1)]
        assert all(torch.equal(rec.state_dict[k], sd[k]) for k in sd)
    else:
        assert not rec.nf4 and not rec.lora
        for k in ref:
            if k in rec.state_dict and not k.startswith('pooler'):
                torch.testing.assert_close(rec.state_dict[k].float().cpu(), ref[k], rtol=0, atol=1e-6, msg=k)


# ------------------------------------------------------------------------------------------- NF4 slot layout
def _family_case(family):
    from transformers import BertConfig
    from transformers import MistralConfig
    from transformers import ModernBertConfig
    from transformers import Qwen3Config

    if family == 'bert':
        cfg = BertConfig(vocab_size=50, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                         intermediate_size=256, max_position_embeddings=32)
        return cfg, W.random_bert_state_dict(cfg, seed=1), W.bert_weight_list, (5, 12, (0, 2, 6, 8)), \
            [BERT_Q.format(0), BERT_V.format(0), BERT_V.format(1), 'encoder.layer.1.output.dense']
    if family in ('mistral', 'qwen3'):
        cls = MistralConfig if family == 'mistral' else Qwen3Config
        cfg = cls(vocab_size=50, hidden_size=256, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1,
                  head_dim=128, intermediate_size=384, max_position_embeddings=32)
        make = W.random_mistral_state_dict if family == 'mistral' else W.random_qwen3_state_dict
        wl = W.mistral_weight_list if family == 'mistral' else W.qwen3_weight_list
        mods = [f'layers.0.self_attn.{n}_proj' for n in ('q', 'v')]
        mods += [f'layers.1.{n}' for n in ('self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj',
                                           'self_attn.o_proj', 'mlp.gate_proj', 'mlp.up_proj', 'mlp.down_proj')]
        return cfg, make(cfg, seed=2), wl, (2, 6 if family == 'mistral' else 8, (1, 2, 4, 5)), mods
    cfg = ModernBertConfig(vocab_size=50, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                           intermediate_size=192, max_position_embeddings=64, local_attention=16, pad_token_id=0,
                           bos_token_id=1, eos_token_id=2, cls_token_id=1, sep_token_id=2)
    mods = [f'layers.{l}.{n}' for l in (0, 1) for n in ('attn.Wqkv', 'attn.Wo', 'mlp.Wi', 'mlp.Wo')]
    return cfg, W.random_modernbert_state_dict(cfg, seed=3), W.modernbert_weight_list, (5, 8, (2, 3, 6, 7)), mods


@pytest.mark.parametrize('family', ['bert', 'mistral', 'qwen3', 'modernbert'])
def test_lora_slot_factors_multiply_to_the_merged_slot_delta(family):
    """B_cat . A_cat of every slot equals, in fp32, the slot the weight builder makes from the merged delta (a zero
    base plus s B A): Q|K|V with some of them adapted, the gate/up interleave, ModernBERT's padded Wi and mlp.Wo."""
    cfg, sd, weight_list, (lead, stride, offsets), mods = _family_case(family)
    t = lora_tensors(sd, mods, 8, 11, scale_b=0.05)
    for i, m in enumerate(mods[:2]):   # two ranks in one slot
        t.update(lora_tensors(sd, [m], 16 + 8 * i, 12 + i, scale_b=0.05))
    adapter = ad.match_adapter(lora_config('base', lora_alpha=24), t, sd)
    zero = {k: torch.zeros_like(v) for k, v in sd.items()}
    delta = weight_list(ad.merge_adapter(zero, adapter), cfg.num_hidden_layers, torch.device('cpu'), torch.float32)
    factors = W.lora_slot_factors(family, cfg, adapter.lora, torch.device('cpu'), torch.float32)
    assert len(factors) == 4 * cfg.num_hidden_layers
    for layer in range(cfg.num_hidden_layers):
        for j, off in enumerate(offsets):
            slot = delta[lead + stride * layer + off]
            f = factors[4 * layer + j]
            if f is None:
                assert not slot.abs().any(), (layer, j)
                continue
            a_cat, b_cat, r = f
            assert r % 64 == 0 and a_cat.shape[0] == (r + 127) // 128 * 128 and b_cat.shape == (slot.shape[0], r)
            assert a_cat.shape[1] == slot.shape[1] and not a_cat[r:].any()
            torch.testing.assert_close(b_cat @ a_cat[:r], slot, rtol=1e-5, atol=1e-6, msg=f'{family} {layer} {j}')


# ------------------------------------------------------------------------------------------- the oracle vs HF hooks
def _hooked(model, tensors, config):
    keys = {k.removeprefix('base_model.model.'): v for k, v in tensors.items()}
    handles = []
    for name, mod in model.named_modules():
        if name + '.lora_A.weight' in keys:
            a, b = keys[name + '.lora_A.weight'], keys[name + '.lora_B.weight']
            s = config['lora_alpha'] / a.shape[0]
            handles.append(mod.register_forward_hook(
                lambda m, inp, out, a=a, b=b, s=s: out + s * (inp[0] @ a.t() @ b.t())))
        elif name + '.ia3_l' in keys:
            l = keys[name + '.ia3_l']
            if l.shape[0] == 1:
                handles.append(mod.register_forward_pre_hook(lambda m, inp, l=l: (inp[0] * l.flatten(),)))
            else:
                handles.append(mod.register_forward_hook(lambda m, inp, out, l=l: out * l.flatten()))
    return handles


@pytest.mark.parametrize('family, kind', [('bert', 'LORA'), ('bert', 'IA3'), ('mistral', 'LORA')])
def test_adapter_oracle_matches_hf_modules_with_forward_hooks(family, kind):
    from transformers import BertConfig
    from transformers import BertModel
    from transformers import MistralConfig
    from transformers import MistralModel

    from oracle import bert as obert
    from oracle import mistral as omistral

    torch.manual_seed(0)
    if family == 'bert':
        cfg = BertConfig(vocab_size=60, hidden_size=64, num_hidden_layers=2, num_attention_heads=2,
                         intermediate_size=128, max_position_embeddings=32, attn_implementation='eager')
        model = BertModel(cfg, add_pooling_layer=False).eval()
        forward = obert.bert_forward
        lin = ['attention.self.query', 'attention.self.value', 'attention.self.key', 'attention.output.dense',
               'output.dense']
        mods = [f'encoder.layer.{l}.{n}' for l in (0, 1) for n in lin]
    else:
        cfg = MistralConfig(vocab_size=60, hidden_size=64, num_hidden_layers=2, num_attention_heads=2,
                            num_key_value_heads=1, head_dim=32, intermediate_size=128, max_position_embeddings=32,
                            attn_implementation='eager')
        model = MistralModel(cfg).eval()
        forward = omistral.mistral_forward
        mods = [f'layers.{l}.{n}' for l in (0, 1) for n in ('self_attn.q_proj', 'self_attn.v_proj', 'self_attn.o_proj',
                                                             'mlp.gate_proj', 'mlp.up_proj', 'mlp.down_proj')]
    sd = model.state_dict()
    g = torch.Generator().manual_seed(3)
    for k in sd:
        if k.endswith('.bias'):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.1
    model.load_state_dict(sd)
    if kind == 'LORA':
        config = {'peft_type': 'LORA', 'lora_alpha': 16}
        tensors = lora_tensors(sd, mods, 8, 21, scale_b=0.05)
    else:
        config = {'peft_type': 'IA3'}
        tensors = ia3_tensors(sd, mods, ff={m for m in mods if m.endswith('layer.0.output.dense')
                                            or m.endswith('layer.1.output.dense')}, seed=22)
    ids = torch.randint(3, 60, (3, 17), generator=g)
    mask = torch.ones_like(ids)
    mask[1, 11:] = 0
    mask[2, 5:] = 0
    handles = _hooked(model, tensors, config)
    with torch.no_grad():
        ref = model(input_ids=ids, attention_mask=mask).last_hidden_state
    for h in handles:
        h.remove()
    with torch.no_grad():
        base = model(input_ids=ids, attention_mask=mask).last_hidden_state
    got = forward(oad.adapted_state_dict(sd, tensors, config), cfg, ids, mask)
    live = mask.bool()
    assert (got - ref)[live].abs().max() <= 5e-5
    assert (base - ref)[live].abs().max() > 1e-2   # the adapter changes the model


def test_create_nf4_lora_refuses_a_negative_rank_even_beside_a_null_factor():
    """Rank 0 or a NULL factor means 'no adapter on this slot'; a negative rank is an error either way, reported before
    any device is touched."""
    import ctypes as C

    from transformers import BertConfig

    from distllm_b200 import _native as nv

    lib = nv.load()
    cfg = BertConfig(vocab_size=50, hidden_size=256, num_hidden_layers=1, num_attention_heads=4,
                     intermediate_size=512, max_position_embeddings=32)
    desc = W.bert_desc(cfg)
    n = lib.b2e_num_weights(C.byref(desc))
    weights = (C.c_void_p * n)(*([16] * n))
    scales = (C.c_void_p * 4)(*([16] * 4))
    a_ptrs = (C.c_void_p * 4)(None, 16, 16, 16)
    b_ptrs = (C.c_void_p * 4)(None, 16, 16, 16)
    handle = C.c_void_p()
    for ranks, slot in (((-64, 0, 0, 0), 0), ((0, 96, 0, 0), 1)):
        rc = lib.b2e_encoder_create_nf4_lora(C.byref(desc), weights, n, scales, 4, a_ptrs, b_ptrs,
                                             (C.c_int * 4)(*ranks), 4, 0, C.byref(handle))
        assert rc != 0 and not handle.value
        assert f'LoRA slot {slot}: rank' in lib.b2e_last_error().decode()
