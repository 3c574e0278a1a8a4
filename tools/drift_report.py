"""Per-layer drift of the native forward pass against the fp32 CPU oracle (SURVEY 7 / VERDICT r1 next #1 iv).

For each encoder family at its BASELINE shape, on N(0, 0.02) weights and on outlier weights
(tools/workloads.add_outliers), the model is run truncated to l = 1..L layers (b2e_debug_set_layers) and every
attended token's hidden state is compared with the oracle's state at the same depth: min / mean cosine per
depth, plus the pooled embedding's cosine at full depth.  Writes a markdown table per case.

usage: drift_report.py [out.md] [families: bert,esm,mistral,qwen3,esmc]
"""
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from distllm_b200 import _native as nv  # noqa: E402
from oracle import pooling as opool  # noqa: E402
from tools.workloads import add_outliers  # noqa: E402


def cos_rows(a, b):
    a = a.astype(np.float64)
    b = b.astype(np.float64)
    return (a * b).sum(-1) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))


def set_layers(enc, n):
    lib = getattr(enc, '_lib', None) or nv.load()
    lib.b2e_debug_set_layers.argtypes = [type(enc._handle), __import__('ctypes').c_int]
    nv.check(lib.b2e_debug_set_layers(enc._handle, n))


def report(name, enc, ids, mask, types, ref_states, ref_pool, pool_kind, lines):
    valid = mask.bool().numpy()
    lines.append(f'\n### {name}\n')
    lines.append('| layers | min token cosine | mean token cosine | 1 - min |')
    lines.append('|---|---|---|---|')
    L = len(ref_states)
    for n in range(1, L + 1):
        set_layers(enc, n)
        hidden = enc.encode(ids, mask, types).cpu().numpy()
        c = cos_rows(hidden[valid], ref_states[n - 1].numpy()[valid])
        lines.append(f'| {n} | {c.min():.6f} | {c.mean():.6f} | {1 - c.min():.2e} |')
    set_layers(enc, 0)
    got = enc.encode_pooled(ids, mask, types, pool_kind, False).cpu().numpy()
    live = np.linalg.norm(ref_pool, axis=-1) > 0
    c = cos_rows(got[live], ref_pool[live])
    lines.append(f'\npooled rows at full depth: min cosine {c.min():.6f} (1 - min = {1 - c.min():.2e}), '
                 f'tolerance 1e-3\n')
    print(name, 'pooled min cosine', c.min(), flush=True)


def run_bert(lines):
    from transformers import BertConfig

    from distllm_b200.embed.encoders.native import NativeBertEncoder
    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    from oracle import bert as obert

    cfg = BertConfig(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                     intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2,
                     layer_norm_eps=1e-12, initializer_range=0.02)
    g = torch.Generator().manual_seed(21)
    b, s = 8, 512
    ids = torch.randint(7, cfg.vocab_size, (b, s), generator=g)
    lens = torch.tensor([512, 300, 64, 511, 129, 2, 450, 257])
    mask = (torch.arange(s)[None] < lens[:, None]).long()
    for w in ('normal', 'outliers'):
        sd = random_bert_state_dict(cfg, seed=0, device='cpu')
        if w == 'outliers':
            add_outliers(sd, 'bert', seed=1)
        states = obert.bert_forward(sd, cfg, ids, mask, None, return_all=True)[1:]
        ref_pool = opool.average_pool(states[-1], mask.clone()).numpy()
        enc = NativeBertEncoder(cfg, sd)
        report(f'C2 BERT-base shape, 12 layers, S=512, ragged batch of 8, {w} weights (mean pooler)', enc, ids,
               mask, None, states, ref_pool, nv.POOL_MEAN_REF, lines)
        enc.close()


def run_esm(lines):
    from transformers import EsmConfig

    from distllm_b200.embed.encoders.native import NativeEsm2Encoder
    from distllm_b200.embed.encoders.weights import random_esm_state_dict
    from oracle import esm as oesm

    cfg = EsmConfig(vocab_size=33, hidden_size=1280, num_hidden_layers=33, num_attention_heads=20,
                    intermediate_size=5120, max_position_embeddings=1026, position_embedding_type='rotary',
                    token_dropout=True, mask_token_id=32, pad_token_id=1, layer_norm_eps=1e-5,
                    emb_layer_norm_before=False, initializer_range=0.02)
    g = torch.Generator().manual_seed(22)
    b, s = 2, 1026
    ids = torch.randint(4, 24, (b, s), generator=g)
    lens = torch.tensor([1026, 700])
    mask = (torch.arange(s)[None] < lens[:, None]).long()
    ids = ids.masked_fill(mask == 0, 1)
    ids[:, 0] = 0
    for w in ('normal', 'outliers'):
        sd = random_esm_state_dict(cfg, seed=3, device='cpu')
        if w == 'outliers':
            add_outliers(sd, 'esm', seed=2)
        states = oesm.esm_forward(sd, cfg, ids, mask, return_all=True)
        ref_pool = opool.average_pool(states[-1], mask.clone()).numpy()
        enc = NativeEsm2Encoder(cfg, sd)
        report(f'C5 ESM2-650M shape, 33 layers, S=1026, {w} weights (mean pooler)', enc, ids, mask, None, states,
               ref_pool, nv.POOL_MEAN_REF, lines)
        enc.close()


def run_mistral(lines):
    from transformers import MistralConfig

    from distllm_b200.embed.encoders.native import NativeMistralEncoder
    from distllm_b200.embed.encoders.weights import random_mistral_state_dict
    from oracle import mistral as omis

    cfg = MistralConfig(vocab_size=32000, hidden_size=4096, num_hidden_layers=32, num_attention_heads=32,
                        num_key_value_heads=8, head_dim=128, intermediate_size=14336,
                        max_position_embeddings=32768, rms_norm_eps=1e-5, sliding_window=4096,
                        initializer_range=0.02)
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(23)
    b, s = 2, 1024
    ids = torch.randint(3, cfg.vocab_size, (b, s), generator=g)
    lens = torch.tensor([1024, 700])
    mask = (torch.arange(s)[None] < lens[:, None]).long()
    for w in ('normal', 'outliers'):
        sd = random_mistral_state_dict(cfg, seed=5, device=dev, dtype=torch.float16)
        if w == 'outliers':
            add_outliers(sd, 'mistral', seed=3)
        t0 = time.time()
        states = omis.mistral_forward(sd, cfg, ids, mask, return_all=True)
        print(f'mistral oracle {time.time() - t0:.1f} s', flush=True)
        ref_pool = opool.last_token_pool(states[-1], mask).numpy()
        enc = NativeMistralEncoder(cfg, sd)
        del sd
        report(f'C3 Mistral-7B shape, 32 layers, S=1024 (rows of 1024 and 700 tokens), {w} weights '
               f'(last_token pooler)', enc, ids, mask, None, states, ref_pool, nv.POOL_LAST_TOKEN, lines)
        enc.close()
        del enc, states
        torch.cuda.empty_cache()


def run_qwen3(lines):
    """Qwen3-Embedding-8B shape (36 layers, H 4096, 32 / 8 heads x 128, I 12288) in BOTH storage builds: the
    measurement behind _native._STORAGE_BY_ARCH['qwen3']."""
    from transformers import Qwen3Config

    from distllm_b200.embed.encoders.native import NativeQwen3Encoder
    from distllm_b200.embed.encoders.weights import random_qwen3_state_dict
    from tools.oracle_qwen3 import qwen3_forward

    cfg = Qwen3Config(vocab_size=32000, hidden_size=4096, num_hidden_layers=36, num_attention_heads=32,
                      num_key_value_heads=8, head_dim=128, intermediate_size=12288, max_position_embeddings=32768,
                      rms_norm_eps=1e-6, rope_parameters={'rope_type': 'default', 'rope_theta': 1e6},
                      initializer_range=0.02, tie_word_embeddings=False)
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(24)
    b, s = 2, 1024
    ids = torch.randint(3, cfg.vocab_size, (b, s), generator=g)
    lens = torch.tensor([1024, 700])
    mask = (torch.arange(s)[None] < lens[:, None]).long()
    for w in ('normal', 'outliers'):
        sd = random_qwen3_state_dict(cfg, seed=6, device=dev, dtype=torch.float16)
        if w == 'outliers':
            add_outliers(sd, 'qwen3', seed=4)
        t0 = time.time()
        states = qwen3_forward(sd, cfg, ids, mask, return_all=True)
        print(f'qwen3 oracle {time.time() - t0:.1f} s', flush=True)
        ref_pool = opool.last_token_pool(states[-1], mask).numpy()
        for storage in ('f16', 'bf16'):
            enc = NativeQwen3Encoder(cfg, sd, storage=storage)
            report(f'Qwen3-Embedding-8B shape, 36 layers, S=1024 (rows of 1024 and 700 tokens), {w} weights, '
                   f'{storage} build (last_token pooler)', enc, ids, mask, None, states, ref_pool,
                   nv.POOL_LAST_TOKEN, lines)
            enc.close()
            del enc
            torch.cuda.empty_cache()
        del sd, states
        torch.cuda.empty_cache()


def run_esmc(lines):
    """esmc-600m shape (36 layers, H 1152, 18 heads x 64, I 3072) at S = 2048, the longest input the tokenizer
    allows, in BOTH storage builds: the measurement behind _native._STORAGE_BY_ARCH['esmc']."""
    from distllm_b200.embed.encoders import weights as W
    from distllm_b200.embed.encoders.native import NativeEsmcEncoder
    from tools.oracle_esmc import esmc_forward

    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(25)
    b, s = 2, 2048
    lens = torch.tensor([2048, 1400])
    ids = torch.randint(4, 24, (b, s), generator=g)
    ids[:, 0] = 0
    ids[torch.arange(b), lens - 1] = 2
    mask = (torch.arange(s)[None] < lens[:, None]).long()
    ids[mask == 0] = 1
    for w in ('normal', 'outliers'):
        sd = W.random_esmc_state_dict(1152, 36, 3072, seed=6, device=dev)
        if w == 'outliers':
            add_outliers(sd, 'esmc', seed=4)
        t0 = time.time()
        states = [t.cpu() for t in esmc_forward(sd, ids.to(dev), mask.to(dev), every_depth=True)]
        print(f'esmc oracle {time.time() - t0:.1f} s', flush=True)
        ref_pool = opool.average_pool(states[-1], mask.clone()).numpy()
        for storage in ('f16', 'bf16'):
            enc = NativeEsmcEncoder(W.esmc_config(sd), sd, device=dev, storage=storage)
            report(f'esmc-600m shape, 36 layers, S=2048 (rows of 2048 and 1400 tokens), {w} weights, {storage} build '
                   f'(mean pooler)', enc, ids, mask, None, states, ref_pool, nv.POOL_MEAN_REF, lines)
            enc.close()
            del enc
            torch.cuda.empty_cache()
        del sd, states
        torch.cuda.empty_cache()


if __name__ == '__main__':
    out = Path(sys.argv[1]) if len(sys.argv) > 1 else Path('gpurun_out/drift_report.md')
    fams = (sys.argv[2] if len(sys.argv) > 2 else 'bert,esm,mistral').split(',')
    lines = ['# Per-layer drift of the native forward pass vs the fp32 CPU oracle',
             '',
             'Model truncated to l layers on both sides (BERT: hidden_states[l]; ESM-2 / Mistral: final norm of the '
             'residual stream after l layers); cosine per attended token.  GEMMs multiply in bf16 with fp32 '
             'accumulation; norm statistics, softmax and pooling are fp32.']
    for fam, fn in (('bert', run_bert), ('esm', run_esm), ('mistral', run_mistral), ('qwen3', run_qwen3),
                    ('esmc', run_esmc)):
        if fam in fams:
            fn(lines)
            out.parent.mkdir(parents=True, exist_ok=True)
            out.write_text('\n'.join(lines) + '\n')
    print(out.read_text())
