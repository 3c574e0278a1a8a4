"""Throughput of the small encoders on the native path vs HuggingFace bf16 + SDPA on the same GPU.

Shapes (synthetic ids, every chunk S tokens long, seeded random weights of the real sizes):
  minilm     all-MiniLM-L6-v2           BERT, 6 layers, H = 384, 12 x 32, I = 1536   B = 512, S = 512
  bge-small  bge-small-en-v1.5 / e5-small-v2, the same at 12 layers                  B = 512, S = 512
  esm2-150m  esm2_t30_150M              ESM-2, 30 layers, H = 640, 20 x 32, I = 2560 B = 64, S = 1026

Per shape: chunks/s of encode_pooled (mean pooler) and of HF BertModel / EsmModel (bf16, attn_implementation='sdpa')
+ the same masked mean, three alternating runs each; the fraction of the 989 TFLOP/s dense BF16 data-sheet peak with
L (8 S H^2 + 4 S H I + 4 S^2 H) FLOPs per chunk; in a separate torch.profiler run the share of the native step's
device time spent in the head_dim-32 attention kernel.  The card's name and power limit are read in the same call.

    python tools/bench_small_encoders.py [--steps 10] [--warmup 3] [--out FILE.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

REPO = Path(__file__).resolve().parents[1]
if str(REPO) not in sys.path:
    sys.path.insert(0, str(REPO))

PEAK_BF16 = 989e12
SHAPES = {
    'minilm': dict(family='bert', layers=6, hidden=384, heads=12, inter=1536, B=512, S=512),
    'bge-small': dict(family='bert', layers=12, hidden=384, heads=12, inter=1536, B=512, S=512),
    'esm2-150m': dict(family='esm', layers=30, hidden=640, heads=20, inter=2560, B=64, S=1026),
}


def flops_per_chunk(sh: dict) -> float:
    L, S, H, I = sh['layers'], sh['S'], sh['hidden'], sh['inter']
    return L * (8 * S * H * H + 4 * S * H * I + 4 * S * S * H)


def build(sh: dict):
    from transformers import BertConfig
    from transformers import EsmConfig

    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    from distllm_b200.embed.encoders.weights import random_esm_state_dict

    if sh['family'] == 'bert':
        cfg = BertConfig(vocab_size=30522, hidden_size=sh['hidden'], num_hidden_layers=sh['layers'],
                         num_attention_heads=sh['heads'], intermediate_size=sh['inter'], max_position_embeddings=512,
                         initializer_range=0.02)
        return cfg, random_bert_state_dict(cfg, seed=0, device='cpu')
    cfg = EsmConfig(vocab_size=33, hidden_size=sh['hidden'], num_hidden_layers=sh['layers'],
                    num_attention_heads=sh['heads'], intermediate_size=sh['inter'], max_position_embeddings=1026,
                    position_embedding_type='rotary', token_dropout=True, mask_token_id=32, pad_token_id=1,
                    layer_norm_eps=1e-5, emb_layer_norm_before=False, initializer_range=0.02)
    return cfg, random_esm_state_dict(cfg, seed=0, device='cpu')


def timed(fn, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_small_encoders needs a CUDA device')
    from transformers import BertModel
    from transformers import EsmModel

    from distllm_b200 import _native as nv
    from distllm_b200.embed.encoders.native import NativeBertEncoder
    from distllm_b200.embed.encoders.native import NativeEsm2Encoder

    dev = torch.device('cuda:0')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True).stdout.strip()
    report = {'card': card, 'steps': args.steps, 'shapes': {}}
    for name in args.shapes.split(','):
        sh = SHAPES[name]
        cfg, sd = build(sh)
        B, S = sh['B'], sh['S']
        g = torch.Generator().manual_seed(1)
        lo, hi = (5, cfg.vocab_size) if sh['family'] == 'bert' else (4, 24)
        ids = torch.randint(lo, hi, (B, S), generator=g)
        if sh['family'] == 'esm':
            ids[:, 0] = 0
        mask = torch.ones(B, S, dtype=torch.int64)
        native = (NativeBertEncoder if sh['family'] == 'bert' else NativeEsm2Encoder)(cfg, sd)
        cfg._attn_implementation = 'sdpa'
        hf = (BertModel(cfg, add_pooling_layer=False) if sh['family'] == 'bert'
              else EsmModel(cfg, add_pooling_layer=False))
        hf.load_state_dict(sd, strict=False)
        hf = hf.to(dev, torch.bfloat16).eval()
        ids_d, mask_d = ids.to(dev), mask.to(dev)

        def run_native():
            native.encode_pooled(ids_d, mask_d, None, nv.POOL_MEAN_REF, False)

        @torch.no_grad()
        def run_hf():
            h = hf(input_ids=ids_d, attention_mask=mask_d).last_hidden_state
            m = mask_d[..., None].to(h.dtype)
            (h * m).sum(1) / m.sum(1)

        res = {'B': B, 'S': S, 'native_chunks_s': [], 'hf_sdpa_bf16_chunks_s': []}
        for _ in range(args.runs):     # alternating
            res['native_chunks_s'].append(round(B * args.steps / timed(run_native, args.steps, args.warmup), 1))
            res['hf_sdpa_bf16_chunks_s'].append(round(B * args.steps / timed(run_hf, args.steps, args.warmup), 1))
        f = flops_per_chunk(sh)
        res['native_peak_fraction'] = [round(c * f / PEAK_BF16, 3) for c in res['native_chunks_s']]
        res['hf_peak_fraction'] = [round(c * f / PEAK_BF16, 3) for c in res['hf_sdpa_bf16_chunks_s']]
        # separate profiled run: device time by kernel
        from torch.profiler import ProfilerActivity
        from torch.profiler import profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                run_native()
            torch.cuda.synchronize()
        from torch.autograd import DeviceType

        total = att = 0.0
        for evt in prof.key_averages():
            if evt.device_type != DeviceType.CUDA:
                continue
            t = getattr(evt, 'self_device_time_total', None) or getattr(evt, 'self_cuda_time_total', 0.0)
            total += t
            if 'attention_kernel<32' in evt.key:
                att += t
        res['d32_attention_share'] = round(att / total, 3) if total else None
        report['shapes'][name] = res
        print(name, json.dumps(res), flush=True)
        native.close()
        del hf, native
        torch.cuda.empty_cache()
    print(json.dumps(report))
    if args.out:
        Path(args.out).write_text(json.dumps(report, indent=1))


if __name__ == '__main__':
    main()
