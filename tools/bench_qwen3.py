"""Qwen3-Embedding throughput on one GPU: the native path against the same shape run as Mistral and against HF.

Shapes (synthetic ids, every row S tokens long, seeded random fp16 weights of the real sizes, vocabulary 32 000):
  0.6b   Qwen3-Embedding-0.6B   28 layers, H = 1024, 16 q / 8 kv heads x 128, I = 3072    B = 64, S = 1024,
                                last_token and mean poolers
  8b     Qwen3-Embedding-8B     36 layers, H = 4096, 32 q / 8 kv heads x 128, I = 12288   B = 16, S = 4096,
                                last_token pooler

Per shape and pooler, three alternating runs each of:
  * qwen3     encode_pooled of NativeQwen3Encoder: sequences/s and algorithmic TFLOP/s
              (bench.py's mistral_flops_per_seq with heads x 128 for the q and o projections and the attention width);
  * mistral   the same weights without q_norm / k_norm on NativeMistralEncoder (rotary alone in place of the fused
              norm + rotary kernel): what the head norms cost;
  * hf        HF Qwen3Model in bfloat16 with attn_implementation='sdpa' + the same pooling, after the native arms.
In a separate torch.profiler run, the share of the qwen3 step's device time in qk_rmsnorm_rope_kernel.  The card's
name and power limit are read in the same call.

    python tools/bench_qwen3.py [--shapes 0.6b,8b] [--steps 3] [--warmup 1] [--runs 3] [--out FILE.json]
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

SHAPES = {
    '0.6b': dict(layers=28, hidden=1024, heads=16, kv=8, inter=3072, B=64, S=1024, poolers=('last_token', 'mean')),
    '8b': dict(layers=36, hidden=4096, heads=32, kv=8, inter=12288, B=16, S=4096, poolers=('last_token',)),
}


def flops_per_seq(sh: dict, s: int) -> float:
    """Per layer: 2 S H (heads + 2 kv) 128 (q, k, v) + 2 S H heads 128 (o) + 6 S H I (gate, up, down) + the
    causal-skipped attention 2 S (S + 128) heads 128 that the kernel's chunk skipping executes."""
    h, i, a = sh['hidden'], sh['inter'], sh['heads'] * 128
    qc = (sh['heads'] + 2 * sh['kv']) * 128
    return sh['layers'] * (2.0 * s * h * qc + 2.0 * s * h * a + 6.0 * s * h * i + 2.0 * s * (s + 128) * a)


def configs(sh: dict):
    from transformers import MistralConfig
    from transformers import Qwen3Config

    common = dict(vocab_size=32000, hidden_size=sh['hidden'], num_hidden_layers=sh['layers'],
                  num_attention_heads=sh['heads'], num_key_value_heads=sh['kv'], head_dim=128,
                  intermediate_size=sh['inter'], max_position_embeddings=32768, rms_norm_eps=1e-6,
                  initializer_range=0.02)
    qcfg = Qwen3Config(**common, rope_parameters={'rope_type': 'default', 'rope_theta': 1e6},
                       tie_word_embeddings=False)
    mcfg = MistralConfig(**common, rope_theta=1e6, sliding_window=None)
    return qcfg, mcfg


def timed(fn, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def kernel_share(fn, name: str) -> float | None:
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = part = 0.0
    for evt in prof.key_averages():
        if evt.device_type != DeviceType.CUDA:
            continue
        t = getattr(evt, 'self_device_time_total', None) or getattr(evt, 'self_cuda_time_total', 0.0)
        total += t
        if name in evt.key:
            part += t
    return round(part / total, 4) if total else None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default=','.join(SHAPES))
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_qwen3 needs a CUDA device')
    from transformers import Qwen3Model

    from distllm_b200 import _native as nv
    from distllm_b200.embed.encoders.native import NativeMistralEncoder
    from distllm_b200.embed.encoders.native import NativeQwen3Encoder
    from distllm_b200.embed.encoders.weights import random_qwen3_state_dict

    dev = torch.device('cuda:0')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                           '-i', '0'], capture_output=True, text=True).stdout.strip()
    report = {'card': card, 'steps': args.steps, 'runs': args.runs, 'shapes': {}}
    print('card:', card, flush=True)
    for name in args.shapes.split(','):
        sh = SHAPES[name]
        qcfg, mcfg = configs(sh)
        B, S = sh['B'], sh['S']
        sd = random_qwen3_state_dict(qcfg, seed=0, device=dev, dtype=torch.float16)
        qwen = NativeQwen3Encoder(qcfg, sd, device=dev)
        mistral = NativeMistralEncoder(mcfg, {k: v for k, v in sd.items() if 'q_norm' not in k and 'k_norm' not in k},
                                       device=dev)
        g = torch.Generator().manual_seed(1)
        ids = torch.randint(3, qcfg.vocab_size, (B, S), generator=g).to(dev)
        mask = torch.ones(B, S, dtype=torch.int64, device=dev)
        out = torch.empty(B, sh['hidden'], device=dev)
        flops = flops_per_seq(sh, S)
        res = {'B': B, 'S': S, 'gflop_per_seq': round(flops / 1e9, 1), 'poolers': {}}
        for pooler in sh['poolers']:
            kind = nv.POOL_LAST_TOKEN if pooler == 'last_token' else nv.POOL_MEAN_REF
            arms = {'qwen3': lambda: qwen.encode_pooled(ids, mask, None, kind, True, out=out),
                    'mistral': lambda: mistral.encode_pooled(ids, mask, None, kind, True, out=out)}
            r = {f'{a}_seq_s': [] for a in arms}
            for _ in range(args.runs):     # alternating arms
                for a, fn in arms.items():
                    r[f'{a}_seq_s'].append(round(B * args.steps / timed(fn, args.steps, args.warmup), 2))
            r['qwen3_tflops'] = [round(x * flops / 1e12, 1) for x in r['qwen3_seq_s']]
            r['mistral_tflops'] = [round(x * flops / 1e12, 1) for x in r['mistral_seq_s']]
            r['qk_norm_rope_share'] = kernel_share(arms['qwen3'], 'qk_rmsnorm_rope_kernel')
            res['poolers'][pooler] = r
            print(name, pooler, json.dumps(r), flush=True)
        qwen.close()
        mistral.close()
        del qwen, mistral
        torch.cuda.empty_cache()

        qcfg._attn_implementation = 'sdpa'
        with torch.device(dev):
            hf = Qwen3Model(qcfg).to(torch.bfloat16)
        hf.load_state_dict(sd, strict=False)
        del sd
        torch.cuda.empty_cache()
        hf.eval()

        for pooler in sh['poolers']:
            @torch.no_grad()
            def run_hf():
                h = hf(input_ids=ids, attention_mask=mask).last_hidden_state
                if pooler == 'last_token':
                    v = h[:, -1]
                else:
                    m = mask[..., None].to(h.dtype)
                    v = (h * m).sum(1) / m.sum(1)
                torch.nn.functional.normalize(v.float(), dim=-1)

            hf_s = [round(B * args.steps / timed(run_hf, args.steps, args.warmup), 2) for _ in range(args.runs)]
            res['poolers'][pooler]['hf_sdpa_bf16_seq_s'] = hf_s
            res['poolers'][pooler]['hf_tflops'] = [round(x * flops / 1e12, 1) for x in hf_s]
            print(name, pooler, 'hf', hf_s, flush=True)
        del hf
        torch.cuda.empty_cache()
        report['shapes'][name] = res
    print(json.dumps(report))
    if args.out:
        Path(args.out).write_text(json.dumps(report, indent=1))


if __name__ == '__main__':
    main()
