"""What a LoRA adapter costs under NF4 storage (quantization=True): U's GEMM and the tail k-blocks of the NF4 GEMM.

Three arms hold the same Mistral-7B model (seeded random weights of the real shapes, rank-16 LoRA on q/v or on all
seven projections, lora_B entries of magnitude 1e-4 .. 1e-2):

  nf4+lora   NF4 weights, the adapter unmerged (b2e_encoder_create_nf4_lora): per adapted slot U = X . A_cat^T on the
             16-bit GEMM, then the NF4 GEMM with R/64 extra k-blocks
  nf4        the same NF4 weights without the adapter
  merged16   16-bit weights to_storage(nf4_roundtrip(W) + s B A): the nf4_storage: false path

  forward    encode_pooled (last token, normalised) at the reference's SFR batch (B 4, S 512) and at C3 (B 16,
             S 4096): sequences/s per arm, arms alternating, three runs each; outputs must repeat bit for bit between
             runs; the LoRA factor bytes and the U workspace bytes
  gemm       per Mistral-7B projection at M in {128, 2048, 65536} with R = 64 (a rank-16 slot padded): microseconds of
             the U GEMM (N = 128), of the NF4 GEMM, and of the NF4 GEMM with its tail (CUDA events)

The card's name and power limit are read in the same call.

    python tools/bench_lora.py [--parts gemm,forward] [--shapes sfr,c3] [--targets qv,all7] [--runs 3] [--steps 2]
                               [--warmup 1] [--out FILE.json]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

REPO = Path(__file__).resolve().parents[1]
if str(REPO) not in sys.path:
    sys.path.insert(0, str(REPO))

from tools.bench_nf4 import configs  # noqa: E402
from tools.bench_nf4 import timed  # noqa: E402

GEMMS = {   # name: (N, K, epilogue)
    'qkv': (6144, 4096, 'bias'),
    'o': (4096, 4096, 'bias'),
    'gate-up': (28672, 4096, 'swiglu'),
    'down': (4096, 14336, 'bias'),
}
GEMM_M = (128, 2048, 65536)
SHAPES = {'sfr': (4, 512), 'c3': (16, 4096)}
TARGETS = {'qv': ('self_attn.q_proj', 'self_attn.v_proj'),
           'all7': ('self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj', 'self_attn.o_proj', 'mlp.gate_proj',
                    'mlp.up_proj', 'mlp.down_proj')}
RANK = 16


def events_us(fn, iters: int) -> float:
    fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) * 1e3 / iters


def bench_gemm(runs: int) -> dict:
    from distllm_b200 import _native as nv
    from distllm_b200.embed.encoders.nf4 import nf4_quantize

    dev = torch.device('cuda:0')
    epis = {'bias': nv.EPI_BIAS, 'swiglu': nv.EPI_SWIGLU}
    out = {}
    for name, (n, k, epi_name) in GEMMS.items():
        epi = epis[epi_name]
        g = torch.Generator(device=dev).manual_seed(n + k)
        codes, absmax = nf4_quantize(torch.randn((n, k), generator=g, device=dev) * 0.02)
        a_cat = (torch.randn((128, k), generator=g, device=dev) * 0.02).half()
        b_cat = (torch.randn((n, 64), generator=g, device=dev) * 0.01).half()
        rows = {}
        for m in GEMM_M:
            x = torch.randn((m, k), generator=g, device=dev).half()
            u = nv.gemm_h16(x, a_cat, None)
            arms = {'u_gemm': lambda: nv.gemm_h16(x, a_cat, None),
                    'nf4': lambda: nv.gemm_nf4(x, codes, absmax, None, None, epi),
                    'nf4_tail': lambda: nv.gemm_nf4_lora(x, codes, absmax, u, b_cat, None, None, epi)}
            iters = int(min(200, max(5, 0.2 / (2.0 * m * n * k / 4e14 + 5e-6))))
            r = {a: [] for a in arms}
            for _ in range(runs):
                for a, fn in arms.items():
                    r[a].append(round(events_us(fn, iters), 1))
            best = {a: min(v) for a, v in r.items()}
            r['tail_us'] = round(best['nf4_tail'] - best['nf4'], 1)
            r['lora_over_nf4'] = round((best['u_gemm'] + best['nf4_tail']) / best['nf4'], 3)
            rows[m] = r
            print('gemm', name, m, json.dumps(r), flush=True)
            del x, u
        out[name] = {'N': n, 'K': k, 'R': 64, 'epilogue': epi_name, 'M': rows}
        torch.cuda.empty_cache()
    return out


def adapter_for(cfg, targets, dev) -> dict:
    g = torch.Generator(device=dev).manual_seed(7)
    h, i = cfg.hidden_size, cfg.intermediate_size
    d, heads, kv = cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
    shapes = {'self_attn.q_proj': (heads * d, h), 'self_attn.k_proj': (kv * d, h), 'self_attn.v_proj': (kv * d, h),
              'self_attn.o_proj': (h, heads * d), 'mlp.gate_proj': (i, h), 'mlp.up_proj': (i, h),
              'mlp.down_proj': (h, i)}
    lora = {}
    for layer in range(cfg.num_hidden_layers):
        for t in targets:
            o, k = shapes[t]
            a = torch.randn((RANK, k), generator=g, device=dev) / k ** 0.5
            mag = 10.0 ** (torch.rand((o, RANK), generator=g, device=dev) * 2.0 - 4.0)
            b = mag * (torch.randint(0, 2, (o, RANK), generator=g, device=dev) * 2 - 1)
            lora[f'layers.{layer}.{t}'] = (a, b, 32.0 / RANK)
    return lora


def bench_forward(shape: str, targets: str, runs: int, steps: int, warmup: int) -> dict:
    from distllm_b200 import _native as nv
    from distllm_b200.embed.encoders import native
    from distllm_b200.embed.encoders import weights as W
    from distllm_b200.embed.encoders.adapters import Adapter
    from distllm_b200.embed.encoders.adapters import merge_adapter
    from distllm_b200.embed.encoders.nf4 import is_quantized_linear
    from distllm_b200.embed.encoders.nf4 import nf4_roundtrip

    cfg = configs('mistral')
    dev = torch.device('cuda:0')
    B, S = SHAPES[shape]
    sd = W.random_mistral_state_dict(cfg, seed=0, device=dev, dtype=torch.float16)
    lora = adapter_for(cfg, TARGETS[targets], dev)
    res = {'B': B, 'S': S, 'targets': targets, 'rank': RANK}
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, cfg.vocab_size, (B, S), generator=g).to(dev)
    mask = torch.ones(B, S, dtype=torch.int64, device=dev)
    kind = nv.POOL_LAST_TOKEN
    encs = {'nf4+lora': native.NativeMistralEncoder(cfg, sd, device=dev, nf4=True, lora=lora),
            'nf4': native.NativeMistralEncoder(cfg, sd, device=dev, nf4=True)}
    dt = nv.STORAGE_TORCH_DTYPE[encs['nf4'].storage]
    merged = {}
    for k, v in sd.items():   # one matrix at a time: an fp32 copy of the whole model would not fit beside the rest
        if is_quantized_linear(k, v):
            m = merge_adapter({k: nf4_roundtrip(v)}, Adapter('LORA', lora={k[:-7]: lora[k[:-7]]}
                                                             if k[:-7] in lora else {}))
            merged[k] = W.to_storage(m[k], dev, dt)
        else:
            merged[k] = v
    del sd
    encs['merged16'] = native.NativeMistralEncoder(cfg, merged, device=dev)
    del merged
    torch.cuda.empty_cache()
    res['lora_factor_bytes'] = encs['nf4+lora'].lora_bytes()
    res['u_workspace_bytes'] = B * S * 128 * 2
    res['nf4_weight_bytes'] = encs['nf4'].weight_bytes()
    res['merged16_weight_bytes'] = encs['merged16'].weight_bytes()
    outs = {a: [] for a in encs}
    for a in encs:
        res[f'{a}_seq_s'] = []
    for _ in range(runs):
        for a, enc in encs.items():
            res[f'{a}_seq_s'].append(round(B * steps / timed(
                lambda: enc.encode_pooled(ids, mask, None, kind, True), steps, warmup), 2))
            outs[a].append(enc.encode_pooled(ids, mask, None, kind, True).cpu())
    res['repeatable'] = all(all(torch.equal(o[0].view(torch.int32), x.view(torch.int32)) for x in o[1:])
                            for o in outs.values())
    cos = torch.nn.functional.cosine_similarity(outs['nf4+lora'][0], outs['merged16'][0], dim=-1)
    res['lora_vs_merged16_min_cos'] = round(float(cos.min()), 6)
    best = {a: max(res[f'{a}_seq_s']) for a in encs}
    res['lora_over_nf4_seq_s'] = round(best['nf4+lora'] / best['nf4'], 3)
    res['lora_over_merged16_seq_s'] = round(best['nf4+lora'] / best['merged16'], 3)
    for enc in encs.values():
        enc.close()
    del encs
    torch.cuda.empty_cache()
    print('forward', shape, targets, json.dumps(res), flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--parts', default='gemm,forward')
    ap.add_argument('--shapes', default=','.join(SHAPES))
    ap.add_argument('--targets', default=','.join(TARGETS))
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=2)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_lora needs a CUDA device')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                           '-i', '0'], capture_output=True, text=True).stdout.strip()
    print('card:', card, flush=True)
    report = {'card': card, 'runs': args.runs}
    parts = args.parts.split(',')
    if 'gemm' in parts:
        report['gemm'] = bench_gemm(args.runs)
    if 'forward' in parts:
        report['forward'] = {f'{s}-{t}': bench_forward(s, t, args.runs, args.steps, args.warmup)
                             for s in args.shapes.split(',') for t in args.targets.split(',')}
    print(json.dumps(report))
    if args.out:
        Path(args.out).write_text(json.dumps(report, indent=1))


if __name__ == '__main__':
    main()
