"""ESM C throughput on one GPU: the native ``esmc`` path against a bfloat16 + SDPA torch transcription of the same model.

Shapes (seeded random weights of the real sizes, ``weights.random_esmc_state_dict``; residues drawn from the 20 amino
acids between <cls> and <eos>; mean pooler):
  300m   esmc-300m   30 layers, H = 960 (15 heads x 64), I = 2560
  600m   esmc-600m   36 layers, H = 1152 (18 heads x 64), I = 3072
Batches: B = 64 rows of S = 1024 tokens ('full'), and B = 64 rows right-padded to 1024 with lengths U{64..1024}
('ragged'; the native path runs the attended tokens only, the torch bar the padded batch, as a torch user would).

Per shape and batch, three alternating runs each of:
  * native   NativeEsmcEncoder.encode_pooled (the ``esmc`` build's storage type): sequences/s and algorithmic
             TFLOP/s over the attended tokens (per layer 8 s H^2 + 6 s H I + 4 s^2 H for a sequence of s tokens);
  * torch    the forward pass of tools/oracle_esmc.py written in bfloat16 with F.scaled_dot_product_attention and the
             boolean key-padding mask, + the same mean pooling.  Neither the esm package nor flash-attn is installed,
             so this is the bar.
In a separate torch.profiler run, the share of the native step's device time in qk_layernorm_rope_kernel.  The card's
name and power limit are read in the same call.

    python tools/bench_esmc.py [--shapes 300m,600m] [--steps 3] [--warmup 1] [--runs 3] [--out FILE.json]
"""

from __future__ import annotations

import argparse
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import torch
import torch.nn.functional as F  # noqa: N812

REPO = Path(__file__).resolve().parents[1]
if str(REPO) not in sys.path:
    sys.path.insert(0, str(REPO))

from tools.bench_qwen3 import kernel_share  # noqa: E402
from tools.bench_qwen3 import timed  # noqa: E402

SHAPES = {'300m': dict(layers=30, hidden=960, inter=2560), '600m': dict(layers=36, hidden=1152, inter=3072)}
B, S = 64, 1024


def flops(sh: dict, lens: torch.Tensor) -> float:
    """Algorithmic FLOPs of a batch: per layer and sequence of s tokens 2 s H 3H (qkv) + 2 s H H (out) + 2 s H 2I
    (gate, up) + 2 s I H (down) + 4 s^2 H (scores and context)."""
    h, i = sh['hidden'], sh['inter']
    s = lens.double()
    return float(sh['layers'] * (s * (8.0 * h * h + 6.0 * h * i) + 4.0 * s * s * h).sum())


def batch(kind: str, seed: int):
    g = torch.Generator().manual_seed(seed)
    lens = torch.full((B,), S) if kind == 'full' else torch.randint(64, S + 1, (B,), generator=g)
    ids = torch.randint(4, 24, (B, S), generator=g)
    ids[:, 0] = 0
    ids[torch.arange(B), lens - 1] = 2
    mask = (torch.arange(S)[None] < lens[:, None]).long()
    ids[mask == 0] = 1
    return ids, mask, lens


def torch_bar(sd: dict, layers: int):
    """ESM C in bfloat16 with SDPA (tools/oracle_esmc.py's steps), mean-pooled: fn(ids, mask) -> [B, H]."""
    from tools import oracle_esmc as O

    w = {k: v.to(torch.bfloat16) for k, v in sd.items() if not k.startswith('sequence_head.')}
    h = w['embed.weight'].shape[1]
    scale = math.sqrt(layers / 36)
    cos, sin = (t.to(w['embed.weight'].device, torch.bfloat16) for t in O.rotary_tables(S))

    @torch.no_grad()
    def run(ids, mask):
        x = w['embed.weight'][ids]
        b, s, _ = x.shape
        key = mask.bool()[:, None, None, :]
        for l in range(layers):
            p = f'transformer.blocks.{l}.'
            y = F.layer_norm(x, (h,), w[p + 'attn.layernorm_qkv.0.weight'], w[p + 'attn.layernorm_qkv.0.bias'], 1e-5)
            q, k, v = F.linear(y, w[p + 'attn.layernorm_qkv.1.weight']).split(h, dim=-1)
            q = O.rotate(F.layer_norm(q, (h,), w[p + 'attn.q_ln.weight'], None, 1e-5).view(b, s, -1, 64), cos, sin)
            k = O.rotate(F.layer_norm(k, (h,), w[p + 'attn.k_ln.weight'], None, 1e-5).view(b, s, -1, 64), cos, sin)
            ctx = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2),
                                                 v.view(b, s, -1, 64).transpose(1, 2), attn_mask=key)
            x = x + F.linear(ctx.transpose(1, 2).reshape(b, s, h), w[p + 'attn.out_proj.weight']) / scale
            y = F.layer_norm(x, (h,), w[p + 'ffn.0.weight'], w[p + 'ffn.0.bias'], 1e-5)
            gate, up = F.linear(y, w[p + 'ffn.1.weight']).chunk(2, dim=-1)
            x = x + F.linear(F.silu(gate) * up, w[p + 'ffn.3.weight']) / scale
        x = F.layer_norm(x, (h,), w['transformer.norm.weight'], None, 1e-5)
        m = mask[..., None].to(x.dtype)
        return ((x * m).sum(1) / m.sum(1)).float()

    return run


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default=','.join(SHAPES))
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_esmc needs a CUDA device')
    from distllm_b200 import _native as nv
    from distllm_b200.embed.encoders import weights as W
    from distllm_b200.embed.encoders.native import NativeEsmcEncoder

    dev = torch.device('cuda:0')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                           '-i', '0'], capture_output=True, text=True).stdout.strip()
    report = {'card': card, 'storage': nv.storage_for_arch('esmc'), 'B': B, 'S': S, 'steps': args.steps,
              'runs': args.runs, 'shapes': {}}
    print('card:', card, flush=True)
    for name in args.shapes.split(','):
        sh = SHAPES[name]
        sd = W.random_esmc_state_dict(sh['hidden'], sh['layers'], sh['inter'], seed=0, device=dev)
        enc = NativeEsmcEncoder(W.esmc_config(sd), sd, device=dev)
        bar = torch_bar(sd, sh['layers'])
        out = torch.empty(B, sh['hidden'], device=dev)
        res = {}
        for kind in ('full', 'ragged'):
            ids, mask, lens = batch(kind, seed=1)
            ids, mask = ids.to(dev), mask.to(dev)
            fl = flops(sh, lens)
            arms = {'native': lambda: enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_PER_ROW, False, out=out),
                    'torch_bf16_sdpa': lambda: bar(ids, mask)}
            r = {f'{a}_seq_s': [] for a in arms}
            for _ in range(args.runs):     # alternating arms
                for a, fn in arms.items():
                    r[f'{a}_seq_s'].append(round(B * args.steps / timed(fn, args.steps, args.warmup), 2))
            for a in arms:
                r[f'{a}_tflops'] = [round(x / B * fl / 1e12, 1) for x in r[f'{a}_seq_s']]
            r['qk_layernorm_rope_share'] = kernel_share(arms['native'], 'qk_layernorm_rope_kernel')
            r['attended_tokens'] = int(lens.sum())
            res[kind] = r
            print(name, kind, json.dumps(r), flush=True)
        enc.close()
        del enc, bar, sd
        torch.cuda.empty_cache()
        report['shapes'][name] = res
    print(json.dumps(report))
    if args.out:
        Path(args.out).write_text(json.dumps(report, indent=1))


if __name__ == '__main__':
    main()
