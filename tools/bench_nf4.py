"""16-bit weights against NF4 weights (quantization=True) on one GPU: the GEMM alone and whole forwards.

Both arms hold the same matrices: the 16-bit arm the load-time round trip to_storage(nf4_roundtrip(W)), the NF4 arm
the codes and scales of nf4_quantize(W) (embed/encoders/nf4.py).  Their outputs must be bitwise equal, and are
checked at every timed size.  The card's name and power limit are read in the same call.

  gemm      the four Mistral-7B projections (QKV 6144 x 4096, O 4096 x 4096, gate/up 28672 x 4096 with SwiGLU,
            down 4096 x 14336) and the BERT-base FFN-up (3072 x 768, GELU) at M in {128, 512, 2048, 16384, 65536}:
            microseconds per call (CUDA events), TFLOP/s and weight GB/s (weight bytes read once / call time)
  forward   encode_pooled on seeded random weights of the real shapes: Mistral-7B last-token at (B 4, S 512) -- the
            reference's SFR batch -- and (B 16, S 4096); Qwen3-Embedding-8B last-token at (B 16, S 4096); BERT-base
            mean at (B 512, S 512).  Sequences/s, device weight bytes and device footprint while running (weights +
            the library's workspace, from cudaMemGetInfo) of each arm, and the peak torch allocation while the NF4
            encoder loads.

Arms alternate, three runs each.

    python tools/bench_nf4.py [--parts gemm,forward] [--forwards mistral-sfr,mistral-c3,qwen3-8b,bert-c2]
                              [--runs 3] [--steps 2] [--warmup 1] [--out FILE.json]
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

GEMMS = {   # name: (N, K, epilogue name, storage)
    'mistral7b-qkv': (6144, 4096, 'bias', 'f16'),
    'mistral7b-o': (4096, 4096, 'bias', 'f16'),
    'mistral7b-gate-up': (28672, 4096, 'swiglu', 'f16'),
    'mistral7b-down': (4096, 14336, 'bias', 'f16'),
    'bert-base-ffn-up': (3072, 768, 'gelu', 'bf16'),
}
GEMM_M = (128, 512, 2048, 16384, 65536)

FORWARDS = {
    'mistral-sfr': dict(family='mistral', B=4, S=512, pool='last_token'),
    'mistral-c3': dict(family='mistral', B=16, S=4096, pool='last_token'),
    'qwen3-8b': dict(family='qwen3', B=16, S=4096, pool='last_token'),
    'bert-c2': dict(family='bert', B=512, S=512, pool='mean'),
}


def nf4_bytes(n: int, k: int) -> int:
    return n * k // 2 + (k // 64) * n * 4


def bench_gemm(runs: int) -> dict:
    from distllm_b200 import _native as nv
    from distllm_b200.embed.encoders.nf4 import nf4_quantize
    from distllm_b200.embed.encoders.nf4 import nf4_dequantize
    from distllm_b200.embed.encoders.weights import to_storage

    dev = torch.device('cuda:0')
    epis = {'bias': nv.EPI_BIAS, 'gelu': nv.EPI_BIAS_GELU, 'swiglu': nv.EPI_SWIGLU}
    out = {}
    for name, (n, k, epi_name, storage) in GEMMS.items():
        dt = {'f16': torch.float16, 'bf16': torch.bfloat16}[storage]
        epi = epis[epi_name]
        g = torch.Generator(device=dev).manual_seed(n + k)
        codes, absmax = nf4_quantize(torch.randn((n, k), generator=g, device=dev) * 0.02)
        w16 = to_storage(nf4_dequantize(codes, absmax), dev, dt)
        bias = None if epi == nv.EPI_SWIGLU else torch.randn(n, generator=g, device=dev) * 0.02
        rows = {}
        for m in GEMM_M:
            a = torch.randn((m, k), generator=g, device=dev).to(dt)
            arms = {'h16': lambda: nv.gemm_h16(a, w16, bias, None, epi),
                    'nf4': lambda: nv.gemm_nf4(a, codes, absmax, bias, None, epi)}
            ref, got = arms['h16'](), arms['nf4']()
            equal = bool(torch.equal(ref.view(torch.int16), got.view(torch.int16)))
            del ref, got
            flop = 2.0 * m * n * k
            iters = int(min(200, max(5, 0.2 / (flop / 4e14 + 5e-6))))
            r = {'bitwise_equal': equal, 'iters': iters}
            for arm in arms:
                r[f'{arm}_us'] = []
            for _ in range(runs):
                for arm, fn in arms.items():
                    fn()
                    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    start.record()
                    for _ in range(iters):
                        fn()
                    stop.record()
                    stop.synchronize()
                    r[f'{arm}_us'].append(round(start.elapsed_time(stop) * 1e3 / iters, 1))
            for arm, wbytes in (('h16', n * k * 2), ('nf4', nf4_bytes(n, k))):
                best = min(r[f'{arm}_us'])
                r[f'{arm}_tflops'] = round(flop / best / 1e6, 1)
                r[f'{arm}_weight_gbs'] = round(wbytes / best / 1e3, 1)
            r['nf4_over_h16'] = round(min(r['nf4_us']) / min(r['h16_us']), 3)
            rows[m] = r
            print('gemm', name, m, json.dumps(r), flush=True)
            del a
        out[name] = {'N': n, 'K': k, 'epilogue': epi_name, 'storage': storage, 'M': rows}
        del codes, absmax, w16
        torch.cuda.empty_cache()
    return out


def configs(family: str):
    from transformers import BertConfig
    from transformers import MistralConfig
    from transformers import Qwen3Config

    if family == 'bert':
        return BertConfig(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                          intermediate_size=3072, max_position_embeddings=512)
    common = dict(vocab_size=32000, hidden_size=4096, num_attention_heads=32, num_key_value_heads=8, head_dim=128,
                  max_position_embeddings=32768, rms_norm_eps=1e-5, initializer_range=0.02)
    if family == 'mistral':   # Mistral-7B-v0.1 / SFR-Embedding-Mistral
        return MistralConfig(**common, num_hidden_layers=32, intermediate_size=14336, rope_theta=10000.0,
                             sliding_window=4096)
    return Qwen3Config(**common, num_hidden_layers=36, intermediate_size=12288,   # Qwen3-Embedding-8B
                       rope_parameters={'rope_type': 'default', 'rope_theta': 1e6}, tie_word_embeddings=False)


def timed(fn, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def bench_forward(name: str, runs: int, steps: int, warmup: int) -> dict:
    from distllm_b200 import _native as nv
    from distllm_b200.embed.encoders import native
    from distllm_b200.embed.encoders import weights as W
    from distllm_b200.embed.encoders.nf4 import is_quantized_linear
    from distllm_b200.embed.encoders.nf4 import nf4_roundtrip

    spec = FORWARDS[name]
    cfg = configs(spec['family'])
    dev = torch.device('cuda:0')
    cls, make = {'bert': (native.NativeBertEncoder, W.random_bert_state_dict),
                 'mistral': (native.NativeMistralEncoder, W.random_mistral_state_dict),
                 'qwen3': (native.NativeQwen3Encoder, W.random_qwen3_state_dict)}[spec['family']]
    kw = {} if spec['family'] == 'bert' else {'dtype': torch.float16}
    sd = make(cfg, seed=0, device=dev, **kw)
    sd_bytes = sum(t.nbytes for t in sd.values())
    res = {**spec}
    B, S = spec['B'], spec['S']
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, cfg.vocab_size, (B, S), generator=g).to(dev)
    mask = torch.ones(B, S, dtype=torch.int64, device=dev)
    kind = nv.POOL_LAST_TOKEN if spec['pool'] == 'last_token' else nv.POOL_MEAN_REF
    outs = {a: torch.empty(B, cfg.hidden_size, device=dev) for a in ('h16', 'nf4')}

    def device_used() -> int:
        """Bytes in use on the device: the library's own workspace is not a torch allocation."""
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free, total = torch.cuda.mem_get_info(dev)
        return total - free

    used0 = device_used()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    enc_q = cls(cfg, sd, device=dev, nf4=True)
    torch.cuda.synchronize()
    res['nf4_load_peak_bytes'] = torch.cuda.max_memory_allocated(dev) - base
    enc_q.encode_pooled(ids, mask, None, kind, True, out=outs['nf4'])
    used1 = device_used()
    # each arm's device footprint while it runs: weights, workspace at this batch, rounded to the allocator's pages
    res['nf4_device_bytes'] = used1 - used0
    # the load-time path's matrices, rounded to 16 bits one at a time (the round trip's fp32 copy of a whole model
    # would not fit beside the rest)
    dt = nv.STORAGE_TORCH_DTYPE[enc_q.storage]
    rt = {k: (W.to_storage(nf4_roundtrip(v), dev, dt) if is_quantized_linear(k, v) else v) for k, v in sd.items()}
    del sd
    enc_h = cls(cfg, rt, device=dev)
    del rt
    enc_h.encode_pooled(ids, mask, None, kind, True, out=outs['h16'])
    res['h16_device_bytes'] = device_used() - used1 + sd_bytes   # sd was freed in between
    res['h16_weight_bytes'] = enc_h.weight_bytes()
    res['nf4_weight_bytes'] = enc_q.weight_bytes()
    arms = {'h16': lambda: enc_h.encode_pooled(ids, mask, None, kind, True, out=outs['h16']),
            'nf4': lambda: enc_q.encode_pooled(ids, mask, None, kind, True, out=outs['nf4'])}
    for a in arms:
        res[f'{a}_seq_s'] = []
    for _ in range(runs):
        for a, fn in arms.items():
            res[f'{a}_seq_s'].append(round(B * steps / timed(fn, steps, warmup), 2))
    res['bitwise_equal'] = bool(torch.equal(outs['h16'].view(torch.int32), outs['nf4'].view(torch.int32)))
    res['nf4_over_h16_seq_s'] = round(max(res['nf4_seq_s']) / max(res['h16_seq_s']), 3)
    enc_h.close()
    enc_q.close()
    del enc_h, enc_q
    torch.cuda.empty_cache()
    print('forward', name, json.dumps(res), flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--parts', default='gemm,forward')
    ap.add_argument('--forwards', default=','.join(FORWARDS))
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=2)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_nf4 needs a CUDA device')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                           '-i', '0'], capture_output=True, text=True).stdout.strip()
    print('card:', card, flush=True)
    report = {'card': card, 'runs': args.runs}
    parts = args.parts.split(',')
    if 'gemm' in parts:
        report['gemm'] = bench_gemm(args.runs)
    if 'forward' in parts:
        report['forward'] = {f: bench_forward(f, args.runs, args.steps, args.warmup) for f in args.forwards.split(',')}
    print(json.dumps(report))
    if args.out:
        Path(args.out).write_text(json.dumps(report, indent=1))


if __name__ == '__main__':
    main()
