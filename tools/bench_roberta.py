"""Throughput of the RoBERTa / XLM-RoBERTa path at published shapes, seeded weights, synthetic ids.

Shapes: BGE-M3 (24 layers, H 1024, 16 x 64, I 4096, vocab 250002, 8194 positions) at B 64 / S 512 and B 4 / S 8192;
multilingual-e5-base (12 layers, H 768) and paraphrase-multilingual-MiniLM-L12-v2 (12 layers, H 384, 12 x 32) at
B 512 / S 512.  Rows are ragged (lengths uniform in [S/2, S], right-padded, pad id 1 behind them).

Arms, alternating, three timed runs each: the native encoder (b2e_encode_pooled, mean pooler, the library's default
storage for BERT) and HF XLMRobertaModel in bfloat16 with SDPA plus the same masked mean, on the same GPU.  Also
reported: whether repeated native runs give bit-identical pooled rows, and the position kernel's share of device time
from torch.profiler.  Prints one JSON object; the card name and power limit are read in the same process.

    python tools/bench_roberta.py [--shapes bge-m3-512,bge-m3-8192,e5-base,minilm] [--steps 5]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from distllm_b200 import _native as nv  # noqa: E402
from distllm_b200.embed.encoders import weights as W  # noqa: E402
from distllm_b200.embed.encoders.native import NativeRobertaEncoder  # noqa: E402

SHAPES = {
    'bge-m3-512': (dict(hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
                        vocab_size=250002, max_position_embeddings=8194), 64, 512),
    'bge-m3-8192': (dict(hidden_size=1024, num_attention_heads=16, intermediate_size=4096, num_hidden_layers=24,
                         vocab_size=250002, max_position_embeddings=8194), 4, 8192),
    'e5-base': (dict(hidden_size=768, num_attention_heads=12, intermediate_size=3072, num_hidden_layers=12,
                     vocab_size=250002, max_position_embeddings=514), 512, 512),
    'minilm': (dict(hidden_size=384, num_attention_heads=12, intermediate_size=1536, num_hidden_layers=12,
                    vocab_size=250002, max_position_embeddings=514), 512, 512),
}


def card() -> dict:
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (x.strip() for x in out.split(','))
        return {'name': name, 'power_limit': power}
    except Exception as e:  # noqa: BLE001
        return {'name': torch.cuda.get_device_name(0), 'power_limit': f'not read ({e})'}


def timed(fn, steps: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps / 1e3


def run_shape(name: str, steps: int) -> dict:
    from transformers import XLMRobertaConfig
    from transformers import XLMRobertaModel

    kw, b, s = SHAPES[name]
    cfg = XLMRobertaConfig(type_vocab_size=1, pad_token_id=1, layer_norm_eps=1e-5, **kw)
    dev = torch.device('cuda:0')
    sd = W.random_bert_state_dict(cfg, seed=0, device=dev)
    g = torch.Generator(device='cpu').manual_seed(1)
    lens = torch.randint(s // 2, s + 1, (b,), generator=g)
    mask = (torch.arange(s)[None] < lens[:, None]).long()
    ids = torch.randint(3, cfg.vocab_size, (b, s), generator=g)
    ids[mask == 0] = 1
    ids, mask = ids.to(dev), mask.to(dev)

    enc = NativeRobertaEncoder(cfg, sd, device=dev)
    out = torch.empty(b, cfg.hidden_size, device=dev)

    def native():
        enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_PER_ROW, False, out=out)

    cfg._attn_implementation = 'sdpa'
    hf = XLMRobertaModel(cfg, add_pooling_layer=False).to(dev, torch.bfloat16).eval()
    hf.load_state_dict({k: v.to(torch.bfloat16) for k, v in sd.items()}, strict=False)
    del sd

    @torch.no_grad()
    def torch_arm():
        y = hf(input_ids=ids, attention_mask=mask).last_hidden_state.float()
        m = mask[..., None].float()
        return (y * m).sum(1) / m.sum(1)

    native()
    torch_arm()
    torch.cuda.synchronize()
    first = out.clone()
    runs = {'native': [], 'torch_bf16_sdpa': []}
    for _ in range(3):
        runs['native'].append(b / timed(native, steps))
        runs['torch_bf16_sdpa'].append(b / timed(torch_arm, steps))
    repeat_equal = bool(torch.equal(first, out))

    from torch.profiler import ProfilerActivity
    from torch.profiler import profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        native()
        torch.cuda.synchronize()
    total = pos = 0.0
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA:   # device kernels and copies only
            continue
        t = e.self_device_time_total
        total += t
        if 'roberta_positions' in e.key:
            pos += t
    enc.close()
    del hf
    torch.cuda.empty_cache()
    return {'B': b, 'S': s, 'layers': cfg.num_hidden_layers, 'hidden': cfg.hidden_size,
            'seq_per_s': {k: [round(x, 1) for x in v] for k, v in runs.items()},
            'pooled_repeat_bitwise_equal': repeat_equal,
            'position_kernel_share': round(pos / total, 6) if total else None}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default=','.join(SHAPES))
    ap.add_argument('--steps', type=int, default=5)
    args = ap.parse_args()
    result = {'card': card(), 'storage': nv.storage_for_arch('bert')}
    for name in args.shapes.split(','):
        result[name] = run_shape(name, args.steps)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
