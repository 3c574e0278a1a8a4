"""Where one C2 step's device time goes: torch.profiler (CUDA activities) over a few warmed steps of
NativeBertEncoder.encode_pooled (BERT-base, B 512, S 512, mean pooler, seeded weights as in bench.py).

Prints one JSON line naming the card and its power limit (read-only nvidia-smi query, same run), then one JSON
line per kernel name: device time per step, share of the step's kernel time, launches per step, and for the GEMMs
and the attention kernel the achieved TFLOP/s (FLOPs from the shapes).  The bias GEMM runs three of the four
linear layers; its launches are split by role from their order in the layer (QKV, attention-out, FFN-up,
FFN-down).  Profile in a run of its own: the tracing slows the host, so take step rates from bench.py."""
import argparse, json, subprocess, sys, tempfile
from collections import defaultdict
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

B, S = 512, 512
GEMM_ROLES = ('qkv', 'attn_out', 'ffn_up', 'ffn_down')


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--steps', type=int, default=3, help='profiled steps (default 3)')
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    import torch
    from transformers import BertConfig
    from torch.profiler import ProfilerActivity, profile

    import bench
    from distllm_b200 import _native as nv
    from distllm_b200.embed.encoders.native import NativeBertEncoder
    from distllm_b200.embed.encoders.weights import random_bert_state_dict
    if not torch.cuda.is_available():
        raise SystemExit('prof_step.py needs a CUDA device')
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({'device': torch.cuda.get_device_name(dev), 'name, power_limit, clocks.max.sm': q}), flush=True)

    cfg = BertConfig(**bench.BERT_BASE)
    h, inter = cfg.hidden_size, cfg.intermediate_size
    enc = NativeBertEncoder(cfg, random_bert_state_dict(cfg, seed=0, device=dev), device=dev)
    ids, mask, types = (t.to(dev) for t in bench.synthetic_batch(B, S, cfg.vocab_size, seed=1000))
    out = torch.empty((B, h), dtype=torch.float32, device=dev)
    for _ in range(args.warmup):
        enc.encode_pooled(ids, mask, types, nv.POOL_MEAN_REF, False, out=out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            enc.encode_pooled(ids, mask, types, nv.POOL_MEAN_REF, False, out=out)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        trace = Path(tmp) / 'trace.json'
        prof.export_chrome_trace(str(trace))
        events = json.loads(trace.read_text())['traceEvents']
    kernels = sorted((e for e in events if e.get('cat') == 'kernel'), key=lambda e: e['ts'])
    enc.close()

    m = B * S   # every chunk is full length: the packed layout keeps all rows
    gemm_flops = {'qkv': 2.0 * m * h * 3 * h, 'attn_out': 2.0 * m * h * h, 'ffn_up': 2.0 * m * h * inter,
                  'ffn_down': 2.0 * m * inter * h}
    att_flops = 4.0 * B * S * S * h   # one launch per layer
    rows = defaultdict(lambda: [0.0, 0, 0.0])   # name -> [us, launches, flops]
    g = 0
    for e in kernels:
        name = e['name']
        if 'gemm_h16_wgmma_kernel' in name:
            role = GEMM_ROLES[g % 4]
            g += 1
            key, fl = f'[{role}] {name}', gemm_flops[role]
        elif 'attention_kernel' in name:
            key, fl = name, att_flops
        else:
            key, fl = name, 0.0
        r = rows[key]
        r[0] += e['dur']
        r[1] += 1
        r[2] += fl
    total = sum(r[0] for r in rows.values())
    print(json.dumps({'steps': args.steps, 'kernel_ms_per_step': round(total / args.steps / 1e3, 3),
                      'gemm_share': round(sum(r[0] for k, r in rows.items() if 'gemm_h16' in k) / total, 4),
                      'gemm_launches_per_step': g / args.steps}), flush=True)
    for name, (us, n, fl) in sorted(rows.items(), key=lambda kv: -kv[1][0]):
        line = {'kernel': name[:120], 'ms_per_step': round(us / args.steps / 1e3, 3), 'share': round(us / total, 4),
                'launches_per_step': n / args.steps}
        if fl:
            line['tflops'] = round(fl / (us * 1e-6) / 1e12, 1)
        print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
