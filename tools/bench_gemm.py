"""The library's GEMM (nv.gemm_h16) against torch.nn.functional.linear (cuBLAS, a ceiling only) at every GEMM shape
bench.py runs: C2 (BERT-base, bfloat16 build), C5 (ESM-2 650M, bfloat16 build) and C3 (Mistral-7B, half build).
Each shape is warmed up, then timed with CUDA events over at least --seconds of back-to-back launches.  Prints
one JSON line per shape (TFLOP/s of both, and the library's fraction of cuBLAS) after one line naming the card,
its power limit and SM clocks (read-only nvidia-smi query)."""
import argparse, json, math, subprocess, sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

# (config, name, M, N, K, epilogue name, dtype name); SwiGLU's N counts the interleaved gate and up rows
SHAPES = [('C2', 'qkv', 512 * 512, 2304, 768, 'BIAS', 'bf16'), ('C2', 'attn_out', 512 * 512, 768, 768, 'BIAS', 'bf16'),
          ('C2', 'ffn_up', 512 * 512, 3072, 768, 'BIAS_GELU', 'bf16'), ('C2', 'ffn_down', 512 * 512, 768, 3072, 'BIAS', 'bf16'),
          ('C5', 'qkv', 64 * 1026, 3840, 1280, 'BIAS', 'bf16'), ('C5', 'attn_out', 64 * 1026, 1280, 1280, 'BIAS', 'bf16'),
          ('C5', 'ffn_up', 64 * 1026, 5120, 1280, 'BIAS_GELU', 'bf16'), ('C5', 'ffn_down', 64 * 1026, 1280, 5120, 'BIAS', 'bf16'),
          ('C3', 'qkv', 16 * 4096, 6144, 4096, 'BIAS', 'f16'), ('C3', 'o_proj', 16 * 4096, 4096, 4096, 'BIAS', 'f16'),
          ('C3', 'gate_up', 16 * 4096, 28672, 4096, 'SWIGLU', 'f16'), ('C3', 'down', 16 * 4096, 4096, 14336, 'BIAS', 'f16')]


def timed(fn, seconds: float) -> float:
    """ms per call: warm-up, a short run to size the window, then >= `seconds` of launches between two events."""
    import torch
    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); [fn() for _ in range(10)]; e1.record(); torch.cuda.synchronize()
    reps = max(20, math.ceil(seconds * 1e3 / (e0.elapsed_time(e1) / 10)))
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--seconds', type=float, default=0.5, help='timed window per shape and kernel (default 0.5)')
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from distllm_b200 import _native as nv
    if not torch.cuda.is_available():
        raise SystemExit('bench_gemm.py needs a CUDA device')
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader',
                        '-i', '0'], capture_output=True, text=True).stdout.strip()
    print(json.dumps({'device': torch.cuda.get_device_name(dev), 'power_limit, clocks.sm, clocks.max.sm': q}), flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    for cfg, name, m, n, k, epi, dt in SHAPES:
        dtype = torch.bfloat16 if dt == 'bf16' else torch.float16
        a = (torch.randn(m, k, device=dev, generator=g) * 0.5).to(dtype)
        w = (torch.randn(n, k, device=dev, generator=g) * 0.02).to(dtype)
        bias = None if epi == 'SWIGLU' else torch.zeros(n, device=dev)
        code = getattr(nv, f'EPI_{epi}')
        ms = timed(lambda: nv.gemm_h16(a, w, bias, None, code), args.seconds)
        bias_h = None if bias is None else bias.to(dtype)
        ms_ref = timed(lambda: F.linear(a, w, bias_h), args.seconds)
        tf, tf_ref = 2.0 * m * n * k / ms / 1e9, 2.0 * m * n * k / ms_ref / 1e9
        print(json.dumps({'config': cfg, 'gemm': name, 'M': m, 'N': n, 'K': k, 'epilogue': epi, 'dtype': dt,
                          'ms': round(ms, 4), 'tflops': round(tf, 1), 'cublas_ms': round(ms_ref, 4),
                          'cublas_tflops': round(tf_ref, 1), 'frac_of_cublas': round(tf / tf_ref, 3)}), flush=True)
        del a, w, bias, bias_h
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
