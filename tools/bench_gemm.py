"""The library's GEMM (nv.gemm_h16) against torch.nn.functional.linear (cuBLAS, a ceiling only) at every GEMM shape
bench.py runs: C2 (BERT-base, bfloat16 build), C5 (ESM-2 650M, bfloat16 build) and C3 (Mistral-7B, half build).
Where the 192-wide tiles exist for a shape, both tile widths are timed (b2e_debug_set_gemm_bn), alternating over
--rounds rounds, and the width the library picks by default is named.  Each timing is warmed up, then taken with
CUDA events over at least --seconds of back-to-back launches.  Prints one JSON line per shape (TFLOP/s of each
width and of cuBLAS, the library's fraction of cuBLAS) after one line naming the card, its power limit and SM
clocks (read-only nvidia-smi query)."""
import argparse, ctypes, json, math, subprocess, sys
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
    ap.add_argument('--rounds', type=int, default=3, help='alternations of the two tile widths (default 3)')
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
        lib = nv.load(dt)
        lib.b2e_debug_set_gemm_bn.argtypes = [ctypes.c_int]
        picked, wide = ctypes.c_int(), ctypes.c_int()
        nv.check(lib.b2e_debug_gemm_bn(n, code, 0, ctypes.byref(picked)), lib)   # the default rule
        nv.check(lib.b2e_debug_set_gemm_bn(192), lib)
        nv.check(lib.b2e_debug_gemm_bn(n, code, 0, ctypes.byref(wide)), lib)     # does a 192-wide kernel exist
        widths = (128, 192) if wide.value == 192 else (128,)
        runs = {bn: [] for bn in widths}
        for _ in range(args.rounds if len(widths) > 1 else 1):
            for bn in widths:
                nv.check(lib.b2e_debug_set_gemm_bn(bn), lib)   # the W map of every call below is built at this width
                runs[bn].append(timed(lambda: nv.gemm_h16(a, w, bias, None, code), args.seconds))
        lib.b2e_debug_set_gemm_bn(0)
        ms = min(runs[picked.value])
        bias_h = None if bias is None else bias.to(dtype)
        ms_ref = timed(lambda: F.linear(a, w, bias_h), args.seconds)
        tf, tf_ref = 2.0 * m * n * k / ms / 1e9, 2.0 * m * n * k / ms_ref / 1e9
        line = {'config': cfg, 'gemm': name, 'M': m, 'N': n, 'K': k, 'epilogue': epi, 'dtype': dt,
                'default_bn': picked.value, 'ms': round(ms, 4), 'tflops': round(tf, 1)}
        for bn, t in runs.items():
            line[f'bn{bn}_ms'] = [round(x, 4) for x in t]
            line[f'bn{bn}_tflops'] = round(2.0 * m * n * k / min(t) / 1e9, 1)
        line.update({'cublas_ms': round(ms_ref, 4), 'cublas_tflops': round(tf_ref, 1),
                     'frac_of_cublas': round(tf / tf_ref, 3)})
        print(json.dumps(line), flush=True)
        del a, w, bias, bias_h
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
