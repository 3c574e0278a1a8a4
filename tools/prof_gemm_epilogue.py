"""How long the GEMM epilogue takes against the main loop, from the clock64 timeline of CTA 0 (the profiling
instantiation that runs while b2e_debug_set_clock_buffer is set), at the four C2 GEMM shapes (BERT-base, B 512,
S 512, bfloat16 build, seeded operands).

The timeline holds 4 x 256 int64 stamps: [0][n] the producer has issued the loads of the CTA's n-th k-block (it
waits for a free stage first, so these follow the consumers' pace), [1][n] consumer 0 has retired its n-th k-block,
[2][e] and [3][e] consumer 0's epilogue of its e-th tile (the CTA's turn 2e) starts (accumulators final) and ends
(TMA store issued).  Per shape, medians over consumer 0's tiles, in SM cycles:
  epilogue       [3][e] - [2][e]
  main_loop      consumer 0's main loop: its first to last k-block retirement of a tile ([1]), times
                 kblocks / (kblocks - 1)
  turn_pair      [2][e + 1] - [2][e]: two turns, one per consumer; 2 x main_loop if the tensor cores never wait
  handover_idle  turn_pair - 2 x main_loop: what the two hand-overs add to the pair of main loops
Prints one JSON line naming the card and its power limit (read-only nvidia-smi query), then one per shape."""
import ctypes, json, statistics, subprocess, sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

M = 512 * 512
SHAPES = [('qkv', 2304, 768, 'BIAS'), ('attn_out', 768, 768, 'BIAS'), ('ffn_up', 3072, 768, 'BIAS_GELU'),
          ('ffn_down', 768, 3072, 'BIAS')]


def main() -> None:
    import torch
    from distllm_b200 import _native as nv
    if not torch.cuda.is_available():
        raise SystemExit('prof_gemm_epilogue.py needs a CUDA device')
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader',
                        '-i', '0'], capture_output=True, text=True).stdout.strip()
    print(json.dumps({'device': torch.cuda.get_device_name(dev), 'name, power_limit, clocks.sm, clocks.max.sm': q}),
          flush=True)
    lib = nv.load('bf16')
    lib.b2e_debug_set_clock_buffer.argtypes = [ctypes.c_void_p]
    g = torch.Generator(device=dev).manual_seed(0)
    for name, n, k, epi in SHAPES:
        a = (torch.randn(M, k, device=dev, generator=g) * 0.5).to(torch.bfloat16)
        w = (torch.randn(n, k, device=dev, generator=g) * 0.02).to(torch.bfloat16)
        bias = torch.randn(n, device=dev, generator=g)
        code = getattr(nv, f'EPI_{epi}')
        buf = torch.zeros(4, 256, dtype=torch.int64, device=dev)
        try:
            nv.check(lib.b2e_debug_set_clock_buffer(buf.data_ptr()), lib)
            for _ in range(3):   # warm: the last launch's stamps are kept
                nv.gemm_h16(a, w, bias, None, code)
            torch.cuda.synchronize()
        finally:
            nv.check(lib.b2e_debug_set_clock_buffer(None), lib)
        s = buf.cpu().tolist()
        kb = k // 64
        ret = [x for x in s[1] if x]
        main_loop = statistics.median((ret[(e + 1) * kb - 1] - ret[e * kb]) * kb / (kb - 1)
                                      for e in range(len(ret) // kb))
        start, end = [x for x in s[2] if x], [x for x in s[3] if x]
        tiles = min(len(start), len(end))
        epi_cyc = statistics.median(end[e] - start[e] for e in range(tiles))
        pair = statistics.median(start[e + 1] - start[e] for e in range(tiles - 1))
        print(json.dumps({'gemm': name, 'M': M, 'N': n, 'K': k, 'epilogue': epi, 'kblocks': kb,
                          'tiles_stamped': tiles, 'epilogue_cycles': epi_cyc, 'main_loop_cycles': round(main_loop),
                          'cycles_per_kblock': round(main_loop / kb, 1), 'turn_pair_cycles': pair,
                          'handover_idle_cycles': round(pair - 2 * main_loop)}), flush=True)


if __name__ == '__main__':
    main()
