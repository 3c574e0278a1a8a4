"""Exact inner-product top-k over a device-resident embedding matrix (retrieval query path): time per
search and achieved HBM bandwidth (algorithmic bytes = one read of the corpus per query tile of 16).
Both scans for a float32 corpus: "fma" = b2e_topk_ip (CUDA cores), "tf32" = b2e_topk_ip_tc (tensor-core scan +
exact fp32 decision; results checked equal to the first on every configuration).
usage: bench_topk.py [N] [H]"""
import json, sys
from pathlib import Path
import torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from distllm_b200 import _native as nv
N = int(sys.argv[1]) if len(sys.argv) > 1 else 2_000_000
H = int(sys.argv[2]) if len(sys.argv) > 2 else 768
dev = torch.device('cuda:0')
pk = Path(__file__).resolve().parents[1] / 'MEASURED_PEAKS.json'
hbm = json.loads(pk.read_text()).get('hbm_gbs', 3350.0) if pk.exists() else 3350.0   # H100 SXM data sheet
g = torch.Generator(device=dev).manual_seed(0)
for dtype in (torch.float32, torch.bfloat16):
    corpus = torch.randn(N, H, device=dev, generator=g)
    corpus = (corpus / corpus.norm(dim=1, keepdim=True)).to(dtype).contiguous()
    for q, k in [(1, 10), (4, 10), (16, 10), (16, 100), (64, 10)]:
        queries = torch.randn(q, H, device=dev, generator=g)
        queries = queries / queries.norm(dim=1, keepdim=True)
        ref = None
        for scan in (('fma', 'tf32') if dtype == torch.float32 else ('fma',)):
            kw = {'max_norm': 1.0001} if scan == 'tf32' else {}
            for _ in range(2): out = nv.topk_ip(queries, corpus, k, **kw)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5): nv.topk_ip(queries, corpus, k, **kw)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            passes = (q + 15) // 16
            gbs = passes * N * H * corpus.element_size() / ms / 1e6
            rec = {'N': N, 'H': H, 'corpus': str(dtype).split('.')[-1], 'scan': scan, 'queries': q, 'k': k,
                   'ms': round(ms, 3), 'queries_per_s': round(q / ms * 1e3, 1), 'corpus_GBps': round(gbs, 1),
                   'frac_of_hbm': round(gbs / hbm, 3)}
            if scan == 'fma':
                ref = out
            else:
                rec['fell_back'] = nv.topk_tc_fell_back()
                rec['same_indices_as_fma'] = round((out[1] == ref[1]).float().mean().item(), 5)
                rec['max_score_diff'] = float((out[0] - ref[0]).abs().max())
            print(json.dumps(rec), flush=True)
    del corpus

# ---- the reference's binary branch (search.py:34-56, :202-336): packed sign bits, Hamming top-(k * multiplier), rescoring
corpus = torch.randn(N, H, device=dev, generator=g)
bits = nv.pack_ubinary(corpus.contiguous())
del corpus
for q, k, mult in [(1, 10, 2), (16, 10, 2), (16, 100, 2), (64, 10, 4)]:
    queries = torch.randn(q, H, device=dev, generator=g)
    for _ in range(2): nv.search_ubinary(queries, bits, k, mult)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5): nv.search_ubinary(queries, bits, k, mult)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    passes = (q + 7) // 8
    gbs = 2 * passes * N * (H // 8) / ms / 1e6     # histogram pass + select pass per tile of 8 queries
    print(json.dumps({'N': N, 'H': H, 'corpus': 'ubinary', 'queries': q, 'k': k, 'rescore_multiplier': mult,
                      'ms': round(ms, 3), 'queries_per_s': round(q / ms * 1e3, 1), 'packed_GBps': round(gbs, 1),
                      'frac_of_hbm': round(gbs / hbm, 3)}), flush=True)
