"""Mistral-7B-shape throughput on one H100 (BASELINE config C3: SFR-Embedding-Mistral shape, L=32,
H=4096, 32 query / 8 kv heads x 128, I=14336, last_token pooler, B=16, S=4096).
Synthetic ids, seeded random bf16 weights.  Prints sequences/s, the fraction of the bf16 roofline
(causal-skipped FLOPs, SURVEY 8d) and a per-kernel breakdown of one layer timed with CUDA events.
usage: bench_mistral.py [B] [S] [layers] [ragged]   (ragged: right-padded lengths ~ U{S/8..S}, first row full)"""
import json, sys
from pathlib import Path
import torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from transformers import MistralConfig
from distllm_b200 import _native as nv
from distllm_b200.embed.encoders.native import NativeMistralEncoder
from distllm_b200.embed.encoders.weights import interleave_gate_up, random_mistral_state_dict

B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
S = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
L = int(sys.argv[3]) if len(sys.argv) > 3 else 32
H, I, HEADS, KV = 4096, 14336, 32, 8
cfg = MistralConfig(vocab_size=32000, hidden_size=H, num_hidden_layers=L, num_attention_heads=HEADS,
                    num_key_value_heads=KV, head_dim=128, intermediate_size=I, max_position_embeddings=32768,
                    rms_norm_eps=1e-5, sliding_window=4096, initializer_range=0.02)
dev = torch.device('cuda:0')
sd = random_mistral_state_dict(cfg, seed=0, device=dev, dtype=torch.float16)
enc = NativeMistralEncoder(cfg, sd, device=dev)
del sd
torch.cuda.empty_cache()
g = torch.Generator().manual_seed(0)
ids = torch.randint(3, 32000, (B, S), generator=g).to(dev)
mask = torch.ones(B, S, dtype=torch.int64, device=dev)
RAGGED = len(sys.argv) > 4 and sys.argv[4] == 'ragged'
if RAGGED:
    lens = torch.randint(S // 8, S + 1, (B,), generator=g)
    lens[0] = S
    mask = (torch.arange(S)[None] < lens[:, None]).long().to(dev)
out = torch.empty(B, H, device=dev)
for _ in range(2):
    enc.encode_pooled(ids, mask, None, nv.POOL_LAST_TOKEN, True, out=out)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
steps = 3
e0.record()
for _ in range(steps):
    enc.encode_pooled(ids, mask, None, nv.POOL_LAST_TOKEN, True, out=out)
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
QC = (HEADS + 2 * KV) * 128
flops_dense = L * (2.0 * S * H * QC + 2.0 * S * H * H + 6.0 * S * H * I + 4.0 * S * S * H)
flops_causal = L * (2.0 * S * H * QC + 2.0 * S * H * H + 6.0 * S * H * I + 2.0 * S * (S + 128) * H)
seqs = B / (ms * 1e-3)
pk = Path(__file__).resolve().parents[1] / 'MEASURED_PEAKS.json'
peaks = json.loads(pk.read_text()) if pk.exists() else {}
sus = peaks.get('bf16_tflops_sustained', 989.0)   # H100 SXM data sheet, dense 16-bit
res = {'workload': f'C3: Mistral-7B shape (L={L}), S={S}, last_token pooler' + (' RAGGED' if RAGGED else ''), 'batch': B,
       'attended_tokens': int(mask.sum().item()), 'padded_tokens': B * S, 'ms_per_step': ms,
       'sequences_per_s': seqs, 'tflops_causal_skipped': seqs * flops_causal / 1e12,
       'frac_of_sustained_bf16': seqs * flops_causal / 1e12 / sus,
       'tflops_dense_counted': seqs * flops_dense / 1e12,
       'workspace_gb': enc.workspace_bytes(B, S) / 1e9}
enc.close()

# ---- one layer, kernel by kernel
def timeit(fn, reps=5):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps
M = B * S
x = torch.randn(M, H, device=dev).half()
wqkv = (torch.randn(QC, H, device=dev) * 0.02).half()
wo = (torch.randn(H, H, device=dev) * 0.02).half()
wgu = (torch.randn(2 * I, H, device=dev) * 0.02).half()
wd = (torch.randn(H, I, device=dev) * 0.02).half()
qkv = nv.gemm_h16(x, wqkv, None)
ffn = nv.gemm_h16(x, wgu, None, None, nv.EPI_SWIGLU)
parts = {
    'gemm_qkv': (timeit(lambda: nv.gemm_h16(x, wqkv, None)), 2.0 * M * H * QC),
    'attention_causal': (timeit(lambda: nv.attention_causal_d128(qkv, mask, B, S, HEADS, KV, 4096)),
                         2.0 * B * S * (S + 128) * H),
    'gemm_o': (timeit(lambda: nv.gemm_h16(x, wo, None)), 2.0 * M * H * H),
    'gemm_gate_up_swiglu': (timeit(lambda: nv.gemm_h16(x, wgu, None, None, nv.EPI_SWIGLU)), 4.0 * M * H * I),
    'gemm_down': (timeit(lambda: nv.gemm_h16(ffn, wd, None)), 2.0 * M * H * I),
}
res['layer_kernels'] = {k: {'ms': round(t, 3), 'tflops': round(f / t / 1e9, 1)} for k, (t, f) in parts.items()}
res['layer_kernels_sum_ms'] = round(sum(t for t, _ in parts.values()), 3)
print(json.dumps(res))
