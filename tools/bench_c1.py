"""BASELINE config C1 on one H100: BERT-base shape, mean pooler, batch_size=8, 1000 chunks of 128 tokens,
through the host-buffer C-ABI call (b2e_embed_host: H2D + 91 launches + D2H per batch of 8).
The small-batch regime is launch-bound; the number is reported for completeness next to C2.
usage: bench_c1.py [batch] [seq] [n_chunks]"""
import json, sys, time
from pathlib import Path
import torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from transformers import BertConfig
from distllm_b200 import _native as nv
from distllm_b200.embed.encoders.native import NativeBertEncoder
from distllm_b200.embed.encoders.weights import random_bert_state_dict

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
S = int(sys.argv[2]) if len(sys.argv) > 2 else 128
N = int(sys.argv[3]) if len(sys.argv) > 3 else 1000
cfg = BertConfig(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
dev = torch.device('cuda:0')
enc = NativeBertEncoder(cfg, random_bert_state_dict(cfg, seed=0, device=dev), device=dev)
g = torch.Generator().manual_seed(0)
ids = torch.randint(7, 30522, (N, S), generator=g); ids[:, 0] = 101; ids[:, -1] = 102
mask = torch.ones(N, S, dtype=torch.int64); types = torch.zeros(N, S, dtype=torch.int64)
ids, mask, types = ids.pin_memory(), mask.pin_memory(), types.pin_memory()
out = torch.empty(N, 768).pin_memory()
enc.embed_host(ids[:B * 4], mask[:B * 4], types[:B * 4], B, nv.POOL_MEAN_REF, False, out=out[:B * 4])
best = 1e9
for _ in range(3):
    t0 = time.perf_counter()
    enc.embed_host(ids, mask, types, B, nv.POOL_MEAN_REF, False, out=out)
    best = min(best, time.perf_counter() - t0)
flops = 12 * (8.0 * S * 768 * 768 + 4.0 * S * 768 * 3072 + 4.0 * S * S * 768)
print(json.dumps({'workload': f'C1: BERT-base shape, mean pooler, batch_size={B}, {N} chunks of {S} tokens, host buffers',
                  'chunks_per_s': N / best, 'ms_per_batch': 1e3 * best / ((N + B - 1) // B),
                  'tflops': N / best * flops / 1e12}))
enc.close()
