"""ESM2-650M-shape throughput on one H100 (BASELINE config C5: 1024 residues -> S=1026, mean pooler).
Synthetic ids, seeded random weights.  Prints sequences/s and the fraction of the bf16 roofline."""
import json, sys, time
from pathlib import Path
import torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from transformers import EsmConfig
from distllm_b200 import _native as nv
from distllm_b200.embed.encoders.native import NativeEsm2Encoder
from distllm_b200.embed.encoders.weights import random_esm_state_dict

B, S = (int(sys.argv[1]) if len(sys.argv) > 1 else 64), 1026
cfg = EsmConfig(vocab_size=33, hidden_size=1280, num_hidden_layers=33, num_attention_heads=20,
                intermediate_size=5120, max_position_embeddings=1026, position_embedding_type='rotary',
                token_dropout=True, mask_token_id=32, pad_token_id=1, layer_norm_eps=1e-5,
                emb_layer_norm_before=False, initializer_range=0.02)
dev = torch.device('cuda:0')
enc = NativeEsm2Encoder(cfg, random_esm_state_dict(cfg, seed=0, device=dev), device=dev)
g = torch.Generator().manual_seed(0)
ids = torch.randint(4, 24, (B, S), generator=g); ids[:, 0] = 0; ids[:, -1] = 2
ids = ids.to(dev); mask = torch.ones(B, S, dtype=torch.int64, device=dev)
out = torch.empty(B, 1280, device=dev)
for _ in range(3):
    enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_REF, False, out=out)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
steps = 5
e0.record()
for _ in range(steps):
    enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_REF, False, out=out)
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
H, I, L = 1280, 5120, 33
flops = L * (8.0 * S * H * H + 4.0 * S * H * I + 4.0 * S * S * H)
seqs = B / (ms * 1e-3)
peaks = json.loads((Path(__file__).resolve().parents[1] / 'MEASURED_PEAKS.json').read_text()) if (Path(__file__).resolve().parents[1] / 'MEASURED_PEAKS.json').exists() else {'bf16_tflops_sustained': 1400.0}
print(json.dumps({'workload': 'C5: ESM2-650M shape, S=1026, mean pooler', 'batch': B, 'ms_per_step': ms,
                  'sequences_per_s': seqs, 'tflops': seqs * flops / 1e12,
                  'frac_of_sustained_bf16': seqs * flops / 1e12 / peaks['bf16_tflops_sustained']}))
enc.close()
