"""End-to-end `embedding_worker` on one H100 with the HOST FEED included: synthetic jsonl documents ->
sentence split -> buffers -> HF fast tokenizer in DataLoader workers -> native encoder -> semantic
chunking -> second pass -> numpy writer (SURVEY 8(f) rank 1: where does the time go once the encoder
runs near the roofline?).  BERT-base shape, seeded random weights saved as a local HF checkpoint.
usage: bench_worker_e2e.py [n_docs] [sentences_per_doc] [batch_size] [num_data_workers]"""
import json, sys, tempfile, time
from pathlib import Path
import numpy as np
import torch
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from transformers import BertConfig, BertModel, BertTokenizerFast
from distllm_b200.distributed_embedding import embedding_worker
from distllm_b200.embed.encoders.weights import random_bert_state_dict

n_docs = int(sys.argv[1]) if len(sys.argv) > 1 else 40
n_sent = int(sys.argv[2]) if len(sys.argv) > 2 else 30
batch = int(sys.argv[3]) if len(sys.argv) > 3 else 512
workers = int(sys.argv[4]) if len(sys.argv) > 4 else 4
rng = np.random.default_rng(0)
words = [f'w{i:04d}' for i in range(2000)]
with tempfile.TemporaryDirectory() as tmp:
    tmp = Path(tmp)
    cfg = BertConfig(vocab_size=2005, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                     intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
    model = BertModel(cfg)
    model.load_state_dict(random_bert_state_dict(cfg, seed=0), strict=False)
    (tmp / 'vocab.txt').write_text('\n'.join(['[PAD]', '[UNK]', '[CLS]', '[SEP]', '[MASK]', *words]) + '\n')
    model.save_pretrained(tmp / 'ckpt')
    BertTokenizerFast(vocab=str(tmp / 'vocab.txt'), do_lower_case=False).save_pretrained(tmp / 'ckpt')
    del model
    docs = []
    for d in range(n_docs):
        sents = ['S' + ' '.join(rng.choice(words, size=rng.integers(40, 81))) + '. ' for _ in range(n_sent)]
        docs.append({'text': ''.join(sents), 'path': f'doc{d}'})
    (tmp / 'in').mkdir()
    f = tmp / 'in' / 'docs.jsonl'
    f.write_text('\n'.join(json.dumps(d) for d in docs))
    kwargs = dict(
        dataset_kwargs={'name': 'jsonl_chunk', 'buffer_size': 4, 'batch_size': batch, 'num_data_workers': workers},
        encoder_kwargs={'name': 'auto', 'pretrained_model_name_or_path': str(tmp / 'ckpt'), 'quantization': False},
        pooler_kwargs={'name': 'mean'},
        embedder_kwargs={'name': 'semantic_chunk', 'chunk_batch_size': batch},
        writer_kwargs={'name': 'numpy'},
    )
    for rep in range(2):   # the second file reuses the registered encoder (warm start), like the reference
        t0 = time.perf_counter()
        embedding_worker(f, tmp / f'out{rep}', **kwargs)
        dt = time.perf_counter() - t0
        out = next((tmp / f'out{rep}').glob('*/embeddings.npy'))
        emb = np.load(out)
        n_buffers = n_docs * n_sent
        print(json.dumps({'rep': rep, 'seconds': dt, 'pass1_buffers': n_buffers, 'final_chunks': int(emb.shape[0]),
                          'encoder_rows_per_s_overall': (n_buffers + emb.shape[0]) / dt,
                          'batch_size': batch, 'num_data_workers': workers}), flush=True)
