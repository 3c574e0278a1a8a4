"""Synthetic inputs for bench.py and the GPU tests: local HF checkpoint directories with seeded random
weights of the real shapes (no checkpoint can be downloaded here) and text files whose rows tokenise to
an exact number of tokens.  Uses transformers only -- nothing of distllm_b200 and nothing of the
reference -- so that BOTH arms of the benchmark can load the very same checkpoint and files.
"""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

BERT_BASE = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2,
                 layer_norm_eps=1e-12, initializer_range=0.02)
N_SPECIAL = 5   # [PAD] [UNK] [CLS] [SEP] [MASK]


def vocab_words(vocab_size: int) -> list[str]:
    """Whole-word WordPiece tokens: every synthetic word is exactly one token."""
    return [f'w{i:05d}' for i in range(vocab_size - N_SPECIAL)]


def write_bert_checkpoint(ckpt_dir: Path, cfg: dict | None = None, seed: int = 0) -> Path:
    """``BertModel`` with HF's own initialisation under ``torch.manual_seed(seed)`` + a synthetic
    ``BertTokenizerFast`` vocabulary, saved with ``save_pretrained`` (what ``AutoModel.from_pretrained``
    / ``AutoTokenizer.from_pretrained`` read: distllm/embed/encoders/auto.py:59-71)."""
    from transformers import BertConfig
    from transformers import BertModel
    from transformers import BertTokenizerFast

    cfg = dict(BERT_BASE if cfg is None else cfg)
    ckpt_dir = Path(ckpt_dir)
    ckpt_dir.mkdir(parents=True, exist_ok=True)
    state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    model = BertModel(BertConfig(**cfg)).eval()
    torch.random.set_rng_state(state)
    # HF zero-initialises every bias and sets LayerNorm to (1, 0); give them small seeded values so that
    # the bias / gamma / beta paths carry information on both arms
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith('LayerNorm.weight'):
                p.add_(0.02 * torch.randn(p.shape, generator=g))
            elif name.endswith('.bias'):
                p.add_(0.02 * torch.randn(p.shape, generator=g))
    model.save_pretrained(ckpt_dir)
    vocab = ['[PAD]', '[UNK]', '[CLS]', '[SEP]', '[MASK]', *vocab_words(cfg['vocab_size'])]
    (ckpt_dir / 'vocab.txt').write_text('\n'.join(vocab) + '\n')
    tok = BertTokenizerFast(vocab=str(ckpt_dir / 'vocab.txt'), do_lower_case=False)
    probe = tok('w00000 w00001')['input_ids']
    if tok.unk_token_id in probe or len(probe) != 4:   # transformers >= 5 ignores the old `vocab_file=` keyword
        raise RuntimeError(f'synthetic vocabulary not loaded: {probe}')
    tok.save_pretrained(ckpt_dir)
    return ckpt_dir


def write_token_rows(path: Path, n_rows: int, n_tokens, vocab_size: int, seed: int = 0,
                     with_path: bool = False) -> Path:
    """jsonl file, one ``{"text": ...}`` row per chunk; a row tokenises to exactly ``n_tokens`` tokens
    ([CLS] + words + [SEP]).  ``n_tokens``: int, or a (lo, hi) pair for lengths ~ U{lo..hi}."""
    rng = np.random.default_rng(seed)
    words = np.array(vocab_words(vocab_size))
    if isinstance(n_tokens, int):
        lengths = np.full(n_rows, n_tokens)
    else:
        lengths = rng.integers(n_tokens[0], n_tokens[1] + 1, size=n_rows)
    with open(path, 'w') as f:
        for i, n in enumerate(lengths):
            row = {'text': ' '.join(words[rng.integers(0, len(words), size=int(n) - 2)])}
            if with_path:
                row['path'] = f'row{i}'
            f.write(json.dumps(row) + '\n')
    return Path(path)


def write_semantic_docs(path: Path, n_docs: int, n_sentences: int, vocab_size: int, seed: int = 0,
                        words_lo: int = 40, words_hi: int = 80) -> Path:
    """jsonl documents for ``jsonl_chunk`` + ``semantic_chunk``: sentences of 40-80 words ending in ". "
    followed by a capital (any sentence splitter cuts them identically), so that buffers and chunks clear
    the 750-character filters (distllm/embed/datasets/jsonl_chunk.py:78-85, semantic_chunk.py:224)."""
    rng = np.random.default_rng(seed)
    words = np.array(vocab_words(vocab_size))
    with open(path, 'w') as f:
        for d in range(n_docs):
            sents = ['S' + ' '.join(words[rng.integers(0, len(words), size=int(rng.integers(words_lo, words_hi + 1)))])
                     + '. ' for _ in range(n_sentences)]
            f.write(json.dumps({'text': ''.join(sents), 'path': f'doc{d}'}) + '\n')
    return Path(path)


# ------------------------------------------------------------------------------- outlier weights
# Trained checkpoints are not N(0, 0.02): a handful of hidden channels carry values tens of times larger
# than the rest and the LayerNorm / RMSNorm gains spread over orders of magnitude.  The parity tests run
# every family on such weights too (VERDICT r1 weak #2).

_OUT_ROWS = {
    'bert': ('attention.output.dense.weight', 'output.dense.weight'),
    'esm': ('attention.output.dense.weight', 'output.dense.weight'),
    'mistral': ('self_attn.o_proj.weight', 'mlp.down_proj.weight'),
    'qwen3': ('self_attn.o_proj.weight', 'mlp.down_proj.weight'),
    'modernbert': ('attn.Wo.weight', 'mlp.Wo.weight'),
}


def add_outliers(state_dict: dict, family: str, seed: int = 0, n_massive: int = 4, scale: float = 50.0,
                 n_loud: int = 8, loud_gain: float = 10.0, gain_range: tuple[float, float] = (0.5, 2.0),
                 massive_gain: float = 0.05) -> dict:
    """In place, on HF state-dict names of BertModel / EsmModel / MistralModel (any device / dtype):

      * MASSIVE channels: the rows of every block-output projection (attention output and FFN-down) that write
        ``n_massive`` fixed hidden channels are multiplied by ``scale``, so those channels of the residual
        stream are ~50x the rest and dominate every norm statistic; like trained checkpoints, the norm gains
        of those channels are small (``massive_gain``);
      * LOUD channels: ``n_loud`` other channels get a norm gain of ``loud_gain`` (= 10);
      * every other norm gain is log-uniform in ``gain_range``, every norm bias N(0, 0.5).

    (A first version drew EVERY gain from [0.1, 10]: with all q/k inputs up to 10x larger the attention
    logits grow ~100x, softmax turns into an arg-max, and the fp32 network itself becomes discontinuous in
    its inputs -- any 16-bit implementation then flips keys at random tokens.)

    Qwen3's per-head q_norm / k_norm gains ([head_dim], applied right before the attention logits) take no part
    in the hidden-channel draws above; for the same reason they get log-uniform gains in ``gain_range`` only,
    from a generator of their own, so the other families' weights are drawn exactly as before."""
    g = torch.Generator().manual_seed(seed)
    out_names = _OUT_ROWS[family]
    hidden = next(v.shape[0] for k, v in state_dict.items() if k.endswith(out_names[0]))
    perm = torch.randperm(hidden, generator=g)
    massive, loud = perm[:n_massive], perm[n_massive:n_massive + n_loud]
    lo, hi = float(np.log(gain_range[0])), float(np.log(gain_range[1]))
    head_norms = ('self_attn.q_norm.weight', 'self_attn.k_norm.weight') if family == 'qwen3' else ()
    for name, t in state_dict.items():
        if head_norms and name.endswith(head_norms):
            continue
        if name.endswith(out_names):
            t[massive.to(t.device)] *= scale
        elif t.dim() == 1 and ('LayerNorm.weight' in name or 'layer_norm_after.weight' in name
                               or name.endswith('layernorm.weight') or name == 'norm.weight'
                               or name.endswith('_norm.weight') or name.endswith('.norm.weight')):
            gain = torch.exp(torch.rand(t.shape, generator=g) * (hi - lo) + lo)
            gain[massive] = massive_gain
            gain[loud] = loud_gain
            t.copy_(gain.to(device=t.device, dtype=t.dtype))
        elif t.dim() == 1 and ('LayerNorm.bias' in name or 'layer_norm_after.bias' in name):
            t.copy_((0.5 * torch.randn(t.shape, generator=g)).to(device=t.device, dtype=t.dtype))
    if head_norms:
        g_head = torch.Generator().manual_seed(seed + 1)
        for name, t in state_dict.items():
            if name.endswith(head_norms):
                gain = torch.exp(torch.rand(t.shape, generator=g_head) * (hi - lo) + lo)
                t.copy_(gain.to(device=t.device, dtype=t.dtype))
    return state_dict
