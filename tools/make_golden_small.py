"""Generate tests/golden/bert_d32_golden.npz and esm_d32_golden.npz by running the UNMODIFIED reference on CPU.

The small encoders -- all-MiniLM-L6-v2 / bge-small-en-v1.5 / e5-small-v2 (BERT, H = 384, 12 heads x 32, I = 1536) and
esm2_t30_150M (ESM-2, H = 640, 20 heads x 32, I = 2560) -- at two layers.  The fixtures are made by
oracle/make_golden.py's own make_bert_golden / make_esm_golden, run with the shape dictionaries below in place of
TINY / TINY_ESM (same seeds, texts, batching, poolers) and writing into a temporary directory; the result is renamed.
oracle/ itself is not touched and the existing fixtures are not rewritten.

The ESM-2 fixture is kept small (a 640-wide hidden state of the first batch is 1.5 MB of incompressible floats):
- the same ten sequences in a different order, so that the first batch holds the four short ones -- 1, 7, 12 residues
  and the 33-residue row with two <mask> tokens (token dropout) -- and the 150-residue and the truncated 200-residue
  rows go to later batches (they still enter pooled/mean);
- the first batch's hidden state is stored at its attended positions only, as batch0/hidden_attended [tokens, H]
  (row-major over the attention mask; padded positions are never compared).

Run in the authoring container only (the reference tree does not exist on the GPU box):

    python tools/make_golden_small.py
"""

from __future__ import annotations

import shutil
import sys
import tempfile
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
GOLDEN = REPO / 'tests' / 'golden'

# 2-layer BERT of the MiniLM / BGE-small / E5-small width; vocabulary, positions and seed as the tiny BERT fixture
BERT_D32 = dict(vocab_size=200, hidden_size=384, num_hidden_layers=2, num_attention_heads=12,
                intermediate_size=1536, max_position_embeddings=64, type_vocab_size=2,
                layer_norm_eps=1e-12, hidden_act='gelu', hidden_dropout_prob=0.0,
                attention_probs_dropout_prob=0.0, initializer_range=0.05)
# 2-layer ESM-2 of the esm2_t30_150M width: rotary positions, token dropout
ESM_D32 = dict(vocab_size=33, hidden_size=640, num_hidden_layers=2, num_attention_heads=20,
               intermediate_size=2560, max_position_embeddings=160, position_embedding_type='rotary',
               token_dropout=True, mask_token_id=32, pad_token_id=1, layer_norm_eps=1e-5,
               emb_layer_norm_before=False, hidden_dropout_prob=0.0,
               attention_probs_dropout_prob=0.0, initializer_range=0.05)
# order of oracle/make_golden.tiny_esm_seqs() in the ESM-2 fixture: lengths 1, 7, 33 (+2 <mask>), 12 first
ESM_D32_ORDER = [3, 7, 2, 0, 1, 4, 5, 6, 8, 9]


def _attended_only(path: Path) -> None:
    """batch0/hidden [B, S, H] -> batch0/hidden_attended [tokens, H] at the attention mask's non-zero positions."""
    with np.load(path) as z:
        out = {k: z[k] for k in z.files}
    hidden = out.pop('batch0/hidden')
    out['batch0/hidden_attended'] = hidden[out['batch0/attention_mask'].astype(bool)]
    np.savez_compressed(path, **out)


def main() -> None:
    from oracle import make_golden as mg

    if not mg.REFERENCE.exists():
        raise SystemExit(f'{mg.REFERENCE} is not available: golden vectors can only be (re)generated in the '
                         'authoring container')
    sys.path.insert(0, str(mg.REFERENCE))
    import torch

    seqs = mg.tiny_esm_seqs
    fixtures = {
        'bert_d32_golden.npz': ('make_bert_golden', 'bert_tiny_golden.npz', {'TINY': BERT_D32}, None),
        'esm_d32_golden.npz': ('make_esm_golden', 'esm_tiny_golden.npz',
                               {'TINY_ESM': ESM_D32, 'tiny_esm_seqs': lambda: [seqs()[i] for i in ESM_D32_ORDER]},
                               _attended_only),
    }
    for name, (maker, made_as, patches, post) in fixtures.items():
        saved = {attr: getattr(mg, attr) for attr in [*patches, 'GOLDEN']}
        with tempfile.TemporaryDirectory() as tmp:
            try:
                for attr, value in patches.items():
                    setattr(mg, attr, value)
                mg.GOLDEN = Path(tmp)
                torch.manual_seed(0)
                getattr(mg, maker)()
            finally:
                for attr, value in saved.items():
                    setattr(mg, attr, value)
            if post is not None:
                post(Path(tmp) / made_as)
            shutil.move(str(Path(tmp) / made_as), GOLDEN / name)
        print(name, (GOLDEN / name).stat().st_size, 'bytes')


if __name__ == '__main__':
    sys.path.insert(0, str(REPO))
    main()
