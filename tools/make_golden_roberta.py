"""Generate tests/golden/xlmr_tiny_golden.npz by running the UNMODIFIED reference on CPU.

The reference's own AutoEncoder, DataCollator, poolers and compute_embeddings (distllm/embed/embedders/
full_sequence.py) on the tiny seeded XLM-RoBERTa checkpoint of tools/oracle_roberta.py, written to a temporary
directory with its SentencePiece-style fast tokenizer (<pad> = 1).  Two of the texts hold a literal <pad> inside the
attended text.  Recorded: the token batches, the first batch's last hidden state, and the pooled embeddings (mean,
mean + normalize, last token), right-padded as the tokenizer pads by default.

Every text is at most 62 tokens, so the reference's model_max_length of max_position_embeddings (66) and ours of
max_position_embeddings - pad_token_id - 1 (64) truncate nothing.

Run in the authoring container only (the reference tree does not exist on the GPU box):

    python tools/make_golden_roberta.py
"""

from __future__ import annotations

import sys
import tempfile
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
GOLDEN = REPO / 'tests' / 'golden'


def main() -> None:
    import torch

    from oracle import make_golden as mg

    if not mg.REFERENCE.exists():
        raise SystemExit(f'{mg.REFERENCE} is not available: golden vectors can only be (re)generated in the '
                         'authoring container')
    sys.path.insert(0, str(mg.REFERENCE))
    from torch.utils.data import DataLoader

    from distllm.embed.datasets.utils import DataCollator
    from distllm.embed.datasets.utils import InMemoryDataset
    from distllm.embed.embedders.full_sequence import compute_embeddings
    from distllm.embed.encoders.auto import AutoEncoder
    from distllm.embed.encoders.auto import AutoEncoderConfig
    from distllm.embed.poolers.last_token import LastTokenPooler
    from distllm.embed.poolers.last_token import LastTokenPoolerConfig
    from distllm.embed.poolers.mean import MeanPooler
    from distllm.embed.poolers.mean import MeanPoolerConfig
    from tools import oracle_roberta as O

    torch.manual_seed(0)
    _, sd = O.tiny_xlmr_state_dict()
    texts = O.tiny_xlmr_texts()
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = Path(tmp) / 'ckpt'
        O.write_tiny_xlmr_checkpoint(ckpt)
        encoder = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(ckpt), quantization=False,
                                                eval_mode=True))
        assert encoder.tokenizer.model_max_length == O.TINY_XLMR['max_position_embeddings']

        def loader() -> DataLoader:
            return DataLoader(InMemoryDataset(texts), batch_size=4, num_workers=0,
                              collate_fn=DataCollator(encoder.tokenizer))

        out = {'weights_sha256': np.array(mg.weights_digest(sd)), 'n_texts': np.array(len(texts))}
        for i, batch in enumerate(loader()):
            out[f'batch{i}/input_ids'] = batch['input_ids'].numpy()
            out[f'batch{i}/attention_mask'] = batch['attention_mask'].numpy()
            if i == 0:
                with torch.no_grad():
                    out['batch0/hidden'] = encoder.encode(batch).numpy()
        out['n_batches'] = np.array(i + 1)
        mean = MeanPooler(MeanPoolerConfig())
        last = LastTokenPooler(LastTokenPoolerConfig())
        out['pooled/mean'] = compute_embeddings(loader(), encoder, mean)
        out['pooled/mean_normalized'] = compute_embeddings(loader(), encoder, mean, normalize=True)
        out['pooled/last_token'] = compute_embeddings(loader(), encoder, last)
    np.savez_compressed(GOLDEN / 'xlmr_tiny_golden.npz', **out)
    print('xlmr_tiny_golden.npz', (GOLDEN / 'xlmr_tiny_golden.npz').stat().st_size, 'bytes')


if __name__ == '__main__':
    sys.path.insert(0, str(REPO))
    main()
