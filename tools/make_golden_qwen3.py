"""Generate tests/golden/qwen3_tiny_golden.npz by running the UNMODIFIED reference on CPU.

The reference's AutoEncoder (``AutoModel.from_pretrained(..., trust_remote_code=True)`` -> HF ``Qwen3Model``) with
its LastTokenPooler / MeanPooler and compute_embeddings (distllm/embed/embedders/full_sequence.py) on a tiny seeded
Qwen3 checkpoint saved with ``save_pretrained`` plus a WordLevel tokenizer: 4 layers, H = 256, 4 q heads and 2 kv
heads of 128 (so the attention width, 512, differs from H), I = 384, rope_theta 1e6, eps 1e-6, 512 positions.
The Mistral fixture's texts (oracle/make_golden.tiny_mistral_texts: 1 to 400 words) plus one of 600 words that is
truncated to 512 tokens, batches of 4, right and left padding:

    {right,left}/batch{i}/input_ids, attention_mask     the reference's token batches
    {right,left}/pooled/last_token                      LastTokenPooler rows
    right/pooled/mean_normalized                        MeanPooler rows, L2-normalised
    right/batch0/hidden_attended                        batch 0's last hidden state at its attended positions
                                                        ([tokens, H], row-major over the mask: keeps the file small)

Run in the authoring container only (the reference tree does not exist on the GPU box):

    python tools/make_golden_qwen3.py
"""

from __future__ import annotations

import sys
import tempfile
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
GOLDEN = REPO / 'tests' / 'golden'

TINY_QWEN3 = dict(vocab_size=320, hidden_size=256, num_hidden_layers=4, num_attention_heads=4,
                  num_key_value_heads=2, head_dim=128, intermediate_size=384, max_position_embeddings=512,
                  rms_norm_eps=1e-6, rope_parameters={'rope_type': 'default', 'rope_theta': 1e6},
                  hidden_act='silu', attention_bias=False, use_sliding_window=False, attention_dropout=0.0,
                  initializer_range=0.05, tie_word_embeddings=False, pad_token_id=0, bos_token_id=1,
                  eos_token_id=2)
TINY_QWEN3_SEED = 3579


def tiny_qwen3_texts() -> list[str]:
    """The Mistral fixture's 12 texts and a 600-word one (truncated to 512 tokens)."""
    from oracle.make_golden import tiny_mistral_texts

    rng = np.random.default_rng(31)
    words = [f'w{i:03d}' for i in range(TINY_QWEN3['vocab_size'] - 4)]
    return [*tiny_mistral_texts(), ' '.join(rng.choice(words, size=600))]


def tiny_qwen3_config():
    from transformers import Qwen3Config

    return Qwen3Config(**TINY_QWEN3)


def write_tiny_qwen3_checkpoint(ckpt_dir: Path) -> Path:
    """The seeded checkpoint (random_qwen3_state_dict) and its WordLevel tokenizer, saved with save_pretrained."""
    from tokenizers import Tokenizer
    from tokenizers.models import WordLevel
    from tokenizers.pre_tokenizers import Whitespace
    from tokenizers.processors import TemplateProcessing
    from transformers import PreTrainedTokenizerFast
    from transformers import Qwen3Model

    from distllm_b200.embed.encoders.weights import random_qwen3_state_dict

    words = [f'w{i:03d}' for i in range(TINY_QWEN3['vocab_size'] - 4)]
    vocab = {t: i for i, t in enumerate(['<pad>', '<s>', '</s>', '<unk>', *words])}
    cfg = tiny_qwen3_config()
    sd = random_qwen3_state_dict(cfg, seed=TINY_QWEN3_SEED, device='cpu')
    model = Qwen3Model(cfg)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all('rotary_emb' in k for k in missing), (missing, unexpected)
    raw = Tokenizer(WordLevel(vocab, unk_token='<unk>'))
    raw.pre_tokenizer = Whitespace()
    raw.post_processor = TemplateProcessing(single='<s> $A', special_tokens=[('<s>', 1)])
    tok = PreTrainedTokenizerFast(tokenizer_object=raw, pad_token='<pad>', bos_token='<s>',
                                  eos_token='</s>', unk_token='<unk>')
    model.eval().save_pretrained(ckpt_dir)
    tok.save_pretrained(ckpt_dir)
    return Path(ckpt_dir)


def make_qwen3_golden() -> None:
    import torch
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
    from distllm_b200.embed.encoders.weights import random_qwen3_state_dict
    from oracle.make_golden import weights_digest

    texts = tiny_qwen3_texts()
    out = {'n_texts': np.array(len(texts)),
           'weights_sha256': np.array(weights_digest(
               random_qwen3_state_dict(tiny_qwen3_config(), seed=TINY_QWEN3_SEED, device='cpu')))}
    with tempfile.TemporaryDirectory() as tmp:
        ckpt = write_tiny_qwen3_checkpoint(Path(tmp) / 'ckpt')
        encoder = AutoEncoder(AutoEncoderConfig(pretrained_model_name_or_path=str(ckpt), quantization=False,
                                                eval_mode=True))
        assert type(encoder.model).__name__ == 'Qwen3Model'
        assert encoder.tokenizer.model_max_length == TINY_QWEN3['max_position_embeddings']

        def loader() -> DataLoader:
            return DataLoader(InMemoryDataset(texts), batch_size=4, num_workers=0,
                              collate_fn=DataCollator(encoder.tokenizer))

        for side in ('right', 'left'):
            encoder.tokenizer.padding_side = side
            for i, batch in enumerate(loader()):
                out[f'{side}/batch{i}/input_ids'] = batch['input_ids'].numpy()
                out[f'{side}/batch{i}/attention_mask'] = batch['attention_mask'].numpy()
                assert 'token_type_ids' not in batch
                if i == 0 and side == 'right':
                    with torch.no_grad():
                        hidden = encoder.encode(batch).numpy()
                    out['right/batch0/hidden_attended'] = hidden[batch['attention_mask'].numpy().astype(bool)]
            out['n_batches'] = np.array(i + 1)
            out[f'{side}/pooled/last_token'] = compute_embeddings(
                loader(), encoder, LastTokenPooler(LastTokenPoolerConfig()))
            if side == 'right':
                out['right/pooled/mean_normalized'] = compute_embeddings(
                    loader(), encoder, MeanPooler(MeanPoolerConfig()), normalize=True)
    assert max(out[f'right/batch{i}/input_ids'].shape[1] for i in range(int(out['n_batches']))) == 512
    np.savez_compressed(GOLDEN / 'qwen3_tiny_golden.npz', **out)


def main() -> None:
    from oracle import make_golden as mg

    if not mg.REFERENCE.exists():
        raise SystemExit(f'{mg.REFERENCE} is not available: golden vectors can only be (re)generated in the '
                         'authoring container')
    sys.path.insert(0, str(mg.REFERENCE))
    import torch

    torch.manual_seed(0)
    make_qwen3_golden()
    path = GOLDEN / 'qwen3_tiny_golden.npz'
    print(path.name, path.stat().st_size, 'bytes')


if __name__ == '__main__':
    sys.path.insert(0, str(REPO))
    main()
