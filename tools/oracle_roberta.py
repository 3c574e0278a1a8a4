"""fp32 CPU restatement of the forward pass the reference runs for RoBERTa / XLM-RoBERTa checkpoints, and the tiny
seeded checkpoint behind tests/golden/xlmr_tiny_golden.npz.

``XLMRobertaModel`` (transformers/models/xlm_roberta/modeling_xlm_roberta.py, and the same in ``roberta``) is BERT's
model with one change in the embedding step: position ids come from ``create_position_ids_from_input_ids``,

    m = input_ids != padding_idx
    pos = cumsum(m, dim=1) * m + padding_idx

so the first non-pad token reads row padding_idx + 1, a pad id reads row padding_idx and does not advance the count,
and left padding starts the count at the first non-pad token.  The embedding sum is (word + token_type) + position.

:func:`roberta_forward` runs oracle/bert.py's ``bert_forward`` unchanged on a rewritten state dict: one token-type row
per token holding ``position[pos]``, the per-token ``word + token_type`` rows as the word table, and a zero position
table.  Its first addition then is HF's second one, and the zero rows add nothing, so the sum is HF's, rounding for
rounding.  No transformers model is on this path.  TEST INFRASTRUCTURE ONLY.
"""

from __future__ import annotations

from pathlib import Path
from typing import Mapping

import numpy as np
import torch

from oracle.bert import bert_forward

# the tiny XLM-R checkpoint of the golden vectors: <pad> = 1 as in every published RoBERTa / XLM-R tokenizer
TINY_XLMR = dict(vocab_size=200, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                 intermediate_size=512, max_position_embeddings=66, type_vocab_size=1, pad_token_id=1,
                 bos_token_id=0, eos_token_id=2, layer_norm_eps=1e-5, hidden_act='gelu', hidden_dropout_prob=0.0,
                 attention_probs_dropout_prob=0.0, initializer_range=0.05)
TINY_XLMR_SEED = 2024
SPECIALS = ['<s>', '<pad>', '</s>', '<unk>']


def position_ids(input_ids: torch.Tensor, padding_idx: int) -> torch.Tensor:
    """``create_position_ids_from_input_ids`` (past_key_values_length 0), int64 [B, S]."""
    m = (input_ids != padding_idx).int()
    return (torch.cumsum(m, dim=1).type_as(m) * m).long() + padding_idx


@torch.no_grad()
def roberta_forward(state_dict: Mapping[str, torch.Tensor], hf_config, input_ids: torch.Tensor,
                    attention_mask: torch.Tensor, token_type_ids: torch.Tensor | None = None) -> torch.Tensor:
    """Last hidden state ``[B, S, H]`` fp32 of ``XLMRobertaModel`` / ``RobertaModel``."""
    sd = {(k[8:] if k.startswith('roberta.') else k): v.detach().to('cpu', torch.float32)
          for k, v in state_dict.items()}
    b, s = input_ids.shape
    h = hf_config.hidden_size
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    pos = position_ids(input_ids, hf_config.pad_token_id)
    word = sd['embeddings.word_embeddings.weight'][input_ids] + sd['embeddings.token_type_embeddings.weight'][
        token_type_ids]
    folded = dict(sd)
    folded['embeddings.word_embeddings.weight'] = word.reshape(b * s, h)
    folded['embeddings.token_type_embeddings.weight'] = sd['embeddings.position_embeddings.weight'][pos].reshape(
        b * s, h)
    folded['embeddings.position_embeddings.weight'] = torch.zeros(max(s, 1), h)
    rows = torch.arange(b * s).view(b, s)
    return bert_forward(folded, hf_config, rows, attention_mask, rows)


def tiny_xlmr_words() -> list[str]:
    return [f'w{i:03d}' for i in range(TINY_XLMR['vocab_size'] - len(SPECIALS))]


def tiny_xlmr_texts() -> list[str]:
    """The texts behind xlmr_tiny_golden.npz: ragged lengths up to 60 words (62 tokens, inside the 64 rows the table
    holds), and two texts with a literal <pad> inside the attended text."""
    words = tiny_xlmr_words()
    rng = np.random.default_rng(9)
    lengths = [3, 17, 40, 1, 25, 25, 9, 60, 12, 30, 2, 44, 7]
    texts = [' '.join(rng.choice(words, size=n)) for n in lengths]
    texts[2] = texts[2].replace(' ', ' <pad> ', 1)
    texts[9] = '<pad> ' + texts[9]
    return texts


def tiny_xlmr_tokenizer():
    """A SentencePiece-style fast tokenizer as XLM-R ships (Unigram model, Metaspace pre-tokenizer, <s> $A </s>),
    built offline: pieces '▁wNNN' after the four specials."""
    from tokenizers import Tokenizer
    from tokenizers import decoders
    from tokenizers import pre_tokenizers
    from tokenizers.models import Unigram
    from tokenizers.processors import TemplateProcessing
    from transformers import PreTrainedTokenizerFast

    pieces = [(t, 0.0) for t in SPECIALS] + [('▁' + w, -1.0) for w in tiny_xlmr_words()]
    raw = Tokenizer(Unigram(pieces, unk_id=3))
    raw.pre_tokenizer = pre_tokenizers.Metaspace()
    raw.decoder = decoders.Metaspace()
    raw.post_processor = TemplateProcessing(single='<s> $A </s>', pair='<s> $A </s> </s> $B </s>',
                                            special_tokens=[('<s>', 0), ('</s>', 2)])
    return PreTrainedTokenizerFast(tokenizer_object=raw, bos_token='<s>', eos_token='</s>', pad_token='<pad>',
                                   unk_token='<unk>', cls_token='<s>', sep_token='</s>',
                                   model_input_names=['input_ids', 'attention_mask'])


def tiny_xlmr_state_dict() -> tuple[object, dict[str, torch.Tensor]]:
    from transformers import XLMRobertaConfig

    from distllm_b200.embed.encoders.weights import random_bert_state_dict

    cfg = XLMRobertaConfig(**TINY_XLMR)
    return cfg, random_bert_state_dict(cfg, seed=TINY_XLMR_SEED, device='cpu')


def write_tiny_xlmr_checkpoint(ckpt_dir: Path) -> None:
    """HF checkpoint directory (config.json, weights, tokenizer files) of the tiny seeded XLM-R."""
    from transformers import XLMRobertaModel

    cfg, sd = tiny_xlmr_state_dict()
    model = XLMRobertaModel(cfg, add_pooling_layer=False)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and not missing, (missing, unexpected)
    ckpt_dir = Path(ckpt_dir)
    ckpt_dir.mkdir(parents=True, exist_ok=True)
    model.eval().save_pretrained(ckpt_dir)
    tiny_xlmr_tokenizer().save_pretrained(ckpt_dir)
