"""``esmc`` encoder: ESM C checkpoints (esmc-300m, esmc-600m) on the native sm_90a forward pass.

Drop-in for distllm/embed/encoders/esmc.py (same config fields, default, validator and error text).  The reference
runs the ``esm`` package's ``ESMC``; here the checkpoint's state dict (a plain ``torch.load``-able ``.pth``) goes to
the native ESMC trunk and the tokenizer is rebuilt from the 33-symbol vocabulary with ``tokenizers``, so the ``esm``
package is not needed.  ``encode`` returns ``ESMCOutput.embeddings`` (after ``transformer.norm``) as float16, as the
reference casts it (esmc.py:131-134).  Values at padded positions are unspecified: no pooler reads them.
"""

from __future__ import annotations

from pathlib import Path
from typing import Literal

import torch
from pydantic import model_validator
from transformers import BatchEncoding
from transformers import PreTrainedTokenizer
from typing_extensions import Self

from distllm_b200.embed.encoders import weights as W
from distllm_b200.embed.encoders.native import NativeEsmcEncoder
from distllm_b200.utils import BaseConfig

# the hub ids the reference names (esmc.py:21-22, :36-39) and the weight file of each repository
ESMC_SIZES = {
    'EvolutionaryScale/esmc-300m-2024-12': 960,
    'EvolutionaryScale/esmc-600m-2024-12': 1152,
}
ESMC_WEIGHT_FILES = {
    'EvolutionaryScale/esmc-300m-2024-12': 'data/weights/esmc_300m_2024_12_v0.pth',
    'EvolutionaryScale/esmc-600m-2024-12': 'data/weights/esmc_600m_2024_12_v0.pth',
}
# The sequence vocabulary of the esm package (ids 0-32).  Ids 0-30 and 32 are ESM-2's; 31 is the chain break.
ESMC_VOCAB = ('<cls>', '<pad>', '<eos>', '<unk>', 'L', 'A', 'G', 'V', 'S', 'E', 'R', 'T', 'I', 'D', 'P', 'K', 'Q',
              'N', 'F', 'Y', 'M', 'H', 'W', 'C', 'X', 'B', 'U', 'Z', 'O', '.', '-', '|', '<mask>')


class EsmCambrianEncoderConfig(BaseConfig):
    """Config for the ESM-Cambrian encoder (fields as in the reference, esmc.py:16-57)."""

    # The name of the encoder
    name: Literal['esmc'] = 'esmc'  # type: ignore[assignment]
    # The model id, options [EvolutionaryScale/esmc-300m-2024-12,
    # EvolutionaryScale/esmc-600m-2024-12]; also a local directory with the repository's data/weights/*.pth layout,
    # or the path of the .pth file itself
    pretrained_model_name_or_path: str = 'EvolutionaryScale/esmc-300m-2024-12'
    # The model embedding size (if you are using a fine-tuned model
    # you should explicitly set this value)
    embedding_size: int | None = None

    @model_validator(mode='after')
    def set_embedding_size(self) -> Self:
        """Set the embedding size based on the model name."""
        if self.embedding_size is not None:
            return self
        embedding_size = ESMC_SIZES.get(self.pretrained_model_name_or_path, None)
        if embedding_size is None:
            raise ValueError(
                f'Invalid model name for ESMC: '
                f'{self.pretrained_model_name_or_path} '
                f'Valid model names are: {", ".join(ESMC_SIZES.keys())}.',
                'Or you can set the embedding_size parameter explicitly ',
                'if you are using a fine-tuned model.',
            )
        self.embedding_size = embedding_size
        return self


def esmc_tokenizer() -> PreTrainedTokenizer:
    """The esm package's ``EsmSequenceTokenizer``, rebuilt: a character-level BPE without merges over
    :data:`ESMC_VOCAB`, ``<unk>`` for unknown characters, the template ``<cls> $A <eos>``, right padding with
    ``<pad>`` and ``model_max_length`` 2048 (esmc.py:82)."""
    from tokenizers import Tokenizer
    from tokenizers.models import BPE
    from tokenizers.processors import TemplateProcessing
    from transformers import PreTrainedTokenizerFast

    vocab = {tok: i for i, tok in enumerate(ESMC_VOCAB)}
    tok = Tokenizer(BPE(vocab, merges=[], unk_token='<unk>'))
    tok.add_special_tokens(['<cls>', '<pad>', '<mask>', '<eos>', '|'])
    tok.post_processor = TemplateProcessing(single='<cls> $A <eos>',
                                            special_tokens=[('<cls>', vocab['<cls>']), ('<eos>', vocab['<eos>'])])
    fast = PreTrainedTokenizerFast(tokenizer_object=tok, unk_token='<unk>', cls_token='<cls>', pad_token='<pad>',
                                   mask_token='<mask>', eos_token='<eos>', additional_special_tokens=['|'])
    fast.model_max_length = W.ESMC_MAX_POS
    return fast


def resolve_checkpoint(name_or_path: str) -> Path:
    """The ``.pth`` of ``name_or_path``: the file itself, ``data/weights/*.pth`` of a local directory (exactly one),
    or, for the reference's hub ids, ``huggingface_hub.hf_hub_download`` of the repository's weight file (its
    cache, or a download where a network exists)."""
    path = Path(name_or_path)
    if path.is_file():
        return path
    if path.is_dir():
        found = sorted((path / 'data' / 'weights').glob('*.pth'))
        if len(found) != 1:
            raise FileNotFoundError(f'{path}: expected exactly one data/weights/*.pth, found {len(found)}')
        return found[0]
    if name_or_path in ESMC_WEIGHT_FILES:
        from huggingface_hub import hf_hub_download

        return Path(hf_hub_download(repo_id=name_or_path, filename=ESMC_WEIGHT_FILES[name_or_path]))
    raise FileNotFoundError(f'{name_or_path}: not a .pth file, a directory with data/weights/*.pth or one of '
                            f'{sorted(ESMC_WEIGHT_FILES)}')


class EsmCambrianEncoder:
    """Encoder for the ESM-Cambrian model on the native kernels.

    For more information on the ESM-Cambrian model, see:
    https://www.evolutionaryscale.ai/blog/esm-cambrian
    """

    def __init__(self, config: EsmCambrianEncoderConfig):
        state_dict = torch.load(resolve_checkpoint(config.pretrained_model_name_or_path), map_location='cpu',
                                weights_only=True)
        esmc_config = W.esmc_config(state_dict)
        if esmc_config.hidden_size != config.embedding_size:
            raise ValueError(f'embedding_size {config.embedding_size} disagrees with the checkpoint '
                             f'{config.pretrained_model_name_or_path}, whose hidden size is {esmc_config.hidden_size}')
        NativeEsmcEncoder.validate(esmc_config)   # unsupported shapes fail before a weight moves to the device
        self.config = config
        self._native = NativeEsmcEncoder(esmc_config, state_dict)
        del state_dict
        self._tokenizer = esmc_tokenizer()
        self._embedding_size = config.embedding_size

    @property
    def dtype(self) -> torch.dtype:
        """float16, as the reference (its bfloat16 model output is cast in ``encode``)."""
        return torch.float16

    @property
    def device(self) -> torch.device:
        return self._native.device

    @property
    def embedding_size(self) -> int:
        return self._embedding_size

    @property
    def tokenizer(self) -> PreTrainedTokenizer:
        return self._tokenizer

    @property
    def native(self) -> NativeEsmcEncoder:
        return self._native

    def encode(self, batch_encoding: BatchEncoding) -> torch.Tensor:
        """``ESMCOutput.embeddings`` ``[B,S,H]`` as float16 (esmc.py:115-134).  The key-padding mask is the
        batch's attention mask, which for right-padded tokenizer batches is ``input_ids != <pad>``, the mask
        ``ESMC.forward`` builds."""
        hidden = self._native.encode(batch_encoding['input_ids'], batch_encoding['attention_mask'], None,
                                     out_dtype=torch.float32)
        return hidden.to(torch.float16)

    def encode_pooled(self, batch_encoding: BatchEncoding, pool_kind: int, normalize: bool,
                      out: torch.Tensor | None = None) -> torch.Tensor:
        """Fused encode + pool (+ normalise) -> fp32 ``[B,H]`` (used by the native embedders)."""
        return self._native.encode_pooled(batch_encoding['input_ids'], batch_encoding['attention_mask'], None,
                                          pool_kind, normalize, out=out)
