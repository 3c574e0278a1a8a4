"""Shared fixtures.  ``-m gpu`` tests need an H100; everything else runs on CPU."""

from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest

REPO = Path(__file__).resolve().parents[1]
if str(REPO) not in sys.path:
    sys.path.insert(0, str(REPO))

GOLDEN = REPO / 'tests' / 'golden'


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA sm_90 device (run with -m gpu on an H100)')


@pytest.fixture(scope='session', autouse=True)
def _native_library():
    """Compile libb2e.so when missing or stale (nvcc cross-compiles without a GPU)."""
    from distllm_b200.build import build_native

    build_native()


@pytest.fixture(scope='session')
def pool_golden():
    return np.load(GOLDEN / 'pool_golden.npz')


@pytest.fixture(scope='session')
def semantic_golden():
    return np.load(GOLDEN / 'semantic_golden.npz')


@pytest.fixture(scope='session')
def bert_golden():
    return np.load(GOLDEN / 'bert_tiny_golden.npz')


@pytest.fixture(scope='session')
def tiny_bert():
    """(HF config, seeded state dict) of the tiny checkpoint the golden vectors were made with."""
    from transformers import BertConfig

    sys.path.insert(0, str(REPO / 'oracle'))
    from oracle.make_golden import TINY
    from oracle.make_golden import TINY_SEED

    from distllm_b200.embed.encoders.weights import random_bert_state_dict

    cfg = BertConfig(**TINY)
    return cfg, random_bert_state_dict(cfg, seed=TINY_SEED, device='cpu')


@pytest.fixture(scope='session')
def esm_golden():
    return np.load(GOLDEN / 'esm_tiny_golden.npz')


@pytest.fixture(scope='session')
def tiny_esm():
    """(HF config, seeded state dict) of the tiny ESM-2 checkpoint behind esm_tiny_golden.npz."""
    from transformers import EsmConfig

    from oracle.make_golden import TINY_ESM
    from oracle.make_golden import TINY_ESM_SEED

    from distllm_b200.embed.encoders.weights import random_esm_state_dict

    cfg = EsmConfig(**TINY_ESM)
    return cfg, random_esm_state_dict(cfg, seed=TINY_ESM_SEED, device='cpu')


@pytest.fixture(scope='session')
def mistral_golden():
    return np.load(GOLDEN / 'mistral_tiny_golden.npz')


def tiny_mistral_variant(variant: str):
    """(HF config, seeded state dict) of the tiny Mistral checkpoint behind mistral_tiny_golden.npz;
    variant 'full' = no sliding window, 'window' = the same weights with a sliding window."""
    from transformers import MistralConfig

    from oracle.make_golden import TINY_MISTRAL
    from oracle.make_golden import TINY_MISTRAL_SEED
    from oracle.make_golden import TINY_MISTRAL_WINDOW

    from distllm_b200.embed.encoders.weights import random_mistral_state_dict

    window = None if variant == 'full' else TINY_MISTRAL_WINDOW
    cfg = MistralConfig(**{**TINY_MISTRAL, 'sliding_window': window})
    return cfg, random_mistral_state_dict(cfg, seed=TINY_MISTRAL_SEED, device='cpu')


def cosine_rows(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    a = a.astype(np.float64)
    b = b.astype(np.float64)
    return (a * b).sum(-1) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))


@pytest.fixture(scope='session')
def modernbert_golden():
    return np.load(GOLDEN / 'modernbert_tiny_golden.npz')


@pytest.fixture(scope='session')
def tiny_modernbert():
    """(HF config, seeded state dict) of the tiny ModernBERT checkpoint behind modernbert_tiny_golden.npz."""
    from transformers import ModernBertConfig

    from oracle.make_golden import TINY_MODERNBERT
    from oracle.make_golden import TINY_MODERNBERT_SEED

    from distllm_b200.embed.encoders.weights import random_modernbert_state_dict

    cfg = ModernBertConfig(**TINY_MODERNBERT)
    return cfg, random_modernbert_state_dict(cfg, seed=TINY_MODERNBERT_SEED, device='cpu')
