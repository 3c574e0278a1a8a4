"""Encoder family: ``auto`` (BERT-family checkpoints), ``esm2`` and ``esmc`` (ESM C), all on the native kernels.
``esmc`` reads the checkpoint's state dict directly: the ``esm`` package is not needed."""

from __future__ import annotations

from typing import Any
from typing import Union

from distllm_b200.embed._factory import build_from_strategies
from distllm_b200.embed.encoders.auto import AutoEncoder
from distllm_b200.embed.encoders.auto import AutoEncoderConfig
from distllm_b200.embed.encoders.base import Encoder
from distllm_b200.embed.encoders.esm2 import Esm2Encoder
from distllm_b200.embed.encoders.esm2 import Esm2EncoderConfig
from distllm_b200.embed.encoders.esmc import EsmCambrianEncoder
from distllm_b200.embed.encoders.esmc import EsmCambrianEncoderConfig
from distllm_b200.registry import registry
from distllm_b200.utils import BaseConfig

EncoderConfigs = Union[Esm2EncoderConfig, EsmCambrianEncoderConfig, AutoEncoderConfig]

STRATEGIES: dict[str, tuple[type[BaseConfig], type[Encoder]]] = {
    'esm2': (Esm2EncoderConfig, Esm2Encoder),
    'esmc': (EsmCambrianEncoderConfig, EsmCambrianEncoder),
    'auto': (AutoEncoderConfig, AutoEncoder),
}


def _factory_fn(**kwargs: Any) -> Encoder:
    # a plain function of hashable kwargs so the warm-start registry can key on it
    return build_from_strategies('encoder', STRATEGIES, kwargs)


def get_encoder(kwargs: dict[str, Any], register: bool = False) -> Encoder:
    """Build (or, with ``register=True``, warm-start from the registry) the named encoder.

    ``register=True`` is what the worker uses (distllm/distributed_embedding.py:49): the encoder,
    its device weights and native workspace survive across input files of the same process.
    """
    if register:
        registry.register(_factory_fn)
        return registry.get(_factory_fn, **kwargs)
    return _factory_fn(**kwargs)
