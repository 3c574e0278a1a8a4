"""distllm_b200: H100-native (sm_90a) implementation of distllm's embedding hot path."""

from __future__ import annotations

__version__ = '0.1.0'
