"""The step lists of oracle/trunks.py, run on fp32 torch stand-ins, against the families' CPU oracles.

tests/test_gpu_trunks_exact.py composes the library's verified kernels by these step lists and asks the encoders'
forward passes to equal them bit for bit.  Here the same lists, with the plain fp32 formula for every block, must
give what oracle.{bert,esm,mistral,modernbert} and tools/oracle_qwen3.py give at every depth, to 1e-5: so a step list
cannot copy a trunk's wiring mistake (a norm reading another slot, a layer kind off by one, a missing eps)."""

from __future__ import annotations

import pytest
import torch

from oracle import trunks as T

CASES = {
    'bert': dict(h=256, heads=4),
    'esm': dict(h=256, heads=8),                  # head_dim 32
    'mistral': dict(h=256, heads=2, kv_heads=1, window=48),
    'mistral-nowindow': dict(h=256, heads=2, kv_heads=1),
    'qwen3': dict(h=256, heads=2, kv_heads=1),
    'modernbert': dict(h=256, heads=4, intermediate=320),   # padded to 384
}


def batch(fam: str, s: int, vocab: int):
    g = torch.Generator().manual_seed(s)
    lens = torch.tensor([s, s - 3, s // 2, 5, 1])
    mask = (torch.arange(s)[None] < lens[:, None]).long()
    ids = torch.randint(4, vocab, (5, s), generator=g)
    if fam == 'esm':
        ids[:, 3::5] = 32                          # mask tokens: token dropout rescales those rows
    types = torch.randint(0, 2, (5, s), generator=g) if fam == 'bert' else None
    return ids, mask, types


@pytest.mark.parametrize('case', list(CASES))
def test_step_list_matches_oracle(case):
    fam = case.split('-')[0]
    kw = dict(CASES[case])
    h = kw.pop('h')
    layers = 4 if fam == 'modernbert' else 3
    cfg = T.config(fam, h, layers, **kw)
    sd = T.state_dict(fam, cfg, seed=11)
    ids, mask, types = batch(fam, 70, cfg.vocab_size)
    blocks = T.TorchBlocks(fam, sd, cfg, mask)
    got = [blocks.unlayout(d[torch.float32]) for d in T.FAMILIES[fam](sd, cfg, blocks, ids, mask, types,
                                                                       every_depth=True)]
    oracle = T.oracle_forward(fam)
    args = (sd, cfg, ids, mask) + ((types,) if fam == 'bert' else ())
    exp = oracle(*args, return_all=True)
    if fam == 'bert':
        exp = exp[1:]                              # hidden_states[0] is the embedding output
    assert len(got) == len(exp) == layers
    live = mask.bool()
    for depth, (a, b) in enumerate(zip(got, exp), start=1):
        err = ((a - b).abs()[live].max() / b[live].abs().max()).item()
        assert err <= 1e-5, (case, depth, err)


def test_step_list_sees_every_norm_slot():
    """The test models tell every norm slot apart: swapping Mistral layer 0's two norm gains, or reading the final norm
    from layer 2's input norm, moves the output by far more than the 1e-5 above."""
    cfg = T.config('mistral', 256, 3, heads=2, kv_heads=1)
    sd = T.state_dict('mistral', cfg, seed=11)
    ids, mask, _ = batch('mistral', 70, cfg.vocab_size)
    blocks = T.TorchBlocks('mistral', sd, cfg, mask)
    base = T.mistral(sd, cfg, blocks, ids, mask)[-1][torch.float32]
    live = mask.reshape(-1).bool()
    for a, b in (('layers.0.input_layernorm.weight', 'layers.0.post_attention_layernorm.weight'),
                 ('norm.weight', 'layers.2.input_layernorm.weight')):
        bad = dict(sd)
        bad[a], bad[b] = sd[b], sd[a]
        blocks = T.TorchBlocks('mistral', bad, cfg, mask)
        out = T.mistral(bad, cfg, blocks, ids, mask)[-1][torch.float32]
        assert ((out - base).abs()[live].max() / base[live].abs().max()).item() > 1e-2, (a, b)
