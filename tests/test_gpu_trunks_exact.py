"""Every encoder's forward pass equals, bit for bit, its verified kernels composed by the HF step list.

oracle/trunks.py lists each family's steps from the HF modules (tests/test_trunks_cpu.py pins those lists against the
CPU oracles).  ``LibBlocks`` runs the list on the library's own blocks, each one already pinned bit for bit by the
GEMM, attention and row tests: ``b2e_gemm_h16`` (NF4 weights dequantised, which ``b2e_gemm_nf4`` equals; NF4 + LoRA
as the K-concatenated GEMM ``b2e_gemm_nf4_lora`` equals, after U = X . A_cat^T), the attention entries,
``b2e_debug_rotary``, ``b2e_debug_embed`` and ``b2e_debug_norm`` with the gains and biases of the HF tensor each step
reads.  Every weight is built here from the HF state dict: never through embed/encoders/weights.py or the slot table.

The models tell every norm slot apart (oracle.trunks.state_dict: gains in +-[0.5, 2], biases N(0, 0.5)), so a step
that reads another slot, another layer kind or another eps changes the bits.

(a) ``b2e_encode`` in fp32 and the storage type at every depth (``b2e_debug_set_layers``), all B*S rows of the padded
    layout, against the composition in that layout.
(b) ``b2e_encode_pooled`` (l2 off) in the packed layout against ``b2e_pool_mean`` / ``b2e_pool_last_token`` over the
    composition's final fp32 state: both mean tails walk the same splits and rows in the same order.
(c) ``b2e_embed_host`` twice (the second call replays the captured graphs) against (b).
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from distllm_b200 import _native as nv
from oracle import trunks as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    return torch.device('cuda:0')


EPI = {T.EPI_BIAS: nv.EPI_BIAS, T.EPI_BIAS_GELU: nv.EPI_BIAS_GELU, T.EPI_SWIGLU: nv.EPI_SWIGLU,
       T.EPI_GEGLU: nv.EPI_GEGLU}
NORM = {'post_ln': nv.NORM_POST_LN, 'add_ln': nv.NORM_ADD_LN, 'add_rms': nv.NORM_ADD_RMS}


def is_packed(mask: torch.Tensor) -> bool:
    """The encoders pack the attended tokens back to back when every mask row is a non-empty prefix."""
    lens = mask.sum(1)
    return bool((lens > 0).all() and (mask == (torch.arange(mask.shape[1], device=mask.device)[None]
                                              < lens[:, None]).long()).all())


class LibBlocks:
    """The library's blocks in the layout of ``b2e_encode`` (``pooled`` False: padded) or ``b2e_encode_pooled``."""

    def __init__(self, enc, sd, cfg, mask, pooled: bool, nf4: bool = False, lora=None):
        from distllm_b200.embed.encoders.nf4 import nf4_dequantize, nf4_quantize

        self.enc, self.mask, self.pooled = enc, mask, pooled
        self.dev = mask.device
        self.dtype = nv.STORAGE_TORCH_DTYPE[enc.storage]
        self.sd = T._strip(sd, {'bert': 'bert.', 'esm': 'esm.'}.get(enc._ARCH, 'model.'))
        self.b, self.s = mask.shape
        self.lora = lora or {}
        self._mats = {}

        def to_dev(t):
            w = t.detach().to(self.dev, torch.float32)
            return nf4_dequantize(*nf4_quantize(w)) if nf4 else w

        self.to_dev = to_dev
        set_packing(enc._lib, pooled)

    def mat(self, name):
        if name not in self._mats:
            self._mats[name] = self.to_dev(self.sd[name]).to(self.dtype)
        return self._mats[name]

    def f32(self, t):
        return None if t is None else t.detach().to(self.dev, torch.float32).contiguous()

    def embed(self, ids, mask, types):
        return nv.debug_embed(self.enc, ids, mask, types)

    def linear(self, x, lin, bias, epi, slot):
        w = T.build_weight(lin, [self.mat(n) for n in lin.names])
        adapted = [n for n in lin.names if n[:-len('.weight')] in self.lora]
        if adapted:
            x, w = self.lora_operands(x, w, lin)
        return nv.gemm_h16(x, w, self.f32(bias), epilogue=EPI[epi])

    def lora_operands(self, x, w, lin):
        """[x | U[:, :R]] and [W | B_cat] with U = x . A_cat^T: A_cat the adapted modules' A rows stacked, B_cat each
        module's s * B in its output rows (the slot's row layout) and the columns of its A rows."""
        mods = [n[:-len('.weight')] for n in lin.names]
        r = sum(self.lora[m][0].shape[0] for m in mods if m in self.lora)
        a_cat = torch.zeros(((r + 127) // 128 * 128, x.shape[1]), device=self.dev)
        blocks, col = [], 0
        for m, n in zip(mods, lin.names):
            rows = self.sd[n].shape[0]
            blk = torch.zeros((rows, r), device=self.dev)
            if m in self.lora:
                a, b, s = self.lora[m]
                a_cat[col:col + a.shape[0]] = a.to(self.dev)
                blk[:, col:col + a.shape[0]] = s * b.to(self.dev)
                col += a.shape[0]
            blocks.append(blk)
        b_cat = T.build_weight(T.Linear(lin.names, lin.layout, lin.pad_rows, 0, lin.split), blocks)
        u = nv.gemm_h16(x, a_cat.to(self.dtype), None)
        return (torch.cat([x, u[:, :r]], dim=1).contiguous(),
                torch.cat([w, b_cat.to(self.dtype)], dim=1).contiguous())

    def rotary(self, qkv, layer):
        nv.debug_rotary_(self.enc, layer, qkv, self.mask)

    def attention(self, qkv, heads, kv, d, window, causal):
        b, s, m = self.b, self.s, self.mask
        if self.pooled:
            return nv.attention_packed(qkv, m, b, s, heads, kv, d, window, causal)
        if causal:
            return nv.attention_causal_d128(qkv, m, b, s, heads, kv, window)
        if d == 32:
            return nv.attention_d32(qkv, m, b, s, heads)
        return nv.attention_d64_window(qkv, m, b, s, heads, window) if window else nv.attention_d64(qkv, m, b, s, heads)

    def norm(self, kind, xres, add, resid, gamma, beta, eps, out_dtype):
        return nv.debug_norm(NORM[kind], xres, add, resid, self.f32(gamma), self.f32(beta), eps,
                             out_dtype or self.dtype)

    def unlayout(self, rows):
        if self.pooled and is_packed(self.mask):
            out = rows.new_zeros((self.b, self.s, rows.shape[1]))
            keep = self.mask.bool()
            out[keep] = rows[:int(keep.sum())]
            return out
        return rows.reshape(self.b, self.s, -1)


def set_packing(lib, on: bool) -> None:
    lib.b2e_debug_set_packing.argtypes = [C.c_int]
    nv.check(lib.b2e_debug_set_packing(int(on)), lib)


def set_layers(enc, n: int) -> None:
    enc._lib.b2e_debug_set_layers.argtypes = [C.c_void_p, C.c_int]
    nv.check(enc._lib.b2e_debug_set_layers(enc._handle, n), enc._lib)


def first_difference(got: torch.Tensor, exp: torch.Tensor) -> str | None:
    """None when the bits agree (+0 == -0), else where the first element differs: (b, s, column) or (b, column)."""
    g, e = got.float().cpu().numpy(), exp.float().cpu().numpy()
    bad = ~((g == e) | (np.isnan(g) & np.isnan(e)))
    if not bad.any():
        return None
    idx = tuple(int(i) for i in np.argwhere(bad)[0])
    return f'{bad.sum()} of {bad.size} differ; first at {idx}: expected {e[idx]!r}, got {g[idx]!r}'


# ------------------------------------------------------------------------------------------------ the cases
def masks(s: int) -> dict[str, torch.Tensor]:
    """Right-padded ragged rows whose lengths cross 128-row tiles (packed layout), left padding and holes (padded
    layout)."""
    lens = torch.tensor([s, s - 1, 130, 127, 1, s // 2 + 3])
    ragged = (torch.arange(s)[None] < lens[:, None]).long()
    left = torch.ones(4, s, dtype=torch.int64)
    left[1, :s // 2] = 0
    left[2, :s - 3] = 0
    holes = torch.ones(4, s, dtype=torch.int64)
    holes[1, 5:s // 3] = 0
    holes[2, 1:] = 0
    holes[3, s - 40:] = 0
    return {'ragged': ragged, 'left': left, 'holes': holes}


MASKS = {129: ('ragged', 'left'), 200: ('ragged', 'holes')}

# name: (family, hidden, config keywords)
MODELS = {
    'bert768': ('bert', 768, dict(heads=12)),
    'bert384': ('bert', 384, dict(heads=12)),                       # head_dim 32
    'esm1280': ('esm', 1280, dict(heads=20)),
    'esm640': ('esm', 640, dict(heads=20)),                         # head_dim 32
    'mistral256w': ('mistral', 256, dict(heads=2, kv_heads=1, window=48)),
    'mistral256': ('mistral', 256, dict(heads=2, kv_heads=1)),
    'mistral4096gqa': ('mistral', 4096, dict(heads=32, kv_heads=8, intermediate=4096)),
    'qwen3_1024': ('qwen3', 1024, dict(heads=8, kv_heads=2)),
    'modernbert768': ('modernbert', 768, dict(heads=12, intermediate=1088)),   # padded to 1152
}
NF4 = {'bert768', 'bert384', 'mistral256w', 'mistral256', 'qwen3_1024', 'modernbert768'}
LORA = {'bert768', 'mistral256w'}


def cases():
    out = []
    for name, (fam, _, _) in MODELS.items():
        storages = ('f16',) if fam in ('mistral', 'qwen3') else ('bf16', 'f16')
        weights = ['h16'] + (['nf4'] if name in NF4 else []) + (['lora'] if name in LORA else [])
        for storage in storages:
            for w in weights:
                out.append(pytest.param(name, storage, w, id=f'{name}-{storage}-{w}'))
    return out


def layers_of(name: str, fam: str) -> int:
    return 1 if name == 'mistral4096gqa' else 4 if fam == 'modernbert' else 3


def lora_modules(fam: str, cfg, seed: int) -> dict:
    """Ranks 64 and 192 on different slots (q and v together in one B_cat), scalings other than 1, and slots without an
    adapter: {module: (A [r, in], B [out, r], s)}."""
    g = torch.Generator().manual_seed(seed)
    h, i = cfg.hidden_size, cfg.intermediate_size

    def ab(r, n_in, n_out):
        return (torch.randn(r, n_in, generator=g) / n_in ** 0.5, torch.randn(n_out, r, generator=g) * 0.05)

    if fam == 'bert':
        p = 'encoder.layer.'
        spec = [(p + '0.attention.self.query', 64, h, h, 2.0), (p + '0.attention.self.value', 64, h, h, 0.5),
                (p + '1.attention.output.dense', 192, h, h, 0.25), (p + '2.intermediate.dense', 64, h, i, 1.5),
                (p + '2.output.dense', 64, i, h, 0.75)]
    else:
        heads, kv = cfg.num_attention_heads, cfg.num_key_value_heads
        spec = [('layers.0.self_attn.q_proj', 64, h, heads * 128, 2.0),
                ('layers.0.self_attn.v_proj', 64, h, kv * 128, 0.5),
                ('layers.1.self_attn.o_proj', 192, heads * 128, h, 0.25),
                ('layers.1.mlp.gate_proj', 64, h, i, 1.5), ('layers.1.mlp.up_proj', 64, h, i, 0.75),
                ('layers.2.mlp.down_proj', 64, i, h, 1.25)]
    return {m: (*ab(r, n_in, n_out), s) for m, r, n_in, n_out, s in spec}


def make_inputs(fam: str, mask: torch.Tensor, vocab: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    b, s = mask.shape
    ids = torch.randint(4, vocab, (b, s), generator=g)
    if fam == 'esm':
        ids[:, 2::9] = 32          # mask tokens: token dropout's rescaling
    types = torch.randint(0, 2, (b, s), generator=g) if fam == 'bert' else None
    return ids, types


@pytest.mark.parametrize('name,storage,weights', cases())
def test_trunk_equals_composition(dev, name, storage, weights):
    from distllm_b200.embed.encoders import native as N

    fam, h, kw = MODELS[name]
    cls = {'bert': N.NativeBertEncoder, 'esm': N.NativeEsm2Encoder, 'modernbert': N.NativeModernBertEncoder,
           'mistral': N.NativeMistralEncoder, 'qwen3': N.NativeQwen3Encoder}[fam]
    n_layers = layers_of(name, fam)
    cfg = T.config(fam, h, n_layers, **kw)
    sd = T.state_dict(fam, cfg, seed=h + n_layers)
    lora = lora_modules(fam, cfg, seed=h) if weights == 'lora' else None
    nf4 = weights != 'h16'
    enc = cls(cfg, sd, device=dev, storage=storage, nf4=nf4, lora=lora)
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    step_list = T.FAMILIES[fam]
    try:
        for s, mnames in MASKS.items():
            for mname in mnames:
                mask = masks(s)[mname].to(dev)
                ids, types = make_inputs(fam, mask.cpu(), cfg.vocab_size, seed=s)
                ids, types = ids.to(dev), None if types is None else types.to(dev)
                case = (name, storage, weights, f'S={s}', mname)

                # (a) b2e_encode at every depth, padded layout
                blocks = LibBlocks(enc, sd, cfg, mask, pooled=False, nf4=nf4, lora=lora)
                depths = step_list(sd, cfg, blocks, ids, mask, types, (torch.float32, dtype), every_depth=True)
                for depth, exp in enumerate(depths, start=1):
                    set_layers(enc, depth)
                    for out_dtype in (torch.float32, dtype):
                        got = enc.encode(ids, mask, types, out_dtype)
                        msg = first_difference(got, blocks.unlayout(exp[out_dtype]))
                        assert msg is None, (*case, 'encode', f'depth {depth}', out_dtype, msg)
                set_layers(enc, 0)

                # (b) b2e_encode_pooled against the standalone poolers over the composition's final state
                blocks = LibBlocks(enc, sd, cfg, mask, pooled=True, nf4=nf4, lora=lora)
                final = blocks.unlayout(step_list(sd, cfg, blocks, ids, mask, types)[-1][torch.float32]).contiguous()
                exp = {nv.POOL_MEAN_REF: nv.pool_mean(final, mask.clone(), nv.POOL_MEAN_REF, False),
                       nv.POOL_MEAN_PER_ROW: nv.pool_mean(final, mask.clone(), nv.POOL_MEAN_PER_ROW, False),
                       nv.POOL_LAST_TOKEN: nv.pool_last_token(final, mask)}
                pooled = {}
                for code, e in exp.items():
                    pooled[code] = enc.encode_pooled(ids, mask, types, code, False)
                    msg = first_difference(pooled[code], e)
                    assert msg is None, (*case, 'pooled', code, msg)

                # (c) b2e_embed_host: the first call runs batch 0 eagerly and captures a graph per staging slot for
                # batches 1 and 2, the second call replays them
                if mname == 'ragged' and (weights == 'lora' or (weights == 'h16' and storage == 'f16')):
                    b = mask.shape[0]
                    rep = lambda t: None if t is None else t.cpu().repeat(3, 1).contiguous()   # noqa: E731
                    for code in (nv.POOL_MEAN_REF, nv.POOL_LAST_TOKEN):
                        for call in range(2):
                            got = enc.embed_host(rep(ids), rep(mask), rep(types), b, code, False)
                            for part in range(3):
                                msg = first_difference(got[part * b:(part + 1) * b], pooled[code])
                                assert msg is None, (*case, 'embed_host', code, f'call {call}', f'batch {part}', msg)
    finally:
        set_layers(enc, 0)
        set_packing(enc._lib, True)
        enc.close()
