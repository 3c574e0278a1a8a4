"""ESM C on the device: the fused q / k LayerNorm + rotary kernel against fp32 torch, the row kernels and GEMMs at the
ESMC widths, whole models against the fp32 restatement (tools/oracle_esmc.py) with normal and outlier weights, the
padded and packed layouts, the forward pass as its verified kernels composed step by step, and the ``esmc`` encoder
through the worker and the retriever on a seeded checkpoint in the published ``data/weights/*.pth`` layout."""

from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F  # noqa: N812

from distllm_b200 import _native as nv
from oracle import gemm as G
from oracle import rows as R
from oracle.rows import ODD
from oracle.rows import esmc_pattern
from tools import oracle_esmc as O

pytestmark = pytest.mark.gpu

# published shapes: hidden -> (layers, intermediate)
SHAPES = {960: (30, 2560), 1152: (36, 3072)}
STORAGES = ('f16', 'bf16')


@pytest.fixture(scope='module')
def dev():
    if not torch.cuda.is_available():
        pytest.fail('-m gpu tests need a CUDA device')
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device('cuda:0')


def cos_rows(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return F.cosine_similarity(a.double(), b.double(), dim=-1)


# ------------------------------------------------------------------------------------ qk_layernorm_rope
def qk_check(got: torch.Tensor, qkv: torch.Tensor, qg, kg, cos, sin, pos: torch.Tensor, dtype) -> str | None:
    """The q and k columns of got within oracle.rows.qk_layernorm_rope_bound of the float64 step, before the one
    16-bit rounding (rows_exact's monotone-rounding interval check)."""
    h = qkv.shape[1] // 3
    x = qkv.double().cpu().numpy()
    p = pos.cpu().numpy()
    for j, g in ((0, qg), (1, kg)):
        ref, bound = R.qk_layernorm_rope_bound(x[:, j * h:(j + 1) * h], g.cpu().numpy(), cos.cpu().numpy(),
                                               sin.cpu().numpy(), p, 1e-5)
        msg = R.interval_check(got[:, j * h:(j + 1) * h].double().cpu().numpy(), ref, bound, dtype)
        if msg is not None:
            return ('q', 'k')[j] + ': ' + msg
    return None


@pytest.mark.parametrize('storage', STORAGES)
@pytest.mark.parametrize('t', [1, 1000, 16897])
@pytest.mark.parametrize('h', sorted(SHAPES))
def test_qk_layernorm_rope(dev, h, t, storage):
    """Random q / k rows (per-row offsets) and gains: every output within the bound of
    oracle.rows.qk_layernorm_rope_bound before the one 16-bit rounding -- the fp32 statistic's relative error over H
    terms ((H + 16) 2^-25 on the scale, (H + 2) 2^-24 mean|x| on the mean), one rounding per product and one per sum
    of the rotation, then the 16-bit rounding, so at most one 16-bit ulp from the rounded float64 result
    (tests/test_esmc_exact_cpu.py: the bound holds for an fp32 restatement of the kernel and is at least ten times
    tighter than the former assert_close tolerance).  The bit-for-bit checks are in tests/test_gpu_esmc_exact.py."""
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    g = torch.Generator().manual_seed(h + t)
    qkv = (torch.randn(t, 3 * h, generator=g) * 3 + torch.randn(t, 1, generator=g)).to(dev, dtype)
    qg = (1 + 0.3 * torch.randn(h, generator=g)).to(dev)
    kg = (1 + 0.3 * torch.randn(h, generator=g)).to(dev)
    cos, sin = (u.to(dev).contiguous() for u in O.rotary_tables(2048))
    # padded layout: position t % 2048 (positions up to 2047 at T = 16 897)
    got = nv.qk_layernorm_rope_(qkv.clone(), qg, kg, cos, sin, 1e-5)
    pos = torch.arange(t, device=dev) % 2048
    msg = qk_check(got, qkv, qg, kg, cos, sin, pos, dtype)
    assert msg is None, ('padded', msg)
    assert torch.equal(got[:, 2 * h:].view(torch.int16), qkv[:, 2 * h:].view(torch.int16))
    # packed layout: rows from t_real on and the V columns untouched byte for byte, positions from tok_src
    used = max(1, (2 * t) // 3)
    t_real = torch.tensor([used, 1], dtype=torch.int32, device=dev)
    src = torch.randint(0, 4 * 2048, (t,), generator=g, dtype=torch.int32)
    got = nv.qk_layernorm_rope_(qkv.clone(), qg, kg, cos, sin, 1e-5, t_real, src.to(dev))
    msg = qk_check(got[:used], qkv[:used], qg, kg, cos, sin, (src[:used] % 2048).long(), dtype)
    assert msg is None, ('packed', msg)
    assert torch.equal(got[used:].view(torch.int16), qkv[used:].view(torch.int16))
    assert torch.equal(got[:, 2 * h:].view(torch.int16), qkv[:, 2 * h:].view(torch.int16))


# ------------------------------------------------------------------------------------ row kernels and GEMMs
# oracle.rows' exact rows (+-2^a times a sign pattern whose sum is 0) at the ESMC widths: oracle.rows.esmc_pattern
def test_exact_layernorm_at_esmc_widths(dev, h16):
    """add-LayerNorm over the fp32 stream (ESMC's step, into fp32 and the storage type) and the post-LN LayerNorm of
    16-bit rows, bit for bit against oracle.rows.layernorm on exact rows with an exact gain and bias."""
    for h in sorted(SHAPES):
        n = h // (ODD[h][0] * ODD[h][1])
        # rows +-2^6: at both widths var + eps rounds to 4^6 for every eps below (2^5 is not enough at 960, eps 1e-5)
        x = np.stack([s * 64.0 * esmc_pattern(h, k) for s in (1.0, -1.0) for k in range(1, n // 2)])
        gamma = -8.0 * esmc_pattern(h, n // 2)
        beta = 4.0 * esmc_pattern(h, n // 2 - 1) + 2.0
        g, b = torch.from_numpy(gamma).float().to(dev), torch.from_numpy(beta).float().to(dev)
        for eps in (1e-12, 1e-5):
            exp = R.layernorm(x, gamma, beta, eps)
            for out_dtype, want in ((torch.float32, exp), (h16, R.round16(exp, h16))):
                xres = torch.from_numpy(x).float().to(dev)
                zero = torch.zeros(x.shape, dtype=h16, device=dev)     # the stream plus a zero GEMM output
                got = nv.debug_norm(nv.NORM_ADD_LN, xres, zero, None, g, b, eps, out_dtype).float().cpu().numpy()
                assert np.array_equal(got, want), (h, eps, out_dtype, 'add_ln')
                got = nv.layernorm(torch.from_numpy(x).to(dev, h16), g, b, eps, out_dtype).float().cpu().numpy()
                assert np.array_equal(got, want), (h, eps, out_dtype, 'post_ln')


@pytest.fixture(params=[torch.float16, torch.bfloat16], ids=['f16', 'bf16'])
def h16(request):
    return request.param


@pytest.mark.parametrize('storage', STORAGES)
@pytest.mark.parametrize('h', sorted(SHAPES))
def test_row_kernels_at_esmc_widths(dev, h, storage):
    """add-LayerNorm of general rows (the residual add written back) and the standalone poolers, exactly."""
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    g = torch.Generator().manual_seed(h)
    rows = 77
    xres = (torch.randn(rows, h, generator=g) * 4 + 2).to(dev)
    add = torch.randn(rows, h, generator=g).to(dev, dtype)
    gamma = (1 + torch.randn(h, generator=g)).to(dev)
    beta = torch.randn(h, generator=g).to(dev)
    ref = F.layer_norm((xres.double() + add.double()), (h,), gamma.double(), beta.double(), 1e-5)
    for out_dtype in (torch.float32, dtype):
        x = xres.clone()
        got = nv.debug_norm(nv.NORM_ADD_LN, x, add, None, gamma, beta, 1e-5, out_dtype)
        torch.testing.assert_close(x, (xres + add.float()))
        torch.testing.assert_close(got.double(), ref.to(out_dtype).double(), rtol=1e-2, atol=1e-4
                                   if out_dtype == torch.float32 else 3e-2)
    # standalone masked mean (exact on integer rows, as tests/test_gpu_rows_exact.py) and last token
    s = 130
    mask = (torch.arange(s)[None] < torch.tensor([s, s - 1, 66, 2, 1, 0])[:, None]).long()
    x = torch.randint(-15, 16, (mask.shape[0], s, h), generator=g).double()
    for kind, code in (('ref', nv.POOL_MEAN_REF), ('per_row', nv.POOL_MEAN_PER_ROW)):
        w = R.pool_weights(mask, kind)
        num = R.round16(np.einsum('bs,bsh->bh', w, x.numpy()), dtype)
        exp = num.astype(np.float32) / np.maximum(w.sum(1).astype(np.float32), R.POOL_EPS)[:, None]
        got = nv.pool_mean(x.to(dev, dtype), mask.to(dev), code, False).cpu().numpy()
        assert np.array_equal(got, exp), kind
    got = nv.pool_last_token(x.to(dev, dtype), mask.to(dev)).cpu().numpy()
    assert np.array_equal(got, R.last_token(x.to(dtype).float().numpy(), mask))


@pytest.mark.parametrize('storage', STORAGES)
@pytest.mark.parametrize('n,k', [(960, 960), (2880, 960), (960, 2560)])
def test_gemm_192_only_shapes_bit_exact(dev, n, k, storage):
    """N a multiple of 192 but not of 128: the 128x192 tile, bit for bit against the exact-arithmetic GEMM oracle;
    forcing 128-wide tiles leaves these shapes on the 192-wide kernel."""
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    gen = torch.Generator().manual_seed(n + k)
    a, w = (t.to(dev) for t in G.ternary_pair(300, n, k, gen, dtype))
    bias = torch.randn(n, generator=gen).to(dev)
    exp = G.epilogue(G.exact_product(a, w), bias, None, dtype)
    lib = nv.load(storage)
    lib.b2e_debug_set_gemm_bn.argtypes = [C.c_int]
    try:
        for bn in (0, 128):
            nv.check(lib.b2e_debug_set_gemm_bn(bn), lib)
            got = nv.gemm_h16(a, w, bias)
            assert torch.equal(got.view(torch.int16), exp.to(dev).view(torch.int16)), bn
    finally:
        nv.check(lib.b2e_debug_set_gemm_bn(0), lib)


# ------------------------------------------------------------------------------------ whole models
def make_model(h: int, layers: int, intermediate: int, seed: int, outliers: bool):
    from distllm_b200.embed.encoders import weights as W
    from tools.workloads import add_outliers

    sd = W.random_esmc_state_dict(h, layers, intermediate, seed=seed)
    if outliers:
        add_outliers(sd, 'esmc', seed=seed)
    return sd


def encoder(sd, dev, storage):
    from distllm_b200.embed.encoders import weights as W
    from distllm_b200.embed.encoders.native import NativeEsmcEncoder

    return NativeEsmcEncoder(W.esmc_config(sd), sd, device=dev, storage=storage)


def ragged_batch(b: int, s: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(s // 4, s + 1, (b,), generator=g)
    lens[0] = s
    mask = (torch.arange(s)[None] < lens[:, None]).long()
    ids = torch.randint(4, 29, (b, s), generator=g)
    ids[:, 0] = 0
    ids[torch.arange(b), lens - 1] = 2
    ids[mask == 0] = 1
    return ids, mask


def mean_rows(hidden: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    m = mask.to(hidden.device, hidden.dtype)[..., None]
    return (hidden * m).sum(1) / m.sum(1)


@pytest.mark.parametrize('outliers', [False, True], ids=['normal', 'outliers'])
@pytest.mark.parametrize('depth', ['2', 'full'])
@pytest.mark.parametrize('h', sorted(SHAPES))
def test_model_against_oracle(dev, h, depth, outliers, capsys):
    """Pooled (per-row mean) rows within 1 - cos <= 1e-3 of the fp32 restatement in the build ``esmc`` runs on; the
    other build's worst value is printed for the storage table."""
    layers, inter = SHAPES[h]
    layers = 2 if depth == '2' else layers
    s = 1024 if depth == 'full' else 300
    sd = make_model(h, layers, inter, seed=h + layers, outliers=outliers)
    ids, mask = ragged_batch(4, s, seed=h)
    ids, mask = ids.to(dev), mask.to(dev)
    # POOL_MEAN_PER_ROW drops each row's first and last token
    w = mask.clone()
    w[:, 0] = 0
    w[torch.arange(w.shape[0]), mask.sum(1) - 1] = 0
    exp = mean_rows(O.esmc_forward(sd, ids, mask), w)
    worst = {}
    for storage in STORAGES:
        enc = encoder(sd, dev, storage)
        try:
            got = enc.encode_pooled(ids, mask, None, nv.POOL_MEAN_PER_ROW, False)
            worst[storage] = float((1 - cos_rows(got, exp)).max())
        finally:
            enc.close()
    with capsys.disabled():
        print(f'\nESMC H={h} L={layers} S={s} {"outliers" if outliers else "normal"}: worst 1-cos pooled '
              + ', '.join(f'{k} {v:.2e}' for k, v in worst.items()))
    assert worst[nv.storage_for_arch('esmc')] <= 1e-3, worst


@pytest.mark.parametrize('storage', STORAGES)
@pytest.mark.parametrize('h', sorted(SHAPES))
def test_padded_and_packed_layouts_agree(dev, h, storage):
    layers, inter = SHAPES[h]
    sd = make_model(h, 2, inter, seed=7, outliers=False)
    ids, mask = ragged_batch(5, 257, seed=3)
    ids, mask = ids.to(dev), mask.to(dev)
    enc = encoder(sd, dev, storage)
    lib = enc._lib
    lib.b2e_debug_set_packing.argtypes = [C.c_int]
    try:
        for code in (nv.POOL_MEAN_REF, nv.POOL_MEAN_PER_ROW, nv.POOL_LAST_TOKEN):
            nv.check(lib.b2e_debug_set_packing(1), lib)
            packed = enc.encode_pooled(ids, mask, None, code, False)
            nv.check(lib.b2e_debug_set_packing(0), lib)
            padded = enc.encode_pooled(ids, mask, None, code, False)
            assert torch.equal(packed, padded), code
    finally:
        nv.check(lib.b2e_debug_set_packing(1), lib)
        enc.close()


class Blocks:
    """The library's verified building blocks in the token layout of b2e_encode (``pooled`` False: padded [B*S]) or of
    b2e_encode_pooled (attended tokens back to back for right-padded masks)."""

    def __init__(self, enc, mask, pooled: bool):
        self.enc, self.mask, self.pooled = enc, mask, pooled
        self.dtype = nv.STORAGE_TORCH_DTYPE[enc.storage]
        self.b, self.s = mask.shape
        enc._lib.b2e_debug_set_packing.argtypes = [C.c_int]
        nv.check(enc._lib.b2e_debug_set_packing(int(pooled)), enc._lib)

    def gemm(self, x, w, epi=nv.EPI_BIAS):
        return nv.gemm_h16(x, w.to(self.dtype).contiguous(), None, epilogue=epi)

    def attention(self, qkv, heads):
        if self.pooled:
            return nv.attention_packed(qkv, self.mask, self.b, self.s, heads, heads, 64)
        return nv.attention_d64(qkv, self.mask, self.b, self.s, heads)

    def norm(self, xres, add, g, b, out_dtype=None):
        return nv.debug_norm(nv.NORM_ADD_LN, xres, add, None, g, b, 1e-5, out_dtype or self.dtype)

    def unlayout(self, rows):
        if not self.pooled:
            return rows.reshape(self.b, self.s, -1)
        out = rows.new_zeros((self.b, self.s, rows.shape[1]))
        keep = self.mask.bool()
        out[keep] = rows[:int(keep.sum())]
        return out


def gate_up_blocks(w1: torch.Tensor, inter: int) -> torch.Tensor:
    """ffn.1's rows as the SwiGLU GEMM takes them: 64 gate rows (ffn.1 rows [0, I)), then the 64 up rows
    (rows [I, 2I)) of the same outputs, and so on."""
    gate, up = w1[:inter].reshape(-1, 64, w1.shape[1]), w1[inter:].reshape(-1, 64, w1.shape[1])
    return torch.stack([gate, up], dim=1).reshape(2 * inter, w1.shape[1])


def esmc_steps(sd, blk: Blocks, ids, mask, out_dtypes):
    """The ESM C block (esm/layers/blocks.py, attention.py) as library steps, with every weight built here from the
    checkpoint tensors: out_proj and ffn.3 divided by sqrt(L / 36) in fp32 before the storage rounding.  Returns the
    final norm in each of ``out_dtypes``."""
    dev = mask.device
    d = {k: v.to(dev) for k, v in sd.items()}
    layers = O.num_layers(d)
    h = d['embed.weight'].shape[1]
    inter = d['transformer.blocks.0.ffn.3.weight'].shape[1]
    scale = math.sqrt(layers / 36)
    _, xres = nv.debug_embed(blk.enc, ids, mask)
    tmp = None
    for l in range(layers):
        p = f'transformer.blocks.{l}.'
        hid = blk.norm(xres, tmp, d[p + 'attn.layernorm_qkv.0.weight'], d[p + 'attn.layernorm_qkv.0.bias'])
        qkv = blk.gemm(hid, d[p + 'attn.layernorm_qkv.1.weight'])
        nv.debug_rotary_(blk.enc, l, qkv, mask)
        ctx = blk.attention(qkv, h // 64)
        tmp = blk.gemm(ctx, d[p + 'attn.out_proj.weight'] / scale)
        hid = blk.norm(xres, tmp, d[p + 'ffn.0.weight'], d[p + 'ffn.0.bias'])
        act = blk.gemm(hid, gate_up_blocks(d[p + 'ffn.1.weight'], inter), nv.EPI_SWIGLU)
        tmp = blk.gemm(act, d[p + 'ffn.3.weight'] / scale)
    zero = torch.zeros(h, device=dev)
    return {dt: blk.unlayout(blk.norm(xres.clone(), tmp, d['transformer.norm.weight'], zero, dt)) for dt in out_dtypes}


@pytest.mark.parametrize('storage', STORAGES)
@pytest.mark.parametrize('h', sorted(SHAPES))
def test_forward_equals_its_kernels_composed(dev, h, storage):
    """Bit for bit against the ESM C steps run one kernel at a time (the embedding gather, add-LayerNorm, the GEMMs,
    the encoder's fused q / k LayerNorm + rotary step on its own tables, head_dim-64 attention): (a) b2e_encode into
    fp32 and into the storage type, padded layout; (b) b2e_encode_pooled with every pooler, packed layout, against the
    standalone poolers over the composed final state (the fused final-norm tails at this width); (c) b2e_embed_host."""
    _, inter = SHAPES[h]
    sd = make_model(h, 3, inter, seed=11, outliers=False)
    ids, mask = ragged_batch(3, 200, seed=5)
    ids, mask = ids.to(dev), mask.to(dev)
    enc = encoder(sd, dev, storage)
    dtype = nv.STORAGE_TORCH_DTYPE[storage]
    try:
        exp = esmc_steps(sd, Blocks(enc, mask, pooled=False), ids, mask, (torch.float32, dtype))
        for out_dtype in (torch.float32, dtype):
            got = enc.encode(ids, mask, None, out_dtype)
            assert torch.equal(got.view(-1), exp[out_dtype].view(-1)), out_dtype
        final = esmc_steps(sd, Blocks(enc, mask, pooled=True), ids, mask, (torch.float32,))[torch.float32]
        final = final.contiguous()
        want = {nv.POOL_MEAN_REF: nv.pool_mean(final, mask.clone(), nv.POOL_MEAN_REF, False),
                nv.POOL_MEAN_PER_ROW: nv.pool_mean(final, mask.clone(), nv.POOL_MEAN_PER_ROW, False),
                nv.POOL_LAST_TOKEN: nv.pool_last_token(final, mask)}
        for code, e in want.items():
            assert torch.equal(enc.encode_pooled(ids, mask, None, code, False), e), code
        for code in (nv.POOL_MEAN_REF, nv.POOL_LAST_TOKEN):
            got = enc.embed_host(ids.cpu().repeat(2, 1).contiguous(), mask.cpu().repeat(2, 1).contiguous(), None,
                                 ids.shape[0], code, False)
            assert torch.equal(got[:ids.shape[0]], want[code].cpu()) and torch.equal(got[ids.shape[0]:],
                                                                                     want[code].cpu()), code
    finally:
        nv.check(enc._lib.b2e_debug_set_packing(1), enc._lib)
        enc.close()


# ------------------------------------------------------------------------------------ the encoder end to end
def write_checkpoint(root, h: int, layers: int, inter: int, seed: int):
    size = {960: '300m', 1152: '600m'}[h]
    from distllm_b200.embed.encoders import weights as W

    sd = W.random_esmc_state_dict(h, layers, inter, seed=seed)
    path = root / 'data' / 'weights' / f'esmc_{size}_2024_12_v0.pth'
    path.parent.mkdir(parents=True)
    torch.save(sd, path)
    return sd


SEQS = ['MKTAYIAKQRQISFVKSHFSRQ', 'MSEQ', 'GAVLIPFYWSTCMNQDEKRHXBUZO', 'MKV' * 120, 'ACDEFGHIKLMNPQRSTVWY' * 3,
        'MLLLLAAGGG', 'MQ']


@pytest.mark.parametrize('h', sorted(SHAPES))
def test_get_encoder_through_the_worker_and_the_retriever(dev, tmp_path, monkeypatch, h):
    """A seeded esmc-300m- or 600m-shaped checkpoint directory (2 layers) -> get_encoder -> FASTA -> embedding_worker ->
    numpy writer; the rows equal the encoder's own mean-pooled rows; then the reference's protein_search.py flow:
    Retriever with the mean pooler and an ExactIndex over the embedded file finds every sequence's own row first."""
    from distllm_b200.distributed_embedding import embedding_worker
    from distllm_b200.embed.encoders import get_encoder
    from distllm_b200.embed.poolers import get_pooler
    from distllm_b200.rag.search import ExactIndex
    from distllm_b200.rag.search import Retriever
    from distllm_b200.registry import registry

    monkeypatch.setenv('HF_HUB_OFFLINE', '1')
    ckpt = tmp_path / 'esmc'
    sd = write_checkpoint(ckpt, h, 2, SHAPES[h][1], seed=21)
    (tmp_path / 'seqs.fasta').write_text(''.join(f'>s{i}\n{s}\n' for i, s in enumerate(SEQS)))
    enc_kw = {'name': 'esmc', 'pretrained_model_name_or_path': str(ckpt), 'embedding_size': h}
    embedding_worker(tmp_path / 'seqs.fasta', tmp_path / 'out',
                     dataset_kwargs={'name': 'fasta', 'batch_size': 3, 'num_data_workers': 0, 'pin_memory': True},
                     encoder_kwargs=enc_kw, pooler_kwargs={'name': 'mean'},
                     embedder_kwargs={'name': 'full_sequence', 'normalize_embeddings': True},
                     writer_kwargs={'name': 'numpy'})
    out = [p for p in (tmp_path / 'out').iterdir() if p.is_dir()]
    assert len(out) == 1
    emb = np.load(out[0] / 'embeddings.npy')
    assert emb.shape == (len(SEQS), h) and np.isfinite(emb).all()

    encoder = get_encoder(enc_kw)
    assert encoder.dtype == torch.float16 and encoder.embedding_size == h
    batch = encoder.tokenizer(SEQS[:3], padding=True, truncation=True, return_tensors='pt').to(encoder.device)
    hidden = encoder.encode(batch)
    assert hidden.dtype == torch.float16 and hidden.shape[-1] == h
    ref = O.esmc_forward(sd, batch['input_ids'], batch['attention_mask'])
    live = batch['attention_mask'].bool()
    assert float((1 - cos_rows(hidden.float()[live], ref[live])).max()) < 1e-3

    pooler = get_pooler({'name': 'mean'})
    index = ExactIndex(emb, device=encoder.device)
    retriever = Retriever(encoder, pooler, index, batch_size=3)
    results, _ = retriever.search(query=SEQS, top_k=2)
    assert [r[0] for r in results.total_indices] == list(range(len(SEQS)))
    registry.clear()
    encoder.native.close()
