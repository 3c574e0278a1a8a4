"""NF4 weight quantisation as the reference's default ``quantization=True`` applies it.

distllm/embed/encoders/auto.py:44-56 loads the checkpoint with
``BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type='nf4', bnb_4bit_use_double_quant=True,
bnb_4bit_compute_dtype=torch.bfloat16)``: every ``nn.Linear`` weight of the model is stored as 4-bit NormalFloat
codes and DEQUANTISED to the compute dtype in front of each matmul.  What reaches the GEMMs is therefore
``dequant(quant(W))``.  This module quantises once, at load time, into the device format of the native NF4 GEMM
(:func:`nf4_quantize`): per ``[N, K]`` matrix (``K % 64 == 0``, so that every 64-element block is one (row, k-block))

  codes   uint8 [N, K/2], row-major; byte j of a row holds column 2j in its high nibble and 2j+1 in its low nibble
  absmax  fp32 [K/64, N], k-block major: the double-quantised block scale absmax' (the fp32 value the dequantisation
          multiplies by, not its 8-bit code), so one tile's 128 scales of a k-block are one 512-byte run

and the GEMM computes ``round16(code[q] * absmax')`` in front of the tensor cores: the same single fp32 product as
:func:`nf4_dequantize`, rounded as ``weights.to_storage`` rounds, i.e. bit for bit the 16-bit matrix
``to_storage(nf4_roundtrip(W))``.  That costs 0.5625 bytes per weight (3.56x less than 16 bits); bitsandbytes'
own storage is ~0.516 bytes, because it keeps the scales as 8-bit codes -- storing the reconstructed fp32 scale is
what makes the GEMM's arithmetic exactly the load-time round trip's.

bitsandbytes (pin >=0.42.0, pyproject.toml) is absent from this image and cannot run on CPU, so this restates
its published algorithm -- PARITY UNPINNED for this branch:

  quantize_4bit(W, blocksize=64, quant_type='nf4')   flatten; per block of 64 values: absmax = max|w|; each
      w / absmax is replaced by the nearest of the 16 NF4 code values (quantiles of N(0,1) normalised to [-1, 1])
  compress_statistics (double quantisation)           offset = mean(absmax); absmax - offset is quantised
      blockwise (blocks of 256) to the 256-entry signed "dynamic" 8-bit code: per block absmax2 = max|x|, each
      x / absmax2 -> nearest code value
  dequantize_4bit                                      absmax' = code8[q] * absmax2 + offset;  w' = nf4[q4] * absmax'
"""

from __future__ import annotations

import torch

NF4_CODE = (
    -1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635,
    -0.18477343022823334, -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725,
    0.24611230194568634, 0.33791524171829224, 0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0,
)


def dynamic_map_8bit() -> torch.Tensor:
    """bitsandbytes.functional.create_dynamic_map(signed=True, max_exponent_bits=7, total_bits=8): 2^i values per
    decade 10^(i-6) (i = 0..6, midpoints of a linear grid over [0.1, 1]) of either sign, plus 0 and 1."""
    data: list[float] = []
    for i in range(7):
        boundaries = torch.linspace(0.1, 1, 2 ** i + 1)
        means = (boundaries[:-1] + boundaries[1:]) / 2.0
        scale = 10.0 ** (-6 + i)
        data += (scale * means).tolist()
        data += (-scale * means).tolist()
    data += [0.0, 1.0]
    assert len(data) == 256
    return torch.tensor(sorted(data), dtype=torch.float32)


def _nearest(values: torch.Tensor, code: torch.Tensor) -> torch.Tensor:
    """Index of the nearest code value (code sorted ascending) for every element."""
    mid = (code[:-1] + code[1:]) / 2.0
    return torch.bucketize(values, mid.to(values.device))


BLOCK = 64
_CHUNK_BLOCKS = 1 << 16   # blocks per step of the code search: bounds its temporaries to ~50 MB


@torch.no_grad()
def _quantize_blocks(blocks: torch.Tensor, double_quant: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """fp32 ``[n_blocks, blocksize]`` -> (codes uint8 ``[n_blocks, blocksize/2]`` packed two per byte, high nibble first; absmax'
    fp32 ``[n_blocks]``).  The code search runs in chunks of blocks so that no full-size temporary is made."""
    code = torch.tensor(NF4_CODE, dtype=torch.float32, device=blocks.device)
    absmax = torch.cat([blocks[i:i + _CHUNK_BLOCKS].abs().amax(dim=1)
                        for i in range(0, blocks.shape[0], _CHUNK_BLOCKS)])
    safe = torch.where(absmax > 0, absmax, torch.ones_like(absmax))
    codes = torch.empty((blocks.shape[0], blocks.shape[1] // 2), dtype=torch.uint8, device=blocks.device)
    for i in range(0, blocks.shape[0], _CHUNK_BLOCKS):
        q4 = _nearest(blocks[i:i + _CHUNK_BLOCKS] / safe[i:i + _CHUNK_BLOCKS, None], code).to(torch.uint8)
        codes[i:i + _CHUNK_BLOCKS] = (q4[:, 0::2] << 4) | q4[:, 1::2]
    if double_quant:
        code8 = dynamic_map_8bit().to(blocks.device)
        offset = absmax.mean()
        centred = absmax - offset
        pad2 = (-centred.numel()) % 256
        c = torch.cat([centred, centred.new_zeros(pad2)]) if pad2 else centred
        c = c.view(-1, 256)
        absmax2 = c.abs().amax(dim=1)
        safe2 = torch.where(absmax2 > 0, absmax2, torch.ones_like(absmax2))
        q8 = _nearest(c / safe2[:, None], code8)
        absmax = (code8[q8] * absmax2[:, None]).flatten()[: absmax.numel()] + offset
    return codes, absmax


def _unpack(codes: torch.Tensor) -> torch.Tensor:
    """uint8 [..., n] -> int64 code indices [..., 2n] (high nibble first)."""
    return torch.stack([codes >> 4, codes & 15], dim=-1).flatten(-2).long()


@torch.no_grad()
def nf4_quantize(weight: torch.Tensor, double_quant: bool = True) -> tuple[torch.Tensor, torch.Tensor]:
    """``quantize_4bit`` of one ``[N, K]`` nn.Linear weight (``K % 64 == 0``) in the device format: (codes uint8
    ``[N, K/2]``, absmax' fp32 ``[K/64, N]``), on ``weight``'s device.  Quantise each checkpoint matrix on its own:
    the double quantisation's offset is the mean over the whole matrix."""
    if weight.dim() != 2 or weight.shape[1] % BLOCK:
        raise ValueError(f'nf4_quantize: need a [N, K] matrix with K % {BLOCK} == 0, got {tuple(weight.shape)}')
    n, k = weight.shape
    w = weight.detach().to(torch.float32).reshape(-1, BLOCK)
    codes, absmax = _quantize_blocks(w, double_quant)
    del w
    return codes.view(n, k // 2), absmax.view(n, k // BLOCK).t().contiguous()


@torch.no_grad()
def nf4_dequantize(codes: torch.Tensor, absmax: torch.Tensor) -> torch.Tensor:
    """Device format -> fp32 ``[N, K]``: ``code[q] * absmax'``, one fp32 product per element."""
    code = torch.tensor(NF4_CODE, dtype=torch.float32, device=codes.device)
    return code[_unpack(codes)] * absmax.t().repeat_interleave(BLOCK, dim=1)


def nf4_storable(weight: torch.Tensor) -> bool:
    """Whether :func:`nf4_quantize` takes this matrix (every quantised matrix of a built checkpoint shape does)."""
    return weight.dim() == 2 and weight.shape[1] % BLOCK == 0


@torch.no_grad()
def nf4_roundtrip(weight: torch.Tensor, blocksize: int = 64, double_quant: bool = True) -> torch.Tensor:
    """``dequantize_4bit(quantize_4bit(weight))`` as fp32, same shape and device as ``weight``: for a matrix the
    device format takes, ``nf4_dequantize(*nf4_quantize(weight))``."""
    if blocksize == BLOCK and nf4_storable(weight):
        return nf4_dequantize(*nf4_quantize(weight, double_quant))
    w = weight.detach().to(torch.float32)
    flat = w.flatten()
    n = flat.numel()
    pad = (-n) % blocksize
    if pad:
        flat = torch.cat([flat, flat.new_zeros(pad)])
    codes, absmax = _quantize_blocks(flat.view(-1, blocksize), double_quant)
    code = torch.tensor(NF4_CODE, dtype=torch.float32, device=w.device)
    out = (code[_unpack(codes)] * absmax[:, None]).flatten()[:n]
    return out.view_as(w)


_LINEAR_SUFFIXES = (
    # BERT / ESM-2
    'attention.self.query.weight', 'attention.self.key.weight', 'attention.self.value.weight',
    'attention.output.dense.weight', 'intermediate.dense.weight', 'output.dense.weight',
    # Mistral
    'self_attn.q_proj.weight', 'self_attn.k_proj.weight', 'self_attn.v_proj.weight', 'self_attn.o_proj.weight',
    'mlp.gate_proj.weight', 'mlp.up_proj.weight', 'mlp.down_proj.weight',
    # ModernBERT
    'attn.Wqkv.weight', 'attn.Wo.weight', 'mlp.Wi.weight', 'mlp.Wo.weight',
)


def is_quantized_linear(name: str, t: torch.Tensor) -> bool:
    """A transformer-block ``nn.Linear`` weight: what bitsandbytes stores in NF4 (embeddings, norms and biases are
    not quantised)."""
    return name.endswith(_LINEAR_SUFFIXES) and t.dim() == 2


def quantize_state_dict_nf4(state_dict: dict[str, torch.Tensor], device: torch.device | str | None = None) -> dict:
    """Copy of ``state_dict`` whose transformer-block ``nn.Linear`` weights went through the NF4 round trip, as
    fp32 (the load-time path: what the 16-bit GEMMs see).  The round trip runs on ``device`` when given."""
    out = {}
    for name, t in state_dict.items():
        if is_quantized_linear(name, t):
            src = t.to(device) if device is not None else t
            out[name] = nf4_roundtrip(src)
        else:
            out[name] = t
    return out
