"""Attention references for the kernel tests (csrc/attention.cuh).  TEST INFRASTRUCTURE ONLY.

* :func:`reference` -- float64 attention for the kernel's three modes, in the padded ``[B*S]`` or the packed token
  layout (csrc/pack.cuh), with the set of rows whose value is specified;
* :func:`error_bound` -- a per-element bound on the kernel's error derived from its arithmetic;
* :func:`count_inputs` / :func:`needle_inputs` -- inputs whose kernel output is known bit for bit;
* :func:`finish` -- the kernel's last steps in float32 (``inv = 1.0f / tot``, ``o * inv``, 16-bit rounding);
* :func:`kernel_model` -- the kernel's whole arithmetic in float32 on the host, with optional perturbations (shows
  that the bound is tight enough to catch them).

Modes: 0 bidirectional with the key-padding mask; 1 adds ``|i - j| <= window``; 2 is causal grouped-query attention
with ``i - j < window`` (window 0: no window).  A row with no visible key is unspecified in modes 1 and 2; in mode 0
a row whose mask is all zero is HF's uniform average over the S keys.
"""

from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

LOG2E = 1.4426950408889634
KC = 64                                       # keys per chunk
UNIT_ROUNDOFF = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
E_EX2 = 2.0 ** -22                            # ex2.approx.ftz.f32, relative
E_POLY = 4e-5                                 # poly_exp2 (variant bits 2-3), relative
MASKED = -3.0e38                              # AT_MASKED
POLY_FLOOR = 2.0 ** -126                      # poly_exp2 clamps its argument at -126


def kernel_scale_log2e(d: int) -> float:
    """The launch's fp32 constant ``1.4426950408889634f / sqrtf(D)``."""
    return float(np.float32(LOG2E) / np.sqrt(np.float32(d)))


def e_exp(variant: int) -> float:
    """Relative error of the exponentials of a head_dim-64 variant (bits 2-3: some run as a polynomial)."""
    return E_POLY if (variant >> 2) & 3 else E_EX2


# ------------------------------------------------------------------------------------------------ token layout
@dataclass(frozen=True)
class Layout:
    """Rows of sequence b: row0[b] .. row0[b] + len[b] - 1 (queries); its key j sits at row row0[b] + j."""

    B: int
    S: int
    row0: tuple[int, ...]
    len: tuple[int, ...]
    packed: bool

    @property
    def rows(self) -> int:
        return self.B * self.S

    def keys(self, b: int) -> int:
        """Keys of sequence b that live in the layout (the rest are masked in both layouts)."""
        return self.len[b] if self.packed else self.S


def layout_of(mask: torch.Tensor, packed: bool) -> Layout:
    """pack_lengths / pack_scan: attended tokens back to back when every mask row is a non-empty prefix."""
    m = mask.cpu().bool()
    b_, s_ = m.shape
    n = m.sum(1).tolist()
    prefix = all(n[b] > 0 and bool(m[b, :n[b]].all()) for b in range(b_))
    if packed and prefix:
        row0 = np.concatenate([[0], np.cumsum(n)[:-1]]).astype(int).tolist()
        return Layout(b_, s_, tuple(row0), tuple(n), True)
    return Layout(b_, s_, tuple(b * s_ for b in range(b_)), (s_,) * b_, False)


def to_layout(x: torch.Tensor, lay: Layout, fill: torch.Tensor | float = 0.0) -> torch.Tensor:
    """[B, S, ...] in the padded layout -> [B*S, ...] rows of `lay`; rows past the last packed token = `fill`."""
    if not lay.packed:
        return x.reshape(lay.rows, *x.shape[2:]).clone()
    out = torch.empty((lay.rows, *x.shape[2:]), dtype=x.dtype, device=x.device)
    out[:] = fill
    for b in range(lay.B):
        out[lay.row0[b]:lay.row0[b] + lay.len[b]] = x[b, :lay.len[b]]
    return out


def visible(mask_row: torch.Tensor, mode: int, window: int, i: torch.Tensor, nk: int) -> torch.Tensor:
    """[len(i), nk] bool: which keys query rows i see.  Mode 0 with an all-zero mask: every key (uniform)."""
    m = mask_row[:nk].bool().to(i.device)
    j = torch.arange(nk, device=i.device)
    vis = m[None, :].expand(len(i), nk).clone()
    if mode == 0 and not bool(m.any()):
        vis[:] = True
    if mode == 1:
        vis &= (i[:, None] - j[None, :]).abs() <= window
    if mode == 2:
        vis &= j[None, :] <= i[:, None]
        if window > 0:
            vis &= (i[:, None] - j[None, :]) < window
    return vis


def loaded_chunks(mask_row: torch.Tensor, mode: int, window: int, q0: int, qt: int, S: int) -> tuple[int, int]:
    """Chunk range [lo, hi) the kernel streams for the query tile starting at q0 (qt rows)."""
    on = torch.nonzero(mask_row[:S]).flatten()
    kvc = (int(on[-1]) + KC) // KC if len(on) else (S + KC - 1) // KC
    lo, hi = 0, kvc
    if mode == 1:
        lo, hi = max(0, q0 - window) // KC, min(kvc, (q0 + qt - 1 + window) // KC + 1)
    elif mode == 2:
        lo, hi = (max(0, q0 - window + 1) // KC if window > 0 else 0), min(kvc, (q0 + qt - 1) // KC + 1)
    return (hi - 1 if lo >= hi else lo), hi


# ---------------------------------------------------------------------------------------------- float64 oracle
@dataclass
class Ref:
    """out [R, heads, D] float64 (0 where unspecified); spec [R] bool; the sums the error bound is made of:
    abs_pv = sum_j p_j |v_j|, dev_pv = sum_j p_j |v_j - out|, sub = max_j p_j * sum_j |v_j| (visible j) per
    element, and score_err [R, heads, 1] = bound on the fp32 error of a score in the log2 domain."""

    out: torch.Tensor
    spec: torch.Tensor
    abs_pv: torch.Tensor
    dev_pv: torch.Tensor
    sub: torch.Tensor
    score_err: torch.Tensor
    chunks: int


def split_qkv(qkv: torch.Tensor, heads: int, kv_heads: int, d: int):
    x = qkv.view(qkv.shape[0], heads + 2 * kv_heads, d)
    return x[:, :heads], x[:, heads:heads + kv_heads], x[:, heads + kv_heads:]


def reference(qkv: torch.Tensor, mask: torch.Tensor, heads: int, kv_heads: int, d: int, mode: int, window: int,
              lay: Layout) -> Ref:
    """Attention in float64 on qkv's device.  qkv: [B*S, (heads + 2 kv_heads) d] in `lay`'s rows."""
    dev = qkv.device
    q, k, v = split_qkv(qkv.to(torch.float64), heads, kv_heads, d)
    c = LOG2E / math.sqrt(d)
    rows = qkv.shape[0]
    out = torch.zeros((rows, heads, d), dtype=torch.float64, device=dev)
    abs_pv, dev_pv, sub = torch.zeros_like(out), torch.zeros_like(out), torch.zeros_like(out)
    score_err = torch.zeros((rows, heads, 1), dtype=torch.float64, device=dev)
    spec = torch.zeros(rows, dtype=torch.bool, device=dev)
    rep = heads // kv_heads
    mask = mask.to(dev)
    for b in range(lay.B):
        n, r0, nk = lay.len[b], lay.row0[b], lay.keys(b)
        vis = visible(mask[b], mode, window, torch.arange(n, device=dev), nk)
        uniform = mode == 0 and not bool(mask[b].any())
        alive = vis.any(1)
        qb = q[r0:r0 + n].transpose(0, 1)                                     # [heads, n, d]
        kb = k[r0:r0 + nk].repeat_interleave(rep, dim=1).transpose(0, 1)      # [heads, nk, d]
        vb = v[r0:r0 + nk].repeat_interleave(rep, dim=1).transpose(0, 1)
        y = c * (qb @ kb.transpose(1, 2))
        if uniform:   # the most-negative bias swallows every score: a plain average
            y = torch.zeros_like(y)
        xmax = y.abs().masked_fill(~vis, 0).amax(-1, keepdim=True)
        qk = (c * (qb.abs() @ kb.abs().transpose(1, 2))).masked_fill(~vis, 0).amax(-1, keepdim=True)
        y = y.masked_fill(~vis, -math.inf)
        ymax = y.amax(-1, keepdim=True).nan_to_num(0.0, neginf=0.0)
        w = torch.exp2(y - ymax)
        tot = w.sum(-1, keepdim=True).clamp_min(1e-300)
        p = w / tot
        o = p @ vb
        out[r0:r0 + n] = o.transpose(0, 1)
        abs_pv[r0:r0 + n] = (p @ vb.abs()).transpose(0, 1)
        dv = torch.empty_like(o)
        for col in range(d):
            dv[..., col] = (p * (vb[:, None, :, col] - o[..., col, None]).abs()).sum(-1)
        dev_pv[r0:r0 + n] = dv.transpose(0, 1)
        sub[r0:r0 + n] = ((vis.double() @ vb.abs()) / tot).transpose(0, 1)
        # |error of x_j - x_k| in fp32: the tensor-core dot product (at most d roundings of 2^-23 relative to
        # sum |q k|), the fma with the scale and the subtraction of the running maximum
        score_err[r0:r0 + n] = (d * 2.0 ** -23 * qk + 3 * 2.0 ** -24 * xmax).transpose(0, 1)
        spec[r0:r0 + n] = alive
    out[~spec] = 0
    return Ref(out, spec, abs_pv, dev_pv, sub, score_err, (lay.S + KC - 1) // KC)


def error_bound(ref: Ref, dtype: torch.dtype, e_exp: float) -> torch.Tensor:
    """Per-element bound on |O - O64| for the kernel in storage type `dtype`:

        |O - O64| <= (1 + 4u) [ (u + g) |O64| + (u + g) sum_j p_j |v_j| + e sum_j p_j |v_j - O64| + s ] + f

    Derivation.  The kernel computes O = sum_j P_j v_j / sum_j p_j with p_j = 2^(x_j - m)(1 + e_j) in fp32 and
    P_j = p_j (1 + r_j) rounded to 16 bits (|r_j| <= u, the storage type's unit roundoff: 2^-11 for half, 2^-8 for
    bfloat16).  Writing p_j = Z p64_j (1 + e_j), to first order

        O - O64 = sum_j p64_j r_j v_j + sum_j p64_j e_j (v_j - O64),

    which gives the u and e terms; rounding the normalised output to 16 bits adds u |O64|.  e is the exponential's
    relative error (e_exp: 2^-22 for ex2.approx, 4e-5 for the polynomial) plus ln 2 times the fp32 error of the
    score difference x_j - m (ref.score_err).  g = (20 chunks + 8) 2^-24 covers the fp32 accumulations (P V
    over the chunks, the row sum, the rescales).  s covers weights too small for a normal 16-bit P: half rounds
    them with an absolute error of 2^-25, so sum_j |P_j - p_j| |v_j| / sum_j p_j <= 2^-25 max_j p64_j sum_j |v_j|
    (bfloat16 and ex2.approx.ftz lose at most 2^-126 per weight).  f is half the smallest 16-bit subnormal, the
    output rounding's absolute floor.  The factor (1 + 4u) absorbs the second-order terms."""
    u = UNIT_ROUNDOFF[dtype]
    g = (20 * ref.chunks + 8) * 2.0 ** -24
    e = e_exp + math.log(2.0) * ref.score_err
    tiny = 2.0 ** -25 if dtype == torch.float16 else 2.0 ** -126
    floor = 2.0 ** -25 if dtype == torch.float16 else 2.0 ** -134
    b = (u + g) * ref.out.abs() + (u + g) * ref.abs_pv + e * ref.dev_pv + tiny * ref.sub
    return (1 + 4 * u) * b + floor


def excess(got: torch.Tensor, ref: Ref, dtype: torch.dtype, e_exp: float) -> float:
    """max over specified elements of |got - O64| / bound (<= 1: within the bound)."""
    err = (got.to(torch.float64).view_as(ref.out) - ref.out).abs()
    ratio = err / error_bound(ref, dtype, e_exp)
    return float(ratio[ref.spec].max()) if bool(ref.spec.any()) else 0.0


# ----------------------------------------------------------------------------------------- float32 last steps
def finish(o: torch.Tensor, tot: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """The kernel's epilogue: inv = 1.0f / tot (IEEE division: the build has no fast math), o * inv, rounded to
    nearest in the 16-bit storage type."""
    o, tot = o.to(torch.float32).cpu(), tot.to(torch.float32).cpu()
    inv = torch.tensor(1.0, dtype=torch.float32) / tot
    return (o * inv).to(dtype)


# ------------------------------------------------------------------------------------- family (a): key counts
def count_weight(b: int, g: int, kv_heads: int) -> int:
    """A small integer per (sequence, kv head), different for neighbours, exact in both 16-bit types."""
    return 1 + (b * kv_heads + g) % 251


def count_inputs(mask: torch.Tensor, heads: int, kv_heads: int, d: int, mode: int, window: int, lay: Layout,
                 dtype: torch.dtype, trap: float = 4096.0, seed: int = 0):
    """q = 0, so every visible key gets p = exp2(0) = 1, and v_j[c] = w [j = c mod d] with w = count_weight.
    Then O[i, c] = w count_c(i) / n(i): integer sums, exact in fp32, so the kernel must return
    round16(fp32(w count_c) * fp32(1 / n)) bit for bit.  K holds random values (q = 0 makes every score 0).
    Rows past the last packed token hold `trap` in K and V.

    Returns (qkv [B*S, cols] dtype, expected [B*S, heads, d] dtype, spec [B*S] bool, zero [B*S, d] bool: the
    columns with count 0)."""
    B, S = lay.B, lay.S
    gen = torch.Generator().manual_seed(seed)
    cols = (heads + 2 * kv_heads) * d
    qkv = torch.full((lay.rows, cols), trap, dtype=torch.float32)
    expected = torch.zeros((lay.rows, heads, d), dtype=dtype)
    spec = torch.zeros(lay.rows, dtype=torch.bool)
    zero = torch.zeros((lay.rows, d), dtype=torch.bool)
    resid = torch.nn.functional.one_hot(torch.arange(S) % d, d).to(torch.float32)        # [S, d]
    for b in range(B):
        n, r0, nk = lay.len[b], lay.row0[b], lay.keys(b)
        blk = qkv[r0:r0 + nk].view(nk, heads + 2 * kv_heads, d)
        blk[:, :heads] = 0.0
        blk[:, heads:heads + kv_heads] = torch.randn((nk, kv_heads, d), generator=gen)
        for g in range(kv_heads):
            blk[:, heads + kv_heads + g] = count_weight(b, g, kv_heads) * resid[:nk]
        vis = visible(mask[b].cpu(), mode, window, torch.arange(n), nk).to(torch.float32)
        cnt = vis @ resid[:nk]                                                            # [n, d]
        tot = vis.sum(1, keepdim=True)
        alive = tot[:, 0] > 0
        w = torch.tensor([count_weight(b, h // (heads // kv_heads), kv_heads) for h in range(heads)],
                         dtype=torch.float32)
        o = w[None, :, None] * cnt[:, None, :]                                            # [n, heads, d]
        expected[r0:r0 + n] = finish(o, tot.clamp_min(1)[:, :, None], dtype)
        spec[r0:r0 + n] = alive
        zero[r0:r0 + n] = cnt == 0
    return qkv.to(dtype), expected, spec, zero


# ------------------------------------------------------------------------------------ family (b): needles
def needle_alpha(d: int) -> float:
    """The query scale: a power of two with (alpha / sqrt(d)) log2(e) >= 40, the margin between the target (two
    matching halves) and any other visible key (at most one)."""
    alpha = 1.0
    while alpha / math.sqrt(d) * LOG2E < 40:
        alpha *= 2
    return alpha


@dataclass
class Needles:
    qkv: torch.Tensor          # [B*S, cols] storage type
    expected: torch.Tensor     # [B*S, heads, d]: v of the target key
    check: torch.Tensor        # [B*S, heads] bool: rows with a target
    target: np.ndarray         # [B*S, heads] layout row of the target (-1: none)
    traps: list                # (query row, head, trap row)
    decoys: int                # checked queries whose loaded chunks before the target's hold a one-half match


def needle_inputs(mask: torch.Tensor, heads: int, kv_heads: int, d: int, mode: int, window: int, lay: Layout,
                  dtype: torch.dtype, seed: int = 0, qt: int = 128) -> Needles:
    """Key j of sequence b carries pattern(j + off): one-hot of (j + off) mod d/2 in the first half of the head
    and one-hot of ((j + off) / (d/2)) mod d/2 in the second (off varies with sequence and kv head).  Query i aims
    at one visible key t(i) with q = alpha pattern(t): t scores 2 alpha, every other visible key at most alpha,
    i.e. at least 40 lower in the log2 domain, so the kernel must return v_t exactly (v: random 16-bit values of
    magnitude in [0.5, 2)).  Targets sit at the edges: first / last visible key, keys 63/64 and 127/128, the
    window edges, the diagonal, the sequence's last key.  Keys the query must not see but the kernel loads for it
    (padding, just outside the window or above the diagonal, the next sequence's first keys, rows past the last
    packed token) become traps 2 pattern(t), which would win by 2 alpha if they leaked -- wherever no query that
    does see the key aims at a pattern sharing a half with it.  Visible keys whose pattern repeats a target's are
    zeroed (sequences longer than (d/2)^2)."""
    rng = np.random.default_rng(seed)
    B, S, R = lay.B, lay.S, lay.rows
    hh = d // 2
    rep = heads // kv_heads
    alpha = needle_alpha(d)
    mask = mask.cpu()
    # owner of every layout row: (sequence, key index), -1 for rows past the last packed token
    own_b = np.full(R, -1)
    own_j = np.full(R, -1)
    for b in range(B):
        nk = lay.keys(b)
        own_b[lay.row0[b]:lay.row0[b] + nk] = b
        own_j[lay.row0[b]:lay.row0[b] + nk] = np.arange(nk)
    pid = np.full((R, kv_heads), -1)                    # pattern id of every key row (-1: K = 0)
    for g in range(kv_heads):
        ok = own_b >= 0
        pid[ok, g] = (own_j[ok] + 37 * own_b[ok] + 11 * g) % (hh * hh)
    target = np.full((R, heads), -1)
    vis_of = {}
    for b in range(B):
        n, r0, nk = lay.len[b], lay.row0[b], lay.keys(b)
        vis = visible(mask[b], mode, window, torch.arange(n), nk).numpy()
        vis_of[b] = vis
        if mode == 0 and not mask[b].any():
            continue   # uniform rows: family (a) pins them
        used_by_group: dict[int, dict[int, int]] = {g: {} for g in range(kv_heads)}
        for h in range(heads):
            g = h // rep
            used = used_by_group[g]
            for i in range(n):
                keys = np.nonzero(vis[i])[0]
                if len(keys) == 0:
                    continue
                kinds = [keys[0], keys[-1], 63, 64, 127, 128, i - window, i + window, i - window + 1, i,
                         n - 1, -1]
                kind = (i + 5 * h + 3 * b) % len(kinds)
                t = kinds[kind]
                if lay.packed and b % 2 == 1:
                    # odd sequences aim only at patterns in the lower half of both halves' ranges: their first keys
                    # can then carry traps for the previous sequence's targets in the upper ranges
                    low = (pid[r0 + keys, g] % hh < hh // 2) & (pid[r0 + keys, g] // hh < hh // 2)
                    if kind == 0 or not low.any():
                        continue
                    keys = keys[low]
                if not (0 <= t < nk and t in keys):
                    t = int(rng.choice(keys))
                p = pid[r0 + t, g]
                if p in used and used[p] != t and vis[i, used[p]]:
                    t = used[p]
                used[pid[r0 + t, g]] = t
                target[r0 + i, h] = r0 + t
    # zero every non-target key that repeats a target's pattern id
    for g in range(kv_heads):
        trows = set(target[:, g * rep:(g + 1) * rep][target[:, g * rep:(g + 1) * rep] >= 0].tolist())
        tp = {pid[r, g] for r in trows}
        for r in np.nonzero(np.isin(pid[:, g], list(tp)))[0]:
            if r not in trows:
                pid[r, g] = -1
    # traps
    ta = np.full((R, heads), -1)
    tb = np.full((R, heads), -1)
    chk = target >= 0
    for h in range(heads):
        tp = pid[np.maximum(target[:, h], 0), h // rep]
        ta[chk[:, h], h] = tp[chk[:, h]] % hh
        tb[chk[:, h], h] = tp[chk[:, h]] // hh
    trap_pid = np.full((R, kv_heads), -1)
    is_target = np.zeros((R, kv_heads), dtype=bool)
    for h in range(heads):
        is_target[target[chk[:, h], h], h // rep] = True
    traps = []

    def seers_clear(r: int, g: int, pa: int, pb: int) -> bool:
        b2 = own_b[r]
        if b2 < 0:
            return True
        j2 = own_j[r]
        seen = np.nonzero(vis_of[b2][:, j2])[0] if j2 < vis_of[b2].shape[1] else np.zeros(0, dtype=int)
        if len(seen) == 0:
            return True
        rows = lay.row0[b2] + seen
        a = ta[rows, g * rep:(g + 1) * rep]
        bb = tb[rows, g * rep:(g + 1) * rep]
        return not bool(((a == pa) | (bb == pb)).any())

    for b in range(B):
        n, r0, nk = lay.len[b], lay.row0[b], lay.keys(b)
        vis = vis_of[b]
        for h in range(heads):
            g = h // rep
            for i in range(n):
                t = target[r0 + i, h]
                if t < 0:
                    continue
                lo, hi = loaded_chunks(mask[b], mode, window, i // qt * qt, qt, S)
                cand = {i + window + 1, i - window - 1, i + 1, i - window, n, n + 1, t - r0 - 1, t - r0 + 1}
                invis = np.nonzero(~vis[i, :min(nk, hi * KC)])[0]
                if len(invis):
                    cand |= {int(invis[0]), int(invis[-1])}
                for j in sorted(cand):
                    r = r0 + j
                    if not (lo * KC <= j < hi * KC and 0 <= r < R) or (j < nk and vis[i, j]) or is_target[r, g]:
                        continue
                    p = pid[t, g]
                    if trap_pid[r, g] not in (-1, p) or not seers_clear(r, g, p % hh, p // hh):
                        continue
                    trap_pid[r, g] = p
                    traps.append((r0 + i, h, r))
    # assemble
    x = torch.zeros((R, heads + 2 * kv_heads, d), dtype=torch.float32)
    idx = np.arange(R)
    for g in range(kv_heads):
        kk = x[:, heads + g]
        on = pid[:, g] >= 0
        kk[idx[on], pid[on, g] % hh] = 1.0
        kk[idx[on], hh + pid[on, g] // hh] = 1.0
        tr = trap_pid[:, g] >= 0
        kk[idx[tr]] = 0.0
        kk[idx[tr], trap_pid[tr, g] % hh] = 2.0
        kk[idx[tr], hh + trap_pid[tr, g] // hh] = 2.0
    gen = torch.Generator().manual_seed(seed)
    mag = 0.5 + 1.5 * torch.rand((R, kv_heads, d), generator=gen)
    sign = torch.where(torch.rand((R, kv_heads, d), generator=gen) < 0.5, -1.0, 1.0)
    x[:, heads + kv_heads:] = (mag * sign).to(dtype).float()
    for h in range(heads):
        on = chk[:, h]
        x[idx[on], h, ta[on, h]] = alpha
        x[idx[on], h, hh + tb[on, h]] = alpha
    qkv = x.reshape(R, -1).to(dtype)
    vv = x[:, heads + kv_heads:]
    expected = torch.zeros((R, heads, d), dtype=dtype)
    for h in range(heads):
        on = chk[:, h]
        expected[idx[on], h] = vv[target[on, h], h // rep].to(dtype)
    # decoys: a key matching one half of the target's pattern in an earlier loaded chunk (the online rescale
    # then fires when the target's chunk arrives)
    decoys = 0
    for b in range(B):
        r0, nk = lay.row0[b], lay.keys(b)
        for h in range(heads):
            g = h // rep
            for i in np.nonzero(chk[r0:r0 + lay.len[b], h])[0]:
                tj = target[r0 + i, h] - r0
                lo, _ = loaded_chunks(mask[b], mode, window, i // qt * qt, qt, S)
                span = np.arange(lo * KC, tj // KC * KC)
                span = span[(span < nk) & vis_of[b][i, np.minimum(span, vis_of[b].shape[1] - 1)]]
                p = pid[r0 + span, g]
                if ((p >= 0) & ((p % hh == ta[r0 + i, h]) | (p // hh == tb[r0 + i, h]))).any():
                    decoys += 1
    return Needles(qkv, expected, torch.from_numpy(chk), target, traps, decoys)


def needle_margins(nd: Needles, heads: int, kv_heads: int, d: int, mask: torch.Tensor, mode: int, window: int,
                   lay: Layout) -> tuple[float, float]:
    """(smallest target-over-rest margin among the visible keys, smallest trap-over-target margin), log2 units."""
    q, k, _ = split_qkv(nd.qkv.to(torch.float64), heads, kv_heads, d)
    c = LOG2E / math.sqrt(d)
    rep = heads // kv_heads
    worst, worst_trap = math.inf, math.inf
    for b in range(lay.B):
        n, r0, nk = lay.len[b], lay.row0[b], lay.keys(b)
        vis = visible(mask[b].cpu(), mode, window, torch.arange(n), nk)
        for h in range(heads):
            rows = np.nonzero(nd.check[r0:r0 + n, h].numpy())[0]
            if len(rows) == 0:
                continue
            x = c * (q[r0 + rows, h] @ k[r0:r0 + nk, h // rep].T)
            t = torch.from_numpy(nd.target[r0 + rows, h] - r0)
            xt = x[torch.arange(len(rows)), t]
            other = x.masked_fill(~vis[rows], -math.inf)
            other[torch.arange(len(rows)), t] = -math.inf
            worst = min(worst, float((xt - other.amax(1)).min()))
    for qr, h, r in nd.traps:
        xt = c * float(q[qr, h] @ k[nd.target[qr, h], h // rep])
        worst_trap = min(worst_trap, c * float(q[qr, h] @ k[r, h // rep]) - xt)
    return worst, worst_trap


# ------------------------------------------------------------------------------- the kernel's arithmetic, host
def kernel_model(qkv: torch.Tensor, mask: torch.Tensor, heads: int, kv_heads: int, d: int, mode: int, window: int,
                 lay: Layout, dtype: torch.dtype, scale: float = 1.0, tot_factor: float = 1.0,
                 p_dtype: torch.dtype | None = None, exp_err: float = 0.0) -> torch.Tensor:
    """attention.cuh's arithmetic in float32 on the host: 64-key chunks, x = fma(s, scale_log2e, bias) with
    masked keys at -3e38, the online maximum and rescale, p = exp2(x - m) in fp32, the row sum of the unrounded p,
    P rounded to the storage type for the P V product, then finish().  Perturbations for the tests of the bound:
    `scale` multiplies scale_log2e, `tot_factor` the final row sum, `p_dtype` replaces the 16-bit type P is
    rounded to, `exp_err` gives the exponentials a relative error exp_err * sin(2 pi frac(x))."""
    q, k, v = split_qkv(qkv.to(torch.float32), heads, kv_heads, d)
    c = np.float32(kernel_scale_log2e(d) * scale)
    rep = heads // kv_heads
    out = torch.zeros((lay.rows, heads, d), dtype=dtype)

    def ex2(x: torch.Tensor) -> torch.Tensor:
        y = torch.exp2(x.double())
        if exp_err:
            f = torch.frac(x.double()).nan_to_num(0.0)
            y = y * (1 + exp_err * torch.sin(2 * math.pi * f))
        return y.float()

    for b in range(lay.B):
        n, r0, nk = lay.len[b], lay.row0[b], lay.keys(b)
        vis = visible(mask[b].cpu(), mode, window, torch.arange(n), nk)
        uniform = mode == 0 and not bool(mask[b].any())
        qb = q[r0:r0 + n].transpose(0, 1)
        kb = k[r0:r0 + nk].repeat_interleave(rep, dim=1).transpose(0, 1)
        vb = v[r0:r0 + nk].repeat_interleave(rep, dim=1).transpose(0, 1)
        m = torch.full((heads, n, 1), -math.inf)
        l = torch.zeros((heads, n, 1))
        o = torch.zeros((heads, n, d))
        for c0 in range(0, nk, KC):
            s = (qb.double() @ kb[:, c0:c0 + KC].double().transpose(1, 2)).float()
            x = (s.double() * float(c)).float()
            on = vis[:, c0:c0 + KC] if not uniform else torch.ones_like(vis[:, c0:c0 + KC])
            x = torch.where(on, x if not uniform else torch.full_like(x, MASKED), torch.full_like(x, MASKED))
            mx = torch.maximum(m, x.amax(-1, keepdim=True))
            alpha = ex2(m - mx)
            m = mx
            p = ex2(x - m)
            rs = p.sum(-1, keepdim=True)
            pr = p.to(p_dtype or dtype).float()
            l = l * alpha + rs
            o = o * alpha + pr @ vb[:, c0:c0 + KC].to(dtype).float()
        out[r0:r0 + n] = finish(o, l * np.float32(tot_factor), dtype).transpose(0, 1)
    return out
