// Streaming self-attention for sm_90a, head_dim 32, 64 or 128, any S.
//
// One CTA per (query tile of 128 rows, head, sequence); two consumer warpgroups own 64 query rows each and
// one producer warp streams the head's K/V through a shared-memory ring in 64-key chunks with TMA, so S is
// not limited by shared memory.  Per chunk and warpgroup:
//
//   S_j = Q K_j^T       wgmma m64n64k16, Q and K_j both K-major (128B-swizzled TMA boxes of 64 columns; at head_dim
//                       32 one 64B-swizzled box of 32 columns) in shared memory
//   online softmax      in registers, exp2 domain; every row's 64 scores live in the 4 lanes of a quad
//   O  += P_j V_j       wgmma m64n64k16 per 64 output columns (m64n32k16 at head_dim 32), P_j from registers (the
//                       S accumulator layout IS the A fragment layout), V_j as an MN-major shared-memory operand
//
// MODE 0  bidirectional attention with the additive key-padding bias (HF SDPA with an additive mask:
//         transformers/models/bert/modeling_bert.py:192-205, :692-716; the same call pattern serves ESM's).
// MODE 1  the same with a bidirectional sliding window |q - k| <= window (ModernBERT's local layers).
// MODE 2  causal grouped-query attention with an optional sliding window q - k < window
//         (transformers/models/mistral/modeling_mistral.py:122-180, masking_utils sliding-window causal mask).
// Variant V of the head_dim-64 bidirectional kernel (b2e_debug_set_att3_variant / B2E_ATT3 select one for
// side-by-side measurements; every instantiated variant passes the same tests):
//   bit 0     fully attended chunks are known from attn_prep (plain_chunks[b]) and skip their bias loads;
//             without it every chunk reads its bias row
//   bits 2-3  exponentials per four that run as a polynomial on the FMA pipe instead of MUFU.EX2 (0, 1, 2)
//   bit 6     four consumer warpgroups (256 query rows per CTA, each K/V chunk loaded once for all of them)
//             instead of two
//   bit 7     epilogue role: full 64-row output tiles are staged in shared memory and the producer warp
//             stores them with TMA, instead of every thread storing its own pairs
//   bit 8     timeline stamps (profiling instantiation, b2e_debug_set_att3_clock)
// Keys outside the window / above the diagonal take the same finite "most negative" value as padded keys,
// so a row whose first visited chunk holds no visible key carries a harmless running maximum that the
// rescale (factor exp2(-3e38 - m) = 0) wipes as soon as a visible key shows up.  Rows that never see a key
// (queries inside left padding) come out finite; they are never read.
#pragma once

#include "common.cuh"

namespace b2e {

constexpr int AT_KC = 64;                  // keys per chunk
constexpr float AT_MASKED = -3.0e38f;

template <int D, int V>
struct AtCfg {
  // one TMA box: 64 rows of one swizzle row each -- 64 h16 columns (128 B, 128-byte swizzle, 8 KiB) for head_dim 64
  // and 128, 32 columns (64 B, 64-byte swizzle, 4 KiB) for head_dim 32
  static constexpr int COLS = D < 64 ? D : 64;
  static constexpr int ROW_BYTES = 2 * COLS;
  static constexpr int BOX = 64 * ROW_BYTES;
  static constexpr int NB = D / COLS;                      // boxes per row of Q / K / V
  static constexpr int NWG = (V & 64) ? 4 : 2;             // consumer warpgroups, 64 query rows each
  static constexpr int QT = 64 * NWG;                      // query rows per CTA
  // + the producer: one warp, or with four consumer warpgroups a whole warpgroup, so that it can hand its
  // registers to the consumers (setmaxnreg works per warpgroup): 640 x 96 at launch, then 24 in the producer
  // and 112 in the consumers -- without that the 544-thread kernel is held to 96 and spills
  static constexpr int THREADS = 128 * NWG + (NWG == 4 ? 128 : 32);
  static constexpr int CONSUMER_REGS = 112, PRODUCER_REGS = 24;
  static constexpr int STAGES = D == 128 ? 3 : 4;
  static constexpr int Q_BYTES = NWG * NB * BOX;           // [warpgroup][box]
  static constexpr int STAGE_BYTES = 2 * NB * BOX;         // K boxes | V boxes
  static_assert(D == 32 || D == 64 || D == 128, "head_dim");
  static constexpr int BAR = Q_BYTES + STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = BAR + 256 + 1024;      // + slack to align the tiles to 1024 B
  static_assert(SMEM_BYTES <= 232448, "shared memory");
};

// profiling aid (b2e_debug_set_att3_clock): CTA 0 of a bit-8 instantiation records (clock64, event)
// pairs of its first consumer warpgroup: [0][0][n] clocks, [0][1][n] event codes (chunk * 2 + 1: scores
// ready, chunk * 2 + 2: P V done); 256 entries
__device__ long long* g_att_clock = nullptr;

// 2^x on the FMA / ALU pipes: Cody-Waite split x = n + f, f in [-0.5, 0.5], 2^f by its degree-4 Taylor
// polynomial in f ln 2 (relative error below 4e-5, under the 16-bit rounding P goes through), n added to the
// exponent field.  x is clamped at -126 (no denormals, no wrap-around for masked scores).
__device__ __forceinline__ float poly_exp2(float x) {
  x = fmaxf(x, -126.0f);
  const float n = rintf(x);
  const float f = x - n;
  float p = fmaf(f, 9.6181291e-3f, 5.5504109e-2f);
  p = fmaf(f, p, 2.4022651e-1f);
  p = fmaf(f, p, 6.9314718e-1f);
  p = fmaf(f, p, 1.0f);
  return __int_as_float(__float_as_int(p) + (static_cast<int>(n) << 23));
}

// shared-memory descriptor of a Q / K / V box (AtCfg::ROW_BYTES: 128- or 64-byte swizzle)
template <int ROW_BYTES>
__device__ __forceinline__ uint64_t at_box_desc(uint32_t saddr) {
  if constexpr (ROW_BYTES == 128) return make_smem_desc_sw128(saddr);
  else return make_smem_desc_sw64(saddr);
}

// bias[b, j] for j < S_pad (multiple of 64) and kv_chunks[b] = chunks holding an attended key
// (all chunks when nothing is attended, so that such a row degenerates to HF's uniform softmax).
// plain_chunks[b] = number of LEADING chunks whose 64 keys are all attended (right-padded batches: every
// chunk but the last one or two).
__global__ void attn_prep_kernel(const int64_t* __restrict__ mask, float* __restrict__ bias,
                                 int* __restrict__ kv_chunks, int* __restrict__ plain_chunks, int B, int S,
                                 int S_pad) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  int last = 0;
  int first_off = S_pad;   // first key position that is NOT attended (padding beyond S counts)
  for (int j = lane; j < S_pad; j += 32) {
    float v = -INFINITY;
    bool on = false;
    if (j < S) {
      on = mask[static_cast<size_t>(b) * S + j] != 0;
      v = on ? 0.0f : AT_MASKED;
      if (on) last = j + 1;
    }
    if (!on) first_off = min(first_off, j);
    bias[static_cast<size_t>(b) * S_pad + j] = v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
    first_off = min(first_off, __shfl_xor_sync(0xffffffffu, first_off, o));
  }
  if (lane == 0) {
    kv_chunks[b] = last > 0 ? (last + AT_KC - 1) / AT_KC : S_pad / AT_KC;
    plain_chunks[b] = first_off / AT_KC;
  }
}

// tm: the whole qkv matrix [T, (heads + 2 kv_heads) D] (columns q heads | k heads | v heads), box 64 x AtCfg::COLS.
// tm_ctx: ctx [T, heads D], the same box (bit-7 variants only).  seq_cu / seq_len (nullable): token layout
// (pack.cuh), rows [row0, row0 + len) hold sequence b; the padded layout (b S, S) when null.
template <int D, int MODE, int V>
// one CTA per SM is what the launch bounds promise: with two the two-warpgroup kernel is held to 96 registers
// and spills
__global__ void __launch_bounds__(AtCfg<D, V>::THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tm_ctx,
                 const float* __restrict__ bias, const int* __restrict__ kv_chunks,
                 const int* __restrict__ plain_chunks, int B, int S, int S_pad, int heads, int kv_heads, int window,
                 float scale_log2e, const int* __restrict__ seq_cu, const int* __restrict__ seq_len,
                 h16* __restrict__ ctx) {
  using Cfg = AtCfg<D, V>;
  constexpr int NB = Cfg::NB;
  constexpr int COLS = Cfg::COLS, BOX = Cfg::BOX, RB = Cfg::ROW_BYTES;
  constexpr int NWG = Cfg::NWG;
  constexpr int POLY = (V >> 2) & 3;
  constexpr bool EPI_ROLE = (V & 128) != 0;
  constexpr bool STAMPS = (V & 256) != 0;
  static_assert(MODE == 0 || (V & ~(64 | 128)) == 0, "windowed / causal attention: warpgroups and epilogue role only");
  // one-dimensional grid, heads fastest, then sequences, then query tiles from the latest (for causal attention:
  // the heaviest) down
  const int h = blockIdx.x % heads;
  const int b = (blockIdx.x / heads) % B;
  const int tile = static_cast<int>(gridDim.x / (heads * B)) - 1 - static_cast<int>(blockIdx.x / (heads * B));
  const int row0 = seq_cu != nullptr ? __ldg(seq_cu + b) : b * S;
  const int len = seq_len != nullptr ? __ldg(seq_len + b) : S;
  const int q0 = tile * Cfg::QT;
  if (q0 >= len) return;
  const int kvc = __ldg(kv_chunks + b);
  const int np = (V & 1) ? __ldg(plain_chunks + b) : 0;
  int lo = 0, hi = kvc;
  if (MODE == 1) {
    lo = max(0, q0 - window) / AT_KC;
    hi = min(kvc, (q0 + Cfg::QT - 1 + window) / AT_KC + 1);
  } else if (MODE == 2) {
    lo = window > 0 ? max(0, q0 - window + 1) / AT_KC : 0;
    hi = min(kvc, (q0 + Cfg::QT - 1) / AT_KC + 1);
  }
  if (lo >= hi) lo = hi - 1;   // at least one chunk: rows of padding tiles must come out finite

  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_bar = sb + Cfg::BAR;
  const uint32_t full_bar = q_bar + 8;
  const uint32_t empty_bar = full_bar + 8u * Cfg::STAGES;
  const uint32_t out_bar = empty_bar + 8u * Cfg::STAGES;   // [NWG]: a warpgroup's output tile is staged
  const int warp = threadIdx.x >> 5;
  const int kvh = h / (heads / kv_heads);
  const int qcol = h * D, kcol = (heads + kvh) * D, vcol = (heads + kv_heads + kvh) * D;

  if (threadIdx.x == 0) {
    mbar_init(q_bar, 1);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(full_bar + 8u * s, 1);
      mbar_init(empty_bar + 8u * s, NWG);
    }
    for (int w = 0; w < NWG; ++w) mbar_init(out_bar + 8u * w, 1);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= 4 * NWG) {
    if constexpr (NWG == 4) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    if (warp == 4 * NWG && elect_one()) {
      tma_prefetch_desc(&tm);
      mbar_expect_tx(q_bar, Cfg::Q_BYTES);
#pragma unroll
      for (int w = 0; w < NWG; ++w)
#pragma unroll
        for (int x = 0; x < NB; ++x)
          tma_load_2d(sb + (w * NB + x) * BOX, &tm, q_bar, qcol + COLS * x, row0 + q0 + 64 * w);
      int stage = 0;
      uint32_t phase = 0;
      for (int c = lo; c < hi; ++c) {
        mbar_wait(empty_bar + 8u * stage, phase ^ 1u);
        const uint32_t fb = full_bar + 8u * stage;
        const uint32_t dst = sb + Cfg::Q_BYTES + stage * Cfg::STAGE_BYTES;
        mbar_expect_tx(fb, Cfg::STAGE_BYTES);
#pragma unroll
        for (int x = 0; x < NB; ++x) {
          tma_load_2d(dst + x * BOX, &tm, fb, kcol + COLS * x, row0 + c * AT_KC);
          tma_load_2d(dst + (NB + x) * BOX, &tm, fb, vcol + COLS * x, row0 + c * AT_KC);
        }
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1u; }
      }
      if constexpr (EPI_ROLE) {
        // each warpgroup's Q boxes hold its normalised output once its last chunk is done
        for (int w = 0; w < NWG; ++w) {
          mbar_wait(out_bar + 8u * w, 0);
          if (q0 + 64 * w + 64 > len) continue;   // partial tile: its warpgroup stored the rows itself
#pragma unroll
          for (int x = 0; x < NB; ++x)
            tma_store_2d(&tm_ctx, sb + (w * NB + x) * BOX, h * D + COLS * x, row0 + q0 + 64 * w);
        }
        tma_store_commit();
        tma_store_wait_all();   // the stores have read shared memory before the CTA leaves
      }
    }
    return;
  }

  if constexpr (NWG == 4) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));
  const int wg = warp >> 2;
  const int t = threadIdx.x & 127;
  const int quad = t & 3;
  const int qr = q0 + 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2);   // query row of half 0; half 1 is qr + 8
  const float* brow = bias + static_cast<size_t>(b) * S_pad;
  const uint32_t q_addr = sb + wg * NB * BOX;
  long long* clk = nullptr;
  int n_stamp = 0;
  if (STAMPS && blockIdx.x == 0 && threadIdx.x == 0) clk = g_att_clock;

  constexpr int OG = COLS / 8;   // 8-column groups of one box's output accumulator (m64nCOLS: 4 OG floats)
  float o[NB][4 * OG];
#pragma unroll
  for (int x = 0; x < NB; ++x)
#pragma unroll
    for (int i = 0; i < 4 * OG; ++i) o[x][i] = 0.0f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.0f, 0.0f};

  mbar_wait(q_bar, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int c = lo; c < hi; ++c) {
    mbar_wait(full_bar + 8u * stage, phase);
    const uint32_t k_addr = sb + Cfg::Q_BYTES + stage * Cfg::STAGE_BYTES;
    const uint32_t v_addr = k_addr + NB * BOX;
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.0f;
    wgmma_fence();
    // k16 steps: COLS / 16 inside each box row (32 B = +2 in the descriptor's address field each), then the next box
    constexpr int KB = COLS / 16;
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
      wgmma_64x64_ss<0>(s, at_box_desc<RB>(q_addr + (kk / KB) * BOX) + 2u * (kk % KB),
                        at_box_desc<RB>(k_addr + (kk / KB) * BOX) + 2u * (kk % KB), kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    if (STAMPS && clk != nullptr && n_stamp < 256) {
      clk[n_stamp] = clock64();
      clk[256 + n_stamp++] = 2 * c + 1;
    }

    // scores -> x = scale * s + bias (or the masked value), in place.  A fully attended chunk of the
    // bidirectional kernel needs no bias: with bit 0 its loads are skipped and the add is a zero add, so both
    // kinds of chunk share one instruction stream (and one register allocation)
    const int kbase = c * AT_KC + 2 * quad;
    const bool plain = MODE == 0 && (V & 1) && c < np;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 bz = plain ? make_float2(0.0f, 0.0f) : *reinterpret_cast<const float2*>(brow + kbase + 8 * j);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kbase + 8 * j + (e & 1);
        const int q = qr + 8 * (e >> 1);
        float x = fmaf(s[4 * j + e], scale_log2e, (e & 1) ? bz.y : bz.x);
        if (MODE == 1 && abs(q - key) > window) x = AT_MASKED;
        if (MODE == 2 && (key > q || (window > 0 && q - key >= window))) x = AT_MASKED;
        s[4 * j + e] = x;
      }
    }
    float alpha[2];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      float mx = m[hf];
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * hf], s[4 * j + 2 * hf + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      alpha[hf] = fast_exp2(m[hf] - mx);   // m = -inf on the first chunk: 0
      m[hf] = mx;
    }
    uint32_t p[4][4];
    float rs[2] = {0.0f, 0.0f};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const float x0 = s[4 * j + 2 * hf] - m[hf], x1 = s[4 * j + 2 * hf + 1] - m[hf];
        // element (j, hf, e) is exponential number 4 (j & 1) + 2 hf + e of its group of eight
        const int k0 = (2 * (j & 1) + hf) * 2;
        const float p0 = (k0 % 4) < POLY ? poly_exp2(x0) : fast_exp2(x0);
        const float p1 = ((k0 + 1) % 4) < POLY ? poly_exp2(x1) : fast_exp2(x1);
        rs[hf] += p0 + p1;
        p[j >> 1][(j & 1) * 2 + hf] = pack_h16x2(p0, p1);
      }
    }
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) l[hf] = l[hf] * alpha[hf] + rs[hf];
#pragma unroll
    for (int x = 0; x < NB; ++x)
#pragma unroll
      for (int j = 0; j < OG; ++j) {
        o[x][4 * j + 0] *= alpha[0];
        o[x][4 * j + 1] *= alpha[0];
        o[x][4 * j + 2] *= alpha[1];
        o[x][4 * j + 3] *= alpha[1];
      }

#pragma unroll
    for (int x = 0; x < NB; ++x) reg_fence(o[x]);
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 4; ++kc)
#pragma unroll
      for (int x = 0; x < NB; ++x) {
        if constexpr (COLS == 64) wgmma_64x64_rs_tb(o[x], p[kc], make_smem_desc_sw128(v_addr + x * BOX + kc * 16 * 128));
        else wgmma_64x32_rs_tb(o[x], p[kc], make_smem_desc_sw64(v_addr + x * BOX + kc * 16 * 64));
      }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int x = 0; x < NB; ++x) reg_fence(o[x]);
    if (STAMPS && clk != nullptr && n_stamp < 256) {
      clk[n_stamp] = clock64();
      clk[256 + n_stamp++] = 2 * c + 2;
    }
    if (t == 0) mbar_arrive(empty_bar + 8u * stage);
    if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1u; }
  }

  // full 64-row tiles of a bit-7 variant go out through shared memory (this warpgroup's Q boxes, free now:
  // its last wgmma has completed) and the producer's TMA store; everything else row by row from registers
  const bool staged = EPI_ROLE && q0 + 64 * wg + 64 <= len;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    float tot = l[hf];
    tot += __shfl_xor_sync(0xffffffffu, tot, 1);
    tot += __shfl_xor_sync(0xffffffffu, tot, 2);
    const float inv = 1.0f / tot;
    const int q = qr + 8 * hf;
    if (staged) {
      // row inside the 64-row tile; 16-byte unit ^= row & 7 (128-byte swizzle) or (row >> 1) & 3 (64-byte swizzle)
      const int r = q - q0 - 64 * wg;
      const int swz = RB == 128 ? (r & 7) : ((r >> 1) & 3);
#pragma unroll
      for (int x = 0; x < NB; ++x)
#pragma unroll
        for (int j = 0; j < OG; ++j) {
          const uint32_t off = r * RB + ((j ^ swz) << 4) + 4 * quad;
          *reinterpret_cast<uint32_t*>(smem_raw + (q_addr - smem_u32(smem_raw)) + x * BOX + off) =
              pack_h16x2(o[x][4 * j + 2 * hf] * inv, o[x][4 * j + 2 * hf + 1] * inv);
        }
      continue;
    }
    if (q >= len) continue;
    h16* orow = ctx + static_cast<size_t>(row0 + q) * (heads * D) + h * D + 2 * quad;
#pragma unroll
    for (int x = 0; x < NB; ++x)
#pragma unroll
      for (int j = 0; j < OG; ++j)
        *reinterpret_cast<uint32_t*>(orow + COLS * x + 8 * j) =
            pack_h16x2(o[x][4 * j + 2 * hf] * inv, o[x][4 * j + 2 * hf + 1] * inv);
  }
  if constexpr (EPI_ROLE) {
    fence_proxy_async_smem();   // the staged tile is read by the TMA (async proxy)
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
    if (t == 0) mbar_arrive(out_bar + 8u * wg);
  }
}

}  // namespace b2e
