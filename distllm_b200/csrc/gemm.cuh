// Persistent, warp-specialised h16 GEMM for sm_90a:  out[M,N] = epi(A[M,K] . W[N,K]^T + bias)
//
//   warpgroup 2   TMA producer (one elected lane, 40 registers; 24 at BN = 192): for every tile of the CTA, the
//                 128 x 64 A box and the BN x 64 W box of each k-block into a 128B-swizzled shared-memory ring of
//                 five stages (three at BN = 192)
//   warpgroups    two consumers (232 registers each; 240 at BN = 192), each owning a whole 128 x BN output tile:
//   0 and 1       two wgmma m64nBNk16 per k16 step sharing the W descriptor, BN fp32 accumulators per thread; the
//                 epilogue (+bias, erf-GELU | +residual | gated activation) runs on those registers, writes h16
//                 pairs into the warpgroup's swizzled staging tile and one thread stores it with TMA
//
// The epilogue picks its path once per tile.  A tile inside the device rows runs straight-line code: the tile's
// bias comes from the consumer's slot in shared memory (loaded from global memory when the turn starts, written
// after the main loop), two 8-column groups of both 64-row halves per step (16 independent pairs, so the GELU
// chains overlap), and each group pair goes into the staging tile with one stmatrix.x4 per half -- no row test,
// no global address and no branch inside the element loop.  The last row tile crossing M stores its rows from
// registers, one row test per pair.
//
// BN (the tile width) is 128 or 192 (GemmPlan).  A 192-wide tile moves a sixth fewer operand bytes through L2 and
// shared memory per FLOP than a 128-wide one; each output element sums the same products in the same order at
// either width, so both give the same bits.  The NF4 producer (one W row per thread of 128) and the gated
// epilogues (gate and up paired in 64-row blocks of a 128-row W tile) exist at BN = 128 only.
//
// One CTA per SM walks the tiles blockIdx.x, blockIdx.x + gridDim.x, ... (N tiles fastest, so that the CTAs
// running together share their A rows in L2); consumer 0 takes the CTA's even-numbered tiles, consumer 1 the
// odd ones.  Ping-pong: two named barriers pass the tensor cores from one consumer to the other at the end of
// each main loop, so the epilogue of one tile runs while the other consumer's main loop keeps the tensor cores
// busy, and the two main loops never interleave.
//
// The NF4 instantiation (NF4 = true, quantization=True) differs only on the producer side: the W tile is written
// into shared memory by the producer warpgroup from 4-bit codes and fp32 block scales (gemm_nf4_producer) instead of
// being loaded by the TMA; consumers, hand-over, tile walk and epilogues are the same code.
//
// gemm_nf4_lora_kernel (a LoRA adapter kept unmerged beside NF4 weights) is the NF4 body with R/64 more k-blocks
// per tile: U = X . A_cat^T and B_cat, both 16-bit, TMA-loaded into the stage as the 16-bit kernel loads A and W, so
// y = epi(X . dequant(W)^T + U . B_cat^T + bias): every epilogue applies to the sum, as peft's layer adds the
// low-rank term before the activation.
//
// This replaces the cuBLAS nn.Linear calls HF BERT issues from
// transformers/models/bert/modeling_bert.py:180-182 (q,k,v), :294-298 (attn out), :339-342 (FFN up +
// GELU), :352-356 (FFN down), reached from distllm/embed/encoders/auto.py:135.
#pragma once

#include "common.cuh"

namespace b2e {

// EPI_SWIGLU: W holds gate and up rows interleaved in blocks of 64 (weights.py: interleave_gate_up),
// so columns [128t, 128t+64) of the product are gate and [128t+64, 128t+128) up of outputs
// [64t, 64t+64); the epilogue writes silu(gate) * up into out [M, N/2].
// EPI_GEGLU: the same layout with erf-GELU on the first half of each pair ("input" rows of ModernBERT's Wi, the
// "gate" rows multiply): out = gelu(input) * gate (transformers/models/modernbert/modeling_modernbert.py:88-91).
enum GemmEpi : int { EPI_BIAS = 0, EPI_BIAS_GELU = 1, EPI_BIAS_RESID = 2, EPI_SWIGLU = 3, EPI_GEGLU = 4 };
__host__ __device__ constexpr bool epi_is_glu(int epi) { return epi == EPI_SWIGLU || epi == EPI_GEGLU; }

constexpr int GEMM_BM = 128;
constexpr int GEMM_BN = 128;
constexpr int GEMM_BK = 64;  // 64 h16 = one 128-byte swizzle row
constexpr int GEMM_STAGES = 5;
constexpr int GEMM_THREADS = 384;   // two consumer warpgroups + the producer warpgroup
constexpr int GEMM_PRODUCER_REGS = 40, GEMM_CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 64 Ki registers
constexpr int GEMM_A_BYTES = GEMM_BM * GEMM_BK * 2;
constexpr int GEMM_STAGE_BYTES = GEMM_A_BYTES + GEMM_BN * GEMM_BK * 2;
constexpr int GEMM_OUT_BOX = GEMM_BM * 64 * 2;   // one 64-column TMA store box of a tile, 16 KiB
// named barriers: GEMM_BAR_TURN + w = consumer w may issue its main loop; GEMM_BAR_STAGE + w = consumer w's
// staging tile is free / written; GEMM_BAR_NF4 = the NF4 producers have dequantised a k-block
constexpr int GEMM_BAR_TURN = 1, GEMM_BAR_STAGE = 3, GEMM_BAR_NF4 = 5;

// NF4 weights (embed/encoders/nf4.py: nf4_quantize): codes uint8 [N, K/2] (byte j of a row = column 2j in the
// high nibble, 2j + 1 in the low one) and fp32 block scales absmax [K/64, N].  The producer warpgroup TMA-loads a
// tile's 128 x 32-byte code box and its 128 scales (one contiguous 512-byte run) into a raw ring, and its 128
// threads (one W row each) write round16(code[q] * absmax) into the stage's W region in the 128B-swizzled layout
// the TMA gives a 16-bit W box: the wgmma sees byte for byte the tile of the 16-bit matrix dequantised on the host.
// The raw ring costs a stage: four instead of five.
constexpr int GEMM_NF4_RAW = 4;                                    // raw ring slots
constexpr int GEMM_NF4_CODE_BYTES = GEMM_BN * GEMM_BK / 2;         // 128 rows x 32 bytes
constexpr int GEMM_NF4_RAW_BYTES = GEMM_NF4_CODE_BYTES + GEMM_BN * 4;   // + 128 fp32 scales

// Shared-memory plan and register split of one instantiation: [stages][output staging][bias slots][raw ring]
// [mbarriers][code table].  At BN = 128 a stage is 32 KiB and each consumer's staging tile two 16 KiB store boxes;
// at BN = 192 a stage is 40 KiB and a staging tile three boxes, which leaves room for three stages.  A bias slot
// holds the BN fp32 bias values of the consumer's current tile.
template <bool NF4, int BN = GEMM_BN>
struct GemmPlan {
  static_assert(BN == 128 || BN == 192, "tile widths");
  static_assert(!NF4 || BN == 128, "the NF4 producer writes one W row per thread of its warpgroup");
  static constexpr int STAGE_BYTES = GEMM_A_BYTES + BN * GEMM_BK * 2;
  static constexpr int OUT_BOXES = BN / 64;   // 64-column TMA store boxes per tile
  static constexpr int STAGES = NF4 ? 4 : BN == 192 ? 3 : GEMM_STAGES;
  static constexpr int OUT_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BIAS_OFFSET = OUT_OFFSET + 2 * OUT_BOXES * GEMM_OUT_BOX;   // [consumer][BN] fp32
  static constexpr int RAW_OFFSET = BIAS_OFFSET + 2 * BN * 4;
  static constexpr int BAR_OFFSET = RAW_OFFSET + (NF4 ? GEMM_NF4_RAW * GEMM_NF4_RAW_BYTES : 0);
  // full[STAGES], empty[STAGES], then (NF4) raw_full[GEMM_NF4_RAW]
  static constexpr int TABLE_OFFSET = BAR_OFFSET + 16 * STAGES + (NF4 ? 8 * GEMM_NF4_RAW : 0);
  static constexpr int SMEM_BYTES = TABLE_OFFSET + (NF4 ? 16 * 4 : 0) + 1024;
  // the dequantising producers need more than the TMA-only producer's 40 registers; 192 fp32 accumulators need
  // more than 232 in the consumers, which the TMA-only producer's 24 leave them
  static constexpr int PRODUCER_REGS = NF4 ? 56 : BN == 192 ? 24 : GEMM_PRODUCER_REGS;
  static constexpr int CONSUMER_REGS = NF4 ? 224 : BN == 192 ? 240 : GEMM_CONSUMER_REGS;
  // setmaxnreg moves registers within what the CTA was launched with (__launch_bounds__(384, 1): 168 per thread);
  // a consumer's increase waits until the producers' decrease has freed enough, so a split beyond it never starts
  static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= GEMM_THREADS * 168, "registers the CTA holds");
  static_assert(SMEM_BYTES <= 232448, "shared memory of one SM");
};
static_assert(GemmPlan<false>::STAGE_BYTES == GEMM_STAGE_BYTES, "the 16-bit plan");

// bitsandbytes' NF4 code values (embed/encoders/nf4.py: NF4_CODE) as fp32 bit patterns
__constant__ uint32_t kNf4CodeBits[16] = {
    0xbf800000u, 0xbf3239b1u, 0xbf066b30u, 0xbeca32a0u, 0xbe91a24du, 0xbe3d353fu, 0xbdba7871u, 0x00000000u,
    0x3da2faffu, 0x3e24cae3u, 0x3e7c04ddu, 0x3ead033au, 0x3ee1a4b8u, 0x3f1007abu, 0x3f3913b3u, 0x3f800000u,
};

// erf-GELU, x * Phi(x), with Phi from the Abramowitz-Stegun 7.1.26 erfc polynomial
// (|erf error| <= 1.5e-7): gelu(x) = max(x,0) - 0.5*|x|*poly(t)*exp(-x^2/2), t = 1/(1 + p*|x|/sqrt2).
// ~14 FP instructions + 2 MUFU per element instead of libdevice erff's ~35: the FFN-up epilogue
// is issue-bound, and the output is rounded to h16 (2^-9) anyway.
// Cheaper variant used by the FFN-up epilogue: erf(x/sqrt2) ~= tanh(x * Q(x^2)) with a cubic Q fitted
// to erf itself (max |erf error| 1.4e-5 before the hardware tanh), one MUFU (tanh.approx.f32, abs error
// ~5e-4) instead of two.  gelu(x) = 0.5 x (1 + erf(x/sqrt2)).  Total absolute error <= ~3e-4 |x|,
// i.e. below the h16 rounding (2^-9 relative) the output goes through anyway.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float xc = fminf(fmaxf(x, -5.65685f), 5.65685f);  // |x|/sqrt2 <= 4: the fit's range
  const float v = xc * xc;
  float q = fmaf(v, -1.35688221e-05f, -1.95764464e-04f);
  q = fmaf(v, q, 3.65498251e-02f);
  q = fmaf(v, q, 7.97818838e-01f);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(xc * q));
  const float h = 0.5f * x;
  return fmaf(h, t, h);
}

__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678f, ax, 1.0f)));
  float p = fmaf(t, 1.061405429f, -1.453152027f);
  p = fmaf(t, p, 1.421413741f);
  p = fmaf(t, p, -0.284496736f);
  p = fmaf(t, p, 0.254829592f);
  p *= t;
  const float e = fast_exp2(ax * ax * (-0.5f * 1.4426950408889634f));
  return fmaxf(x, 0.0f) - 0.5f * ax * p * e;
}

__device__ __forceinline__ float silu(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + fast_exp2(-1.4426950408889634f * x)));
  return x * r;
}


// profiling aid (b2e_debug_set_clock_buffer): CTA 0 of the TL instantiation records clock64() once per
// K block in the producer ([0][n], after issuing the loads) and in the first consumer warpgroup ([1][n], when
// the block's MMAs have been retired), and at the start and end of each epilogue of the first consumer ([2][e]
// when its accumulators are final, [3][e] after its TMA store is issued; e = its e-th tile); 4 x 256 int64
__device__ long long* g_gemm_clock = nullptr;

// The tiles of CTA blockIdx.x: first, first + stride, ... (count of them) of the linear tile index, N tiles
// fastest, over the rows [0, M) the kernel was given.  Every role derives its sequence from here, so that the
// producer pushes exactly the k-blocks the consumers pop and both consumers agree on whose turn is next.
struct GemmTiles {
  int first, stride, count, n_tiles;
};
template <int BN>
__device__ __forceinline__ GemmTiles gemm_tiles(int M, int N) {
  const int n_tiles = N / BN;
  const int tiles = n_tiles * ((M + GEMM_BM - 1) / GEMM_BM);
  const int first = static_cast<int>(blockIdx.x), stride = static_cast<int>(gridDim.x);
  return {first, stride, first < tiles ? (tiles - 1 - first) / stride + 1 : 0, n_tiles};
}

// a read of data that stays constant once written (the NF4 code table): free to schedule, so that the producers
// keep many lookups in flight
__device__ __forceinline__ float ld_shared_const_f32(uint32_t addr) {
  float v;
  asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ float ld_shared_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ float2 ld_shared_f32x2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_f32x2(uint32_t addr, float2 v) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}
// four 8 x 8 b16 matrices: lanes 8i .. 8i + 7 give the 16-byte row addresses of matrix i, and register i of lane l
// holds row l / 4, columns 2 (l % 4) + {0, 1} of matrix i -- the layout of a wgmma accumulator's 8-column group
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}

// The NF4 producer warpgroup (all 128 threads; thread p dequantises W row p of every tile).  Thread 0 also issues
// the loads: the A box of each k-block once its stage is free, and the code box + scales of the k-block
// GEMM_NF4_RAW ahead into the raw slot the warpgroup has just finished reading.  A stage's full barrier completes
// on the A bytes plus thread 0's arrival after the warpgroup's named-barrier sync.
//
// LORA: each tile's K/64 NF4 k-blocks are followed by r_blocks tail k-blocks of the low-rank term U . B_cat^T
// (U = X . A_cat^T, 16-bit [M, R]; B_cat 16-bit [N, R], the scaling folded in).  A tail stage is two TMA loads in
// the 16-bit GEMM's layout -- U at (64 r, m0) into the A region, B_cat at (64 r, n0) into the W region -- and
// thread 0 completes its full barrier with the expect_tx of the whole stage and its second arrival.  No
// dequantisation, no proxy fence, no named-barrier sync; the raw ring counts base k-blocks only.  All 128 threads
// still wait for each tail stage to be free, so that none of them is ever more than one stage ahead of the ring.
template <bool LORA = false>
__device__ __forceinline__ void gemm_nf4_producer(const CUtensorMap* tm_a, const CUtensorMap* tm_codes,
                                                  const float* __restrict__ absmax, const GemmTiles& tl, int N,
                                                  int kblocks, uint32_t sb, uint32_t full_bar, uint32_t empty_bar,
                                                  const CUtensorMap* tm_u = nullptr,
                                                  const CUtensorMap* tm_bl = nullptr, int r_blocks = 0) {
  using P = GemmPlan<true>;
  const int p = static_cast<int>(threadIdx.x) - 256;
  const uint32_t raw0 = sb + P::RAW_OFFSET;
  const uint32_t raw_bar = empty_bar + 8u * P::STAGES;
  const uint32_t table = sb + P::TABLE_OFFSET;
  const int total = tl.count * kblocks;
  int ld = 0, ld_tile = 0, ld_kb = 0;   // thread 0: the next raw load (global k-block index, its tile and k-block)
  auto load_raw = [&]() {
    const int slot = ld % GEMM_NF4_RAW;
    const int tile = tl.first + ld_tile * tl.stride;
    const int n0 = (tile % tl.n_tiles) * GEMM_BN;
    const uint32_t dst = raw0 + slot * GEMM_NF4_RAW_BYTES, bar = raw_bar + 8u * slot;
    mbar_expect_tx(bar, GEMM_NF4_RAW_BYTES);
    tma_load_2d(dst, tm_codes, bar, ld_kb * (GEMM_BK / 2), n0);
    bulk_load_1d(dst + GEMM_NF4_CODE_BYTES, absmax + static_cast<size_t>(ld_kb) * N + n0, GEMM_BN * 4, bar);
    ++ld;
    if (++ld_kb == kblocks) { ld_kb = 0; ++ld_tile; }
  };
  if (p == 0) {
    tma_prefetch_desc(tm_a);
    tma_prefetch_desc(tm_codes);
    if constexpr (LORA) {
      tma_prefetch_desc(tm_u);
      tma_prefetch_desc(tm_bl);
    }
    while (ld < total && ld < GEMM_NF4_RAW) load_raw();
  }
  int stage = 0, slot = 0;
  uint32_t phase = 0, raw_phase = 0;
  for (int i = 0; i < tl.count; ++i) {
    const int m0 = ((tl.first + i * tl.stride) / tl.n_tiles) * GEMM_BM;
    for (int kb = 0; kb < kblocks; ++kb) {
      mbar_wait(empty_bar + 8u * stage, phase ^ 1u);
      const uint32_t dst = sb + stage * GEMM_STAGE_BYTES;
      const uint32_t fb = full_bar + 8u * stage;
      if (p == 0) {
        mbar_expect_tx(fb, GEMM_A_BYTES);
        tma_load_2d(dst, tm_a, fb, kb * GEMM_BK, m0);
      }
      mbar_wait(raw_bar + 8u * slot, raw_phase);
      const uint32_t src = raw0 + slot * GEMM_NF4_RAW_BYTES;
      const uint4 c0 = ld_shared_v4(src + 32 * p), c1 = ld_shared_v4(src + 32 * p + 16);
      const float s = ld_shared_f32(src + GEMM_NF4_CODE_BYTES + 4 * p);
      const uint32_t words[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      const uint32_t row = dst + GEMM_A_BYTES + 128 * p;
#pragma unroll
      for (int c = 0; c < 8; ++c) {   // 16-byte chunk c = columns [8c, 8c + 8) = code bytes [4c, 4c + 4)
        uint32_t v[4];
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const uint32_t byte = (words[c] >> (8 * b)) & 0xffu;
          // exactly nf4_dequantize's single fp32 product, then the storage rounding of weights.to_storage: bfloat16
          // round-to-nearest-even, or (half) the +-65504 clamp and round-to-nearest, which cvt.rn.satfinite is
          // for every finite product
          const float lo = __fmul_rn(ld_shared_const_f32(table + ((byte >> 4) << 2)), s);
          const float hi = __fmul_rn(ld_shared_const_f32(table + ((byte & 15u) << 2)), s);
          v[b] = pack_h16x2(lo, hi);
        }
        st_shared_v4(row + ((c ^ (p & 7)) << 4), v[0], v[1], v[2], v[3]);
      }
      fence_proxy_async_smem();   // the W tile is read by wgmma (async proxy)
      named_bar_sync(GEMM_BAR_NF4, 128);
      if (p == 0) {
        mbar_arrive(fb);
        if (ld < total) load_raw();   // into the slot every producer has just read
      }
      if (++stage == P::STAGES) { stage = 0; phase ^= 1u; }
      if (++slot == GEMM_NF4_RAW) { slot = 0; raw_phase ^= 1u; }
    }
    if constexpr (LORA) {
      const int n0 = ((tl.first + i * tl.stride) % tl.n_tiles) * GEMM_BN;
      for (int r = 0; r < r_blocks; ++r) {
        // every producer thread waits, although only thread 0 loads: a thread that skipped these waits would reach
        // the next tile's NF4 stages up to r_blocks positions ahead, and from STAGES positions on its parity wait
        // could pass on a phase that completed a whole ring earlier
        mbar_wait(empty_bar + 8u * stage, phase ^ 1u);
        if (p == 0) {
          const uint32_t dst = sb + stage * GEMM_STAGE_BYTES;
          const uint32_t fb = full_bar + 8u * stage;
          mbar_expect_tx(fb, GEMM_STAGE_BYTES);
          tma_load_2d(dst, tm_u, fb, r * GEMM_BK, m0);
          tma_load_2d(dst + GEMM_A_BYTES, tm_bl, fb, r * GEMM_BK, n0);
          mbar_arrive(fb);
        }
        if (++stage == P::STAGES) { stage = 0; phase ^= 1u; }
      }
    }
  }
}

// The kernel body: gemm_h16_wgmma_kernel, and (LORA) gemm_nf4_lora_kernel.  NF4 = false: W is a 16-bit [N,K] map.
// NF4 = true: tm_b is the uint8 code map [N,K/2] (box 32 x 128) and absmax the block scales [K/64, N]
// (gemm_nf4_producer).  LORA: the consumers run K/64 + r_blocks k-blocks per tile, the tail ones over U and B_cat.
template <int EPI, bool TL, bool NF4, int BN, bool LORA>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tm_a, const CUtensorMap& tm_b, const CUtensorMap& tm_out,
                                          h16* __restrict__ out, const float* __restrict__ bias,
                                          const h16* __restrict__ resid, int M, int N, int K,
                                          const int* __restrict__ m_dev, const float* __restrict__ absmax,
                                          const CUtensorMap* tm_u, const CUtensorMap* tm_bl, int r_blocks) {
  using P = GemmPlan<NF4, BN>;
  static_assert(!epi_is_glu(EPI) || BN == 128, "the gated epilogues pair gate and up within a 128-row W tile");
  static_assert(!LORA || (NF4 && !TL), "the low-rank tail rides on the NF4 producer");
  if (m_dev != nullptr) M = __ldg(m_dev);   // device-resident row count (packed token layout)
  const GemmTiles tl = gemm_tiles<BN>(M, N);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;   // the swizzled tiles need a 1024-byte aligned base
  const uint32_t full_bar = sb + P::BAR_OFFSET;
  const uint32_t empty_bar = full_bar + 8u * P::STAGES;
  const int warp = threadIdx.x >> 5;
  const int kblocks = K / GEMM_BK;
  const int kb_tile = LORA ? kblocks + r_blocks : kblocks;   // the k-blocks of one tile in the ring

  if (threadIdx.x == 0) {
    for (int s = 0; s < P::STAGES; ++s) {
      mbar_init(full_bar + 8u * s, NF4 ? 2 : 1);   // NF4: the A bytes' expect_tx and the dequantisers' arrival
      mbar_init(empty_bar + 8u * s, 1);   // released by the one consumer whose tile the k-block belongs to
    }
    if constexpr (NF4)
      for (int s = 0; s < GEMM_NF4_RAW; ++s) mbar_init(empty_bar + 8u * (P::STAGES + s), 1);
    mbar_fence_init();
  }
  if constexpr (NF4)
    if (threadIdx.x < 16) st_shared_u32(sb + P::TABLE_OFFSET + 4 * threadIdx.x, kNf4CodeBits[threadIdx.x]);
  __syncthreads();

  long long* clk = (TL && blockIdx.x == 0) ? g_gemm_clock : nullptr;
  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(P::PRODUCER_REGS));
    if constexpr (NF4) {
      gemm_nf4_producer<LORA>(&tm_a, &tm_b, absmax, tl, N, kblocks, sb, full_bar, empty_bar, tm_u, tm_bl, r_blocks);
    } else if (warp == 8 && elect_one()) {
      tma_prefetch_desc(&tm_a);
      tma_prefetch_desc(&tm_b);
      int stage = 0, n = 0;
      uint32_t phase = 0;
      for (int i = 0; i < tl.count; ++i) {
        const int tile = tl.first + i * tl.stride;
        const int m0 = (tile / tl.n_tiles) * GEMM_BM, n0 = (tile % tl.n_tiles) * BN;
        for (int kb = 0; kb < kblocks; ++kb, ++n) {
          mbar_wait(empty_bar + 8u * stage, phase ^ 1u);
          const uint32_t dst = sb + stage * P::STAGE_BYTES;
          const uint32_t fb = full_bar + 8u * stage;
          mbar_expect_tx(fb, P::STAGE_BYTES);
          tma_load_2d(dst, &tm_a, fb, kb * GEMM_BK, m0);
          tma_load_2d(dst + GEMM_A_BYTES, &tm_b, fb, kb * GEMM_BK, n0);
          if (TL && clk != nullptr && n < 256) clk[n] = clock64();
          if (++stage == P::STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(P::CONSUMER_REGS));
  const int wg = warp >> 2;
  const int t = threadIdx.x & 127;
  const int quad = t & 3;
  const int r_lo = 16 * (t >> 5) + ((t & 31) >> 2);   // row of acc[h][4j + {0,1}] in its 64-row half
  const uint32_t stg = sb + P::OUT_OFFSET + wg * (P::OUT_BOXES * GEMM_OUT_BOX);
  const uint32_t bias_slot = sb + P::BIAS_OFFSET + wg * (BN * 4);
  // stmatrix row address of this lane in the staging tile, for the four matrices (group j0 + i / 2, rows + 8 (i % 2))
  // of groups j0, j0 + 1 (j0 even) at j0 = 0: lane 8i + k gives row 16 (t / 32) + 8 (i % 2) + k, whose unit
  // (i / 2) sits at (i / 2) ^ k.  The staging tile is 1024-byte aligned, so the swizzle of a later j0 is an XOR of
  // this address with ((j0 & 7) << 4).
  const int lane = t & 31;
  const uint32_t stm_addr = stg + (16 * (t >> 5) + 8 * ((lane >> 3) & 1) + (lane & 7)) * 128 +
                            ((((lane >> 4) ^ lane) & 7) << 4);
  int retired = 0;
  // Turn i (the CTA's i-th tile) belongs to consumer i % 2.  The hand-over into turn i (1 <= i < count) is one
  // arrive by the consumer of turn i - 1 after issuing its main loop and one sync by the consumer of turn i
  // before starting its own: every arrive has its sync, and with 0 or 1 tiles nobody waits.
  for (int i = wg; i < tl.count; i += 2) {
    const int tile = tl.first + i * tl.stride;
    const int m0 = (tile / tl.n_tiles) * GEMM_BM, n_blk = tile % tl.n_tiles;
    // the tile's bias, loaded here and written to the consumer's slot after the main loop (threads t < BN / 2, one
    // pair each); without a bias the slot holds -0, which leaves every sum as it is, -0 included
    float2 bias_pair = make_float2(-0.0f, -0.0f);
    if constexpr (!epi_is_glu(EPI))
      if (bias != nullptr && t < BN / 2) bias_pair = __ldg(reinterpret_cast<const float2*>(bias + n_blk * BN) + t);
    float acc[2][BN / 2];   // rows [64 h, 64 h + 64) of the tile
#pragma unroll
    for (int x = 0; x < BN / 2; ++x) acc[0][x] = acc[1][x] = 0.0f;
    if (i > 0) named_bar_sync(GEMM_BAR_TURN + wg, 256);
    // this tile's k-blocks follow the i * kb_tile ones of the earlier turns in the ring
    const int it = i * kb_tile;
    int stage = it % P::STAGES;
    uint32_t phase = (it / P::STAGES) & 1u;
    int prev = -1;
    for (int kb = 0; kb < kb_tile; ++kb) {
      mbar_wait(full_bar + 8u * stage, phase);
      const uint32_t a_addr = sb + stage * P::STAGE_BYTES;
      const uint64_t a0 = make_smem_desc_sw128(a_addr), a1 = make_smem_desc_sw128(a_addr + 64 * 128);
      const uint64_t b_desc = make_smem_desc_sw128(a_addr + GEMM_A_BYTES);
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BK / 16; ++k) {
        if constexpr (BN == 192) {
          wgmma_64x192_ss(acc[0], a0 + 2u * k, b_desc + 2u * k, (kb | k) != 0);
          wgmma_64x192_ss(acc[1], a1 + 2u * k, b_desc + 2u * k, (kb | k) != 0);
        } else {
          wgmma_64x128_ss(acc[0], a0 + 2u * k, b_desc + 2u * k, (kb | k) != 0);
          wgmma_64x128_ss(acc[1], a1 + 2u * k, b_desc + 2u * k, (kb | k) != 0);
        }
      }
      wgmma_commit();
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      // keep one stage of MMAs in flight: the previous one has finished reading its operands
      wgmma_wait<1>();
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      if (prev >= 0 && t == 0) mbar_arrive(empty_bar + 8u * prev);
      if (TL && clk != nullptr && wg == 0 && t == 0 && retired < 256) clk[256 + retired] = clock64();
      ++retired;
      prev = stage;
      if (++stage == P::STAGES) { stage = 0; phase ^= 1u; }
    }
    if (i + 1 < tl.count) named_bar_arrive(GEMM_BAR_TURN + (wg ^ 1), 256);   // the other consumer's turn
    wgmma_wait<0>();
    reg_fence(acc[0]);
    reg_fence(acc[1]);
    if (t == 0) mbar_arrive(empty_bar + 8u * prev);
    if (TL && clk != nullptr && wg == 0 && t == 0 && i / 2 < 256) clk[512 + i / 2] = clock64();
    // Every thread of this warpgroup left the slot's previous tile behind before the turn sync above (i >= 2).
    if constexpr (!epi_is_glu(EPI))
      if (t < BN / 2) st_shared_f32x2(bias_slot + 8 * t, bias_pair);

    // Epilogue: fp32 acc (+ bias, then erf-GELU | + residual | the gated activation), rounded to h16 pairs.  A tile
    // inside the device rows goes out through the staging tile (128-byte swizzle, the layout of the store map:
    // 16-byte unit u of row r sits at unit u ^ (r & 7), so that the eight rows of a matrix hit distinct banks) and
    // TMA, with no test or global address inside its element loop; the last row tile crossing M stores its rows
    // from registers.
    const bool staged = m0 + GEMM_BM <= M;
    if (staged && t == 0) tma_store_wait_read<0>();   // the previous tile's stores have read the staging tile
    named_bar_sync(GEMM_BAR_STAGE + wg, 128);          // ... and the bias slot is written
    // the output pair of acc[h][4j + 2 half + {0, 1}]: row 64 h + r_lo + 8 half, columns 8 j + 2 quad + {0, 1} of
    // the tile (the gated epilogues: of the 64-column output block); b = the bias pair of group j, res = the
    // residual pair
    auto out_pair = [&](int h, int j, int half, float2 b, uint32_t res) -> uint32_t {
      if constexpr (epi_is_glu(EPI)) {
        const float g0 = acc[h][4 * j + 2 * half], g1 = acc[h][4 * j + 2 * half + 1];
        const float u0 = acc[h][4 * (j + 8) + 2 * half], u1 = acc[h][4 * (j + 8) + 2 * half + 1];
        if constexpr (EPI == EPI_GEGLU) return pack_h16x2(gelu_erf_fast(g0) * u0, gelu_erf_fast(g1) * u1);
        else return pack_h16x2(silu(g0) * u0, silu(g1) * u1);
      } else {
        float v0 = acc[h][4 * j + 2 * half] + b.x, v1 = acc[h][4 * j + 2 * half + 1] + b.y;
        if constexpr (EPI == EPI_BIAS_GELU) {
          v0 = gelu_erf_fast(v0);
          v1 = gelu_erf_fast(v1);
        }
        if constexpr (EPI == EPI_BIAS_RESID) {
          const float2 rv = unpack_h16x2(res);
          v0 += rv.x;
          v1 += rv.y;
        }
        return pack_h16x2(v0, v1);
      }
    };
    constexpr int GROUPS = epi_is_glu(EPI) ? 8 : BN / 8;   // 8-column output groups
    const int n_out = epi_is_glu(EPI) ? N / 2 : N;
    const int col0 = n_blk * (epi_is_glu(EPI) ? GEMM_BN / 2 : BN) + 2 * quad;
    const h16* res_row = EPI == EPI_BIAS_RESID ? resid + static_cast<size_t>(m0 + r_lo) * N + col0 : nullptr;
    if (staged) {
      // Groups j0, j0 + 1 of both 64-row halves per step: 16 independent pairs, two stmatrix.x4, and the
      // accumulators of the step die as it is written.  The next step's bias (and residual) pairs are read first.
      const size_t rs8 = static_cast<size_t>(8) * N;   // residual rows 8 apart
      float2 b[2][2];
      uint32_t res[2][2][2][2] = {};   // [buffer][h][group of the step][half]
      auto load_step = [&](int s, int buf) {
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          b[buf][g] = epi_is_glu(EPI) ? make_float2(0.0f, 0.0f) : ld_shared_f32x2(bias_slot + 4 * (8 * (2 * s + g) + 2 * quad));
          if constexpr (EPI == EPI_BIAS_RESID)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int half = 0; half < 2; ++half)
                res[buf][h][g][half] =
                    __ldg(reinterpret_cast<const uint32_t*>(res_row + rs8 * (8 * h + half) + 8 * (2 * s + g)));
        }
      };
      load_step(0, 0);
#pragma unroll
      for (int s = 0; s < GROUPS / 2; ++s) {
        if (s + 1 < GROUPS / 2) load_step(s + 1, (s + 1) & 1);
        const int j0 = 2 * s, buf = s & 1;
        const uint32_t addr = (stm_addr ^ ((j0 & 7) << 4)) + (j0 >> 3) * GEMM_OUT_BOX;
#pragma unroll
        for (int h = 0; h < 2; ++h)
          stmatrix_x4(addr + h * 64 * 128, out_pair(h, j0, 0, b[buf][0], res[buf][h][0][0]),
                      out_pair(h, j0, 1, b[buf][0], res[buf][h][0][1]), out_pair(h, j0 + 1, 0, b[buf][1], res[buf][h][1][0]),
                      out_pair(h, j0 + 1, 1, b[buf][1], res[buf][h][1][1]));
      }
    } else {
#pragma unroll
      for (int j = 0; j < GROUPS; ++j) {
        const float2 b = epi_is_glu(EPI) ? make_float2(0.0f, 0.0f) : ld_shared_f32x2(bias_slot + 4 * (8 * j + 2 * quad));
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int r = 64 * h + r_lo + 8 * half;
            if (m0 + r >= M) continue;
            const size_t off = static_cast<size_t>(m0 + r) * n_out + col0 + 8 * j;
            const uint32_t res = EPI == EPI_BIAS_RESID ? *reinterpret_cast<const uint32_t*>(resid + off) : 0u;
            *reinterpret_cast<uint32_t*>(out + off) = out_pair(h, j, half, b, res);
          }
      }
    }
    if (staged) {
      fence_proxy_async_smem();   // the staging tile is read by the TMA (async proxy)
      named_bar_sync(GEMM_BAR_STAGE + wg, 128);
      if (t == 0) {
        if constexpr (epi_is_glu(EPI)) {
          tma_store_2d(&tm_out, stg, n_blk * (GEMM_BN / 2), m0);
        } else {
#pragma unroll
          for (int b = 0; b < P::OUT_BOXES; ++b) tma_store_2d(&tm_out, stg + b * GEMM_OUT_BOX, n_blk * BN + 64 * b, m0);
        }
        tma_store_commit();
      }
    }
    if (TL && clk != nullptr && wg == 0 && t == 0 && i / 2 < 256) clk[768 + i / 2] = clock64();
  }
  if (t == 0) tma_store_wait_all();   // the stores have read shared memory before the CTA leaves
}

template <int EPI, bool TL = false, bool NF4 = false, int BN = GEMM_BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_h16_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a,    // [M,K] box 64 x 128
                      const __grid_constant__ CUtensorMap tm_b,    // [N,K] box 64 x BN
                      const __grid_constant__ CUtensorMap tm_out,  // out [M,N] (GLU: [M,N/2]) box 64 x 128
                      h16* __restrict__ out, const float* __restrict__ bias, const h16* __restrict__ resid,
                      int M, int N, int K, const int* __restrict__ m_dev, const float* __restrict__ absmax) {
  gemm_body<EPI, TL, NF4, BN, false>(tm_a, tm_b, tm_out, out, bias, resid, M, N, K, m_dev, absmax, nullptr, nullptr, 0);
}

// y = epi(A . dequant(W)^T + U . B_cat^T + bias [+ resid]): the NF4 GEMM with r_blocks = R/64 extra k-blocks per
// tile.  Each output sums the same products in the same order as the 16-bit GEMM over the K-concatenated operands
// [A | U] and [round16(dequant(W)) | B_cat].
template <int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_nf4_lora_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                     const __grid_constant__ CUtensorMap tm_out, h16* __restrict__ out,
                     const float* __restrict__ bias, const h16* __restrict__ resid, int M, int N, int K,
                     const int* __restrict__ m_dev, const float* __restrict__ absmax,
                     const __grid_constant__ CUtensorMap tm_u,    // U [M, >= R] box 64 x 128
                     const __grid_constant__ CUtensorMap tm_bl,   // B_cat [N, R] box 64 x 128
                     int r_blocks) {
  gemm_body<EPI, false, true, GEMM_BN, true>(tm_a, tm_b, tm_out, out, bias, resid, M, N, K, m_dev, absmax, &tm_u,
                                             &tm_bl, r_blocks);
}

}  // namespace b2e
