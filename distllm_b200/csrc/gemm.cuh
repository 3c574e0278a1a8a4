// Warp-specialised h16 GEMM for sm_90a:  out[M,N] = epi(A[M,K] . W[N,K]^T + bias)
//
//   warp 8      TMA producer (one elected lane): 128 x 64 A tile and 128 x 64 W tile per stage into a
//               128B-swizzled shared-memory ring
//   warps 0-7   two consumer warpgroups, 64 output rows each: wgmma m64n128k16 with both operands read
//               from shared memory, fp32 accumulators in registers; the epilogue (+bias, erf-GELU |
//               +residual | gated activation) runs on those registers and stores h16 pairs
//
// One CTA per 128 x 128 output tile; three 32 KiB stages keep two CTAs resident per SM, so the epilogue
// of one overlaps the main loop of the other.
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
constexpr int GEMM_STAGES = 3;
constexpr int GEMM_THREADS = 288;   // two consumer warpgroups + the producer warp
constexpr int GEMM_A_BYTES = GEMM_BM * GEMM_BK * 2;
constexpr int GEMM_STAGE_BYTES = GEMM_A_BYTES + GEMM_BN * GEMM_BK * 2;
constexpr int GEMM_BAR_OFFSET = GEMM_STAGES * GEMM_STAGE_BYTES;
constexpr int GEMM_SMEM_BYTES = GEMM_BAR_OFFSET + 64 + 1024;   // + slack to align the ring to 1024 B
static_assert(2 * GEMM_SMEM_BYTES <= 232448, "two CTAs per SM");

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
// the block's MMAs have been retired); 4 x 256 int64
__device__ long long* g_gemm_clock = nullptr;

template <int EPI, bool TL = false>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
gemm_h16_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a,    // [M,K] box 64 x 128
                      const __grid_constant__ CUtensorMap tm_b,    // [N,K] box 64 x 128
                      h16* __restrict__ out, const float* __restrict__ bias, const h16* __restrict__ resid,
                      int M, int N, int K, const int* __restrict__ m_dev) {
  if (m_dev != nullptr) M = __ldg(m_dev);   // device-resident row count (packed token layout)
  // one-dimensional grid, N tiles fastest: the CTAs resident together share their A rows in L2
  const int n_blk = static_cast<int>(blockIdx.x % (N / GEMM_BN)), m_blk = static_cast<int>(blockIdx.x / (N / GEMM_BN));
  if (m_blk * GEMM_BM >= M) return;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sb = (raw + 1023u) & ~1023u;   // the swizzled tiles need a 1024-byte aligned base
  const uint32_t full_bar = sb + GEMM_BAR_OFFSET;
  const uint32_t empty_bar = full_bar + 8u * GEMM_STAGES;
  const int warp = threadIdx.x >> 5;
  const int kblocks = K / GEMM_BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < GEMM_STAGES; ++s) {
      mbar_init(full_bar + 8u * s, 1);
      mbar_init(empty_bar + 8u * s, 2);   // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  long long* clk = (TL && blockIdx.x == 0) ? g_gemm_clock : nullptr;
  if (warp == 8) {
    if (elect_one()) {
      tma_prefetch_desc(&tm_a);
      tma_prefetch_desc(&tm_b);
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(empty_bar + 8u * stage, phase ^ 1u);
        const uint32_t dst = sb + stage * GEMM_STAGE_BYTES;
        const uint32_t fb = full_bar + 8u * stage;
        mbar_expect_tx(fb, GEMM_STAGE_BYTES);
        tma_load_2d(dst, &tm_a, fb, kb * GEMM_BK, m_blk * GEMM_BM);
        tma_load_2d(dst + GEMM_A_BYTES, &tm_b, fb, kb * GEMM_BK, n_blk * GEMM_BN);
        if (TL && clk != nullptr && kb < 256) clk[kb] = clock64();
        if (++stage == GEMM_STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  const int wg = warp >> 2;                  // consumer warpgroup: rows [64 wg, 64 wg + 64) of the tile
  const int t = threadIdx.x & 127;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
  int stage = 0;
  uint32_t phase = 0;
  int prev = -1;
  for (int kb = 0; kb < kblocks; ++kb) {
    mbar_wait(full_bar + 8u * stage, phase);
    const uint32_t a_addr = sb + stage * GEMM_STAGE_BYTES + wg * (64 * 128);
    const uint64_t a_desc = make_smem_desc_sw128(a_addr);
    const uint64_t b_desc = make_smem_desc_sw128(sb + stage * GEMM_STAGE_BYTES + GEMM_A_BYTES);
    reg_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_64x128_ss(acc, a_desc + 2u * k, b_desc + 2u * k, (kb | k) != 0);
    wgmma_commit();
    reg_fence(acc);
    // keep one stage of MMAs in flight: the previous one has finished reading its operands
    wgmma_wait<1>();
    reg_fence(acc);
    if (prev >= 0 && t == 0) mbar_arrive(empty_bar + 8u * prev);
    if (TL && clk != nullptr && threadIdx.x == 0 && kb < 256) clk[256 + kb] = clock64();
    prev = stage;
    if (++stage == GEMM_STAGES) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  reg_fence(acc);

  const int r_lo = m_blk * GEMM_BM + wg * 64 + 16 * (t >> 5) + ((t & 31) >> 2);
  const int c_in = 2 * (t & 3);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int row = r_lo + 8 * half;
    if (row >= M) continue;
    if constexpr (epi_is_glu(EPI)) {
      const int n_out = N / 2;
      h16* orow = out + static_cast<size_t>(row) * n_out + n_blk * (GEMM_BN / 2);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float g0 = acc[4 * j + 2 * half], g1 = acc[4 * j + 2 * half + 1];
        const float u0 = acc[4 * (j + 8) + 2 * half], u1 = acc[4 * (j + 8) + 2 * half + 1];
        float v0, v1;
        if (EPI == EPI_GEGLU) {
          v0 = gelu_erf_fast(g0) * u0;
          v1 = gelu_erf_fast(g1) * u1;
        } else {
          v0 = silu(g0) * u0;
          v1 = silu(g1) * u1;
        }
        *reinterpret_cast<uint32_t*>(orow + 8 * j + c_in) = pack_h16x2(v0, v1);
      }
    } else {
      const int col0 = n_blk * GEMM_BN + c_in;
      h16* orow = out + static_cast<size_t>(row) * N + col0;
      const h16* rrow = (EPI == EPI_BIAS_RESID) ? resid + static_cast<size_t>(row) * N + col0 : nullptr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float v0 = acc[4 * j + 2 * half], v1 = acc[4 * j + 2 * half + 1];
        if (bias != nullptr) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col0 + 8 * j));
          v0 += b.x;
          v1 += b.y;
        }
        if (EPI == EPI_BIAS_GELU) {
          v0 = gelu_erf_fast(v0);
          v1 = gelu_erf_fast(v1);
        }
        if (EPI == EPI_BIAS_RESID) {
          const float2 r = unpack_h16x2(*reinterpret_cast<const uint32_t*>(rrow + 8 * j));
          v0 += r.x;
          v1 += r.y;
        }
        *reinterpret_cast<uint32_t*>(orow + 8 * j) = pack_h16x2(v0, v1);
      }
    }
  }
}

}  // namespace b2e
