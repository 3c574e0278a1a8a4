// Exact inner-product top-k, fast path for a float32 corpus: the scan runs on the tensor cores in TF32, the
// k best are then decided on exact fp32 dot products of a small candidate set.  Same contract as topk.cuh
// (faiss.IndexFlatIP.search as called from distllm/rag/search.py:280-336): fp32 scores, descending, ties by
// ascending row id.
//
//   1. tf32_scan_kernel      S[n, q] ~ <corpus_n, query_q> for all rows and up to 16 queries per pass: persistent
//                            CTAs, TMA streams 128-row x 32-float corpus tiles (and the matching 16 x 32 query
//                            slice) through an 8-stage ring, one warpgroup runs wgmma m64n16k8 (tf32) on both
//                            64-row halves of a tile and writes the 128 x 16 accumulator to the score matrix.  HBM-bound:
//                            N * H * 4 bytes in, N * 64 bytes out.
//   2. score_hist_kernel     per query a 2048-bin LINEAR histogram of S over [-R, R], R = |q| * max_n |corpus_n|
//                            (Cauchy-Schwarz: no score lies outside).
//   3. score_threshold_kernel  bin holding the k-th largest approximate score -> threshold = its lower edge - 2 eps,
//                            eps = 1.5 * 2^-9 * R.  The wgmma reads each fp32 operand as TF32 by TRUNCATION (low 13
//                            mantissa bits dropped; measured on an H100 80GB HBM3, tests/test_gpu_retrieval_tf32.py):
//                            relative error < 2^-10 per operand, so conversion moves S by < 2^-9 * sum |q_i c_i|
//                            <= 2^-9 * |q| |c| (Cauchy-Schwarz).  The products (22 bits) are exact in fp32; summing H
//                            of them in fp32, in any order, adds at most (H - 1) * 2^-23 * sum |q_i c_i| < 2^-10 * R
//                            for H <= 8192: the other 0.5 * 2^-9 * R of eps.  Measured |S - exact| / eps: at most 0.47
//                            on inputs rounded maximally (H = 128 .. 8192), 0.11 on random rows; the accumulation
//                            stayed within 0.6 % of its bound.  Every row whose EXACT score could reach the exact k-th
//                            best has S >= threshold.
//   4. score_select_kernel   rows with S >= threshold -> candidate list (at most TC_MAX_CAND per query).
//   5. exact_rescore_kernel  fp32 dot product of every candidate, bitonic sort (score desc, row asc), top k out.
//
// A query whose candidate list overflows (scores packed closer than eps around the k-th: duplicates, degenerate
// corpora) raises a device-side flag; the exact FMA scan of topk.cuh then runs for the call (it returns at once
// when the flag is clear), so the result never depends on the approximation.
//
// Squared-L2 search (the <L2 = true> instantiations; faiss.IndexFlatL2 of distllm/rag/search.py:402-666): the
// scan is the same kernel, S ~ q.x.  Rows are ranked on v = S - n/2, n = fl(|x|^2) from row_norm2_kernel (stored
// with the index), which orders them like -D because D = |q|^2 + |x|^2 - 2 q.x = |q|^2 - 2 v_exact.  With M >=
// every |x| (corpus_max_norm) and r = |q| M:
//   range      v in [-r - M^2/2, r]: the histogram's bins cover that interval instead of [-r, r] (M^2 must bound
//              every stored n too, so that a k-th value in the lowest bin selects every row and overflows).
//   eps_S      |S - q.x| <= 1.5 * 2^-9 * r, as above.
//   norm       n sums H squares in fp32 (depth < H): |n - |x|^2| <= 1.01 H 2^-24 |x|^2 <= H 2^-23 M^2, and v takes
//              half of it: at most H 2^-24 M^2.
//   subtract   v = fl(S - n/2) (n/2 is exact): one rounding of a value below r + M^2/2, at most 2^-23 (r + M^2).
//   distance   the decision computes D~ = fl(sum (q_i - x_i)^2) directly: each difference rounded once, a sum of
//              non-negative terms of depth < H, so |D~ - D| <= (H + 2) 2^-24 D (1.01) <= H 2^-23 (|q| + M)^2 = e_D.
// With d = eps_S + H 2^-24 M^2 + 2^-23 (r + M^2) bounding |v - v_exact|: at least `need` rows have v >= edge, so
// D~ <= |q|^2 - 2 (edge - d) + e_D for each of them, while a row with v < thr has D~ > |q|^2 - 2 (thr + d) - e_D.
// thr = edge - 2 d - e_D (minus one bin width for the bin arithmetic, as above) therefore leaves out only rows
// whose computed distance is STRICTLY larger than that of `need` candidates: the decision on D~ (ascending, ties
// by ascending row id) is the one the exact CUDA-core scan makes.  tc_prepare_queries_kernel<true> stores
// eps = d + e_D / 2, so the threshold keeps the inner-product form edge - 2 eps - bin.
#pragma once

#include "common.cuh"

namespace b2e {

constexpr int TC_ROWS = 128;                 // corpus rows per tile (MMA M)
constexpr int TC_NQ = 16;                    // queries per pass (MMA N)
constexpr int TC_KB = 32;                    // floats per k-block = one 128-byte swizzle row
constexpr int TC_STAGES = 8;
constexpr int TC_A_BYTES = TC_ROWS * TC_KB * 4;    // 16 KiB
constexpr int TC_B_BYTES = TC_NQ * TC_KB * 4;      // 2 KiB
constexpr int TC_STAGE_BYTES = TC_A_BYTES + TC_B_BYTES;
constexpr int TC_SMEM_BAR = TC_STAGES * TC_STAGE_BYTES;
constexpr int TC_THREADS = 160;              // warps 0-3: the MMA warpgroup, warp 4: TMA loader
constexpr int TC_BINS = 2048;
constexpr int TC_MAX_CAND = 4096;
constexpr int TC_SMEM_BYTES = TC_SMEM_BAR + 256 + 1024;   // + slack to align the ring to 1024 B
static_assert(TC_STAGE_BYTES % 1024 == 0, "swizzled tiles need 1024-byte alignment");

// scores [tiles * 128, 16]: row n, query q at n * 16 + q (rows >= N come out 0: the TMA zero-fills them)
__global__ void __launch_bounds__(TC_THREADS, 1)
tf32_scan_kernel(const __grid_constant__ CUtensorMap tm_corpus,    // [N, H] f32, box 32 x 128
                 const __grid_constant__ CUtensorMap tm_queries,   // [16, H] f32 (zero rows beyond nq), box 32 x 16
                 float* __restrict__ scores, long long tiles, int H) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5;
  const uint32_t full = sb + TC_SMEM_BAR;              // [STAGES]
  const uint32_t empty = full + 8 * TC_STAGES;         // [STAGES]
  const int kblocks = H / TC_KB;

  if (threadIdx.x == 0) {
    for (int i = 0; i < TC_STAGES; ++i) {
      mbar_init(full + 8u * i, 1);
      mbar_init(empty + 8u * i, 1);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      // ---------------------------------------------------------------- loader
      tma_prefetch_desc(&tm_corpus);
      tma_prefetch_desc(&tm_queries);
      uint32_t c = 0;
      for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        for (int kb = 0; kb < kblocks; ++kb, ++c) {
          const int st = c % TC_STAGES;
          const uint32_t use = c / TC_STAGES;
          if (use > 0) mbar_wait(empty + 8u * st, (use - 1) & 1u);
          const uint32_t fb = full + 8u * st;
          mbar_expect_tx(fb, TC_STAGE_BYTES);
          const uint32_t dst = sb + st * TC_STAGE_BYTES;
          tma_load_2d(dst, &tm_corpus, fb, kb * TC_KB, static_cast<int>(tile * TC_ROWS));
          tma_load_2d(dst + TC_A_BYTES, &tm_queries, fb, kb * TC_KB, 0);
        }
      }
    }
    return;
  }
  // ------------------------------------------------------------------ MMA warpgroup + epilogue
  const int t = threadIdx.x;
  uint32_t c = 0;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    float acc[2][8];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[hf][i] = 0.0f;
    for (int kb = 0; kb < kblocks; ++kb, ++c) {
      const int st = c % TC_STAGES;
      mbar_wait(full + 8u * st, (c / TC_STAGES) & 1u);
      const uint32_t a_addr = sb + st * TC_STAGE_BYTES;
      const uint64_t b_desc = make_smem_desc_sw128(a_addr + TC_A_BYTES);
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_KB / 8; ++k)   // 8 floats = 32 bytes per MMA: +2 in the descriptor's 16-byte units
#pragma unroll
        for (int hf = 0; hf < 2; ++hf)
          wgmma_64x16_tf32(acc[hf], make_smem_desc_sw128(a_addr + hf * (64 * 128)) + 2u * k, b_desc + 2u * k,
                           (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      if (t == 0) mbar_arrive(empty + 8u * st);
    }
    // accumulator layout (common.cuh): rows 16 (t / 32) + (t % 32) / 4 (+ 8), query columns 8 j + 2 (t % 4)
    const size_t r_lo = static_cast<size_t>(tile) * TC_ROWS + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int r8 = 0; r8 < 2; ++r8)
          *reinterpret_cast<float2*>(scores + (r_lo + 64 * hf + 8 * r8) * TC_NQ + 8 * j + 2 * (t & 3)) =
              make_float2(acc[hf][4 * j + 2 * r8], acc[hf][4 * j + 2 * r8 + 1]);
  }
}

// |row|^2 of every row (fp32, a fixed summation order) into norm2 [N] (nullable), and their maximum, what bounds
// every score by Cauchy-Schwarz, into *out.  One warp per row, atomicMax on the bit pattern (non-negative floats
// order like their integers).  out must be zeroed first.
__global__ void row_norm2_kernel(const float* __restrict__ x, long long N, int H, float* __restrict__ norm2,
                                 float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  float best = 0.0f;
  for (long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N;
       row += warps) {
    const float4* p = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * H);
    float s = 0.0f;
    for (int i = lane; i < H / 4; i += 32) {
      const float4 v = p[i];
      s = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, s))));
    }
    s = warp_sum(s);
    if (norm2 != nullptr && lane == 0) norm2[row] = s;
    best = fmaxf(best, s);
  }
  if (lane == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(best));
}

// per query: R = |q| * max_norm (score range), eps = TF32 error bound (L2: the margin of the file header, halved);
// zero-padded copy of the queries for the scan's B operand.  One CTA per query slot (16).
struct TcQuery {
  float r;        // every score lies in [-r, r] (L2: every v in [-r - shift, r], shift = max_norm^2 / 2)
  float eps;
  float thr;      // filled by score_threshold_kernel
  int need;       // min(k, N): rows this query must return
};
template <bool L2 = false>
__global__ void tc_prepare_queries_kernel(const float* __restrict__ queries, int nq, int H, float max_norm,
                                          float* __restrict__ qpad, TcQuery* __restrict__ meta) {
  const int q = blockIdx.x;
  float s = 0.0f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const float v = q < nq ? queries[static_cast<size_t>(q) * H + i] : 0.0f;
    qpad[static_cast<size_t>(q) * H + i] = v;
    s = fmaf(v, v, s);
  }
  __shared__ float part[8];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.0f;
    for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) tot += part[i];
    // a hair above the true bound so that rounding in the norms themselves cannot put a score outside
    const float r = sqrtf(tot) * max_norm * 1.0001f + 1e-30f;
    meta[q].r = r;
    meta[q].eps = r * (1.5f / 512.0f);
    if constexpr (L2) {
      const float m2 = max_norm * max_norm;
      const float qm = sqrtf(tot) * 1.0001f + max_norm;
      const float d = r * (1.5f / 512.0f) + static_cast<float>(H) * 0x1p-24f * m2 + 0x1p-23f * (r + m2);
      meta[q].eps = (d + static_cast<float>(H) * 0x1p-24f * qm * qm) * 1.0001f;
    }
    meta[q].thr = -INFINITY;
    meta[q].need = 0;
  }
}

__device__ __forceinline__ int tc_bin(float s, float r) {
  // linear bins over [-r, r]; the comparison form keeps NaN (cannot occur for finite inputs) in bin 0
  const float u = (s + r) * (static_cast<float>(TC_BINS) * 0.5f) / r;
  int b = static_cast<int>(u);
  if (!(u > 0.0f)) b = 0;
  return b > TC_BINS - 1 ? TC_BINS - 1 : b;
}

// L2: the ranked value v = S - n/2 of the file header, rounded once (never contracted into an FMA, so the
// histogram and the selection see the same bits), and its linear bin over [lo, lo + BINS / scale]
__device__ __forceinline__ float l2_value(float s, float n2) { return __fsub_rn(s, __fmul_rn(0.5f, n2)); }
__device__ __forceinline__ int tc_bin_l2(float v, float lo, float scale) {
  const float u = (v - lo) * scale;
  int b = static_cast<int>(u);
  if (!(u > 0.0f)) b = 0;
  return b > TC_BINS - 1 ? TC_BINS - 1 : b;
}

// hist [16][TC_BINS] (zeroed before): shared-memory histograms per CTA, flushed with atomics.  L2: of
// v = S - norm2[row] / 2 over [-r - shift, r].
template <bool L2 = false>
__global__ void __launch_bounds__(512)
score_hist_kernel(const float* __restrict__ scores, long long N, int nq, const TcQuery* __restrict__ meta,
                  unsigned* __restrict__ hist, const float* __restrict__ norm2 = nullptr, float shift = 0.0f) {
  extern __shared__ unsigned sh[];   // [nq][TC_BINS]
  for (int i = threadIdx.x; i < nq * TC_BINS; i += blockDim.x) sh[i] = 0u;
  __shared__ float rr[TC_NQ], lo[TC_NQ];
  if (threadIdx.x < TC_NQ) {
    const float r = meta[threadIdx.x].r;
    rr[threadIdx.x] = L2 ? static_cast<float>(TC_BINS) / (2.0f * r + shift) : r;
    lo[threadIdx.x] = -r - shift;
  }
  __syncthreads();
  for (long long row = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; row < N;
       row += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4* p = reinterpret_cast<const float4*>(scores + static_cast<size_t>(row) * TC_NQ);
    float n2 = 0.0f;
    if constexpr (L2) n2 = norm2[row];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 v = p[i];
      const float s[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int q = 4 * i + j;
        if constexpr (L2) {
          if (q < nq) atomicAdd(&sh[q * TC_BINS + tc_bin_l2(l2_value(s[j], n2), lo[q], rr[q])], 1u);
        } else {
          if (q < nq) atomicAdd(&sh[q * TC_BINS + tc_bin(s[j], rr[q])], 1u);
        }
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nq * TC_BINS; i += blockDim.x)
    if (sh[i] != 0u) atomicAdd(&hist[i], sh[i]);
}

// one warp per query: walk the bins from the top until `need` rows are covered
template <bool L2 = false>
__global__ void score_threshold_kernel(const unsigned* __restrict__ hist, int nq, long long N, int k,
                                       TcQuery* __restrict__ meta, float shift = 0.0f) {
  const int q = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (q >= nq) return;
  const long long need = N < k ? N : k;
  long long acc = 0;
  int found = 0;
  for (int hi = TC_BINS - 1; hi >= 0; hi -= 32) {
    const int b = hi - lane;
    const unsigned c = b >= 0 ? hist[q * TC_BINS + b] : 0u;
    // inclusive prefix over lanes (lane 0 = highest bin of the group)
    unsigned run = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned n = __shfl_up_sync(0xffffffffu, run, o);
      if (lane >= o) run += n;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, acc + run >= need);
    if (hit != 0u) {
      found = hi - (__ffs(hit) - 1);
      break;
    }
    acc += __shfl_sync(0xffffffffu, run, 31);
  }
  if (lane == 0) {
    const float r = meta[q].r;
    if constexpr (L2) {
      const float bin = (2.0f * r + shift) / static_cast<float>(TC_BINS);
      meta[q].thr = (-r - shift + static_cast<float>(found) * bin) - 2.0f * meta[q].eps - bin;
    } else {
      const float edge = -r + static_cast<float>(found) * (2.0f * r / static_cast<float>(TC_BINS));
      // one extra bin width covers the rounding of the bin arithmetic itself
      meta[q].thr = edge - 2.0f * meta[q].eps - 2.0f * r / static_cast<float>(TC_BINS);
    }
    meta[q].need = static_cast<int>(need);
  }
}

// cand [16][TC_MAX_CAND] row ids, n_cand [16] (zeroed before); counts keep growing past the cap (overflow test).
// L2: rows with v = S - norm2[row] / 2 >= thr.
template <bool L2 = false>
__global__ void __launch_bounds__(512)
score_select_kernel(const float* __restrict__ scores, long long N, int nq, const TcQuery* __restrict__ meta,
                    unsigned* __restrict__ cand, unsigned* __restrict__ n_cand, const float* __restrict__ norm2 = nullptr) {
  __shared__ float thr[TC_NQ];
  if (threadIdx.x < TC_NQ) thr[threadIdx.x] = threadIdx.x < nq ? meta[threadIdx.x].thr : INFINITY;
  __syncthreads();
  for (long long row = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; row < N;
       row += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4* p = reinterpret_cast<const float4*>(scores + static_cast<size_t>(row) * TC_NQ);
    float n2 = 0.0f;
    if constexpr (L2) n2 = norm2[row];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 v = p[i];
      float s[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int q = 4 * i + j;
        if constexpr (L2) s[j] = l2_value(s[j], n2);
        if (s[j] >= thr[q]) {
          const unsigned pos = atomicAdd(&n_cand[q], 1u);
          if (pos < TC_MAX_CAND) cand[q * TC_MAX_CAND + pos] = static_cast<unsigned>(row);
        }
      }
    }
  }
}

// One CTA per query: exact fp32 score of every candidate, sort (score descending, row ascending), top k out.
// A list that overflowed or came out shorter than `need` raises *fallback (the exact scan then redoes the call).
// L2: the score is -D, D = sum (q_i - x_i)^2 in fp32, and D is written out (ascending; a short tail is +inf / -1).
template <bool L2 = false>
__global__ void __launch_bounds__(512)
exact_rescore_kernel(const unsigned* __restrict__ cand, const unsigned* __restrict__ n_cand,
                     const TcQuery* __restrict__ meta, const float* __restrict__ queries,
                     const float* __restrict__ corpus, int H, int k, float* __restrict__ out_score,
                     int64_t* __restrict__ out_index, int* __restrict__ fallback) {
  extern __shared__ __align__(16) unsigned long long keys[];   // [n_pow2] then the query [H] f32
  const int q = blockIdx.x;
  const unsigned n_raw = n_cand[q];
  const int need = meta[q].need;
  if (n_raw > TC_MAX_CAND || static_cast<int>(n_raw) < need) {
    if (threadIdx.x == 0) atomicExch(fallback, 1);
    return;
  }
  const int n = static_cast<int>(n_raw);
  int n_pow2 = 2;   // at least 16 bytes of keys: the query copy behind them is read as float4
  while (n_pow2 < n) n_pow2 <<= 1;
  float* qs = reinterpret_cast<float*>(keys + n_pow2);
  for (int i = threadIdx.x; i < H; i += blockDim.x) qs[i] = queries[static_cast<size_t>(q) * H + i];
  for (int i = n + threadIdx.x; i < n_pow2; i += blockDim.x) keys[i] = 0ull;   // sorts last
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int c = threadIdx.x >> 5; c < n; c += blockDim.x >> 5) {
    const unsigned row = cand[q * TC_MAX_CAND + c];
    const float4* p = reinterpret_cast<const float4*>(corpus + static_cast<size_t>(row) * H);
    float s = 0.0f;
    if constexpr (L2) {
      // unrolled by two: at the compiler's own choice (four) this loop spills
#pragma unroll 2
      for (int i = lane; i < H / 4; i += 32) {
        const float4 v = p[i];
        const float4 w = *reinterpret_cast<const float4*>(qs + 4 * i);
        const float dx = w.x - v.x, dy = w.y - v.y, dz = w.z - v.z, dw = w.w - v.w;
        s = fmaf(dx, dx, fmaf(dy, dy, fmaf(dz, dz, fmaf(dw, dw, s))));
      }
    } else {
      for (int i = lane; i < H / 4; i += 32) {
        const float4 v = p[i];
        const float4 w = *reinterpret_cast<const float4*>(qs + 4 * i);
        s = fmaf(v.x, w.x, fmaf(v.y, w.y, fmaf(v.z, w.z, fmaf(v.w, w.w, s))));
      }
    }
    s = warp_sum(s);
    if constexpr (L2) s = -s;
    if (lane == 0) {
      // order-preserving key of the float (larger score = larger key, never 0), then the inverted row id
      unsigned u = __float_as_uint(s);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
      if (u == 0u) u = 1u;
      keys[c] = (static_cast<unsigned long long>(u) << 32) | static_cast<unsigned long long>(~row);
    }
  }
  __syncthreads();
  for (int size = 2; size <= n_pow2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
        const int j = i ^ stride;
        if (j > i) {
          const bool desc = (i & size) == 0;
          const unsigned long long a = keys[i], b = keys[j];
          if (desc ? a < b : a > b) {
            keys[i] = b;
            keys[j] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    float s = -INFINITY;
    int64_t idx = -1;
    if (i < n) {
      const unsigned long long key = keys[i];
      unsigned u = static_cast<unsigned>(key >> 32);
      u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
      s = __uint_as_float(u);
      idx = static_cast<int64_t>(~static_cast<unsigned>(key & 0xffffffffu));
    }
    out_score[static_cast<size_t>(q) * k + i] = L2 ? -s : s;
    out_index[static_cast<size_t>(q) * k + i] = idx;
  }
}

}  // namespace b2e
