// HBM-bound row kernels of the embedding path (one warp per row, 16-byte vector accesses):
//   embedding gather + LayerNorm, LayerNorm, LayerNorm fused with masked-mean pooling,
//   pool-weight construction (including the reference's cross-row mask quirk), standalone pooling,
//   last-token gather, L2 normalise and the adjacent-cosine distance used by the semantic splitter.
#pragma once

#include <cuda_fp16.h>

#include "common.cuh"

namespace b2e {

constexpr int ROW_WARPS = 8;
constexpr int ROW_THREADS = ROW_WARPS * 32;

// A row of H columns is held as row_passes(H) passes of 256 columns, lane owning columns v*256 + lane*8 .. +8 of
// pass v.  The row kernels are instantiated per H (DISPATCH_H): 256 x {1,2,3,4,5,8,10,16}, 384, 640, 960 and 1152.  A
// width with a remainder ends on a partial pass of (H % 256) / 8 lanes: a 128-column half pass (384, 640, 1152: lanes
// 16-31 off) or a 192-column pass (960: lanes 24-31 off).  Off lanes (row_lane_on) hold zeros, load and store nothing
// and add nothing to the row statistics, which still divide by H.  For H % 256 == 0 the predicate is the constant true
// and the kernels are the same code as with whole passes only.
__host__ __device__ constexpr int row_passes(int H) { return (H + 255) / 256; }
template <int H>
__device__ __forceinline__ bool row_lane_on(int v, int lane) {
  return H % 256 == 0 || v < H / 256 || lane < (H % 256) / 8;
}

// ---- 8-element vector load/store helpers (lane owns columns v*256 + lane*8 .. +8)
__device__ __forceinline__ void load8(const bf16* p, float (&v)[8]) {   // bf16 hidden states at the API
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __bfloat1622float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void load8(const __half* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(h[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8(h16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_h16x2(v[0], v[1]);
  u.y = pack_h16x2(v[2], v[3]);
  u.z = pack_h16x2(v[4], v[5]);
  u.w = pack_h16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
#ifndef B2E_STORAGE_BF16   // (in the bfloat16 build the overload above already is the bf16 store)
__device__ __forceinline__ void store8(bf16* p, const float (&v)[8]) {   // caller-provided bf16 outputs
  __nv_bfloat162 h[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(h);
}
#endif
__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void zero8(float (&v)[8]) {   // the values of an off lane (row_lane_on)
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.0f;
}

// LayerNorm of one row held as NV x 8 values per lane (biased variance, like torch.layer_norm); the values of off
// lanes (row_lane_on) are zeros.  BIAS == false: no bias (ESMC's q_ln / k_ln), beta is not read.
template <int H, bool BIAS = true>
__device__ __forceinline__ void warp_layernorm(float (&x)[row_passes(H)][8], const float* __restrict__ gamma,
                                               const float* __restrict__ beta, int lane, float eps) {
  constexpr int NV = row_passes(H);
  constexpr float inv_h = 1.0f / static_cast<float>(H);
  float s = 0.0f;
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int e = 0; e < 8; ++e) s += x[v][e];
  // rounded on its own: contracted into x - mean (one fma), a constant row c at H = 3 * 2^k or 5 * 2^k, where
  // H * fl(1/H) != 1, leaves d = -c * 2^-25 or -c * 2^-26 instead of 0, which eps = 1e-12 scales up to ~0.03 c
  const float mean = __fmul_rn(warp_sum(s), inv_h);
  float ss = 0.0f;
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) continue;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float d = x[v][e] - mean;
      ss = fmaf(d, d, ss);
    }
  }
  const float rstd = rsqrtf(warp_sum(ss) * inv_h + eps);
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) continue;
    float g[8];
    load8(gamma + v * 256 + lane * 8, g);
    if constexpr (BIAS) {
      float b[8];
      load8(beta + v * 256 + lane * 8, b);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[v][e] = fmaf((x[v][e] - mean) * rstd, g[e], b[e]);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) x[v][e] = ((x[v][e] - mean) * rstd) * g[e];
    }
  }
}

// RoBERTa / XLM-RoBERTa position ids (create_position_ids_from_input_ids, transformers/models/xlm_roberta/
// modeling_xlm_roberta.py): with m = ids != pad, pos = cumsum(m) * m + pad along each sequence.  A pad id inside the
// attended text reads row pad and does not advance the count; left padding starts the count at the first non-pad id.
// One CTA per sequence of S ids, over chunks of POS_THREADS ids: an inclusive warp-shuffle scan of m, a scan of the 32
// warp totals by warp 0, and the running count carried to the next chunk.  pos is [B, S], the padded layout, whatever
// layout the embedding step then reads it in.
constexpr int POS_THREADS = 1024;
__global__ void __launch_bounds__(POS_THREADS)
roberta_positions_kernel(const int64_t* __restrict__ ids, int* __restrict__ pos, int S, int pad) {
  __shared__ int warp_total[POS_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t base = static_cast<size_t>(blockIdx.x) * S;
  int carry = 0;
  for (int c0 = 0; c0 < S; c0 += POS_THREADS) {
    const int s = c0 + threadIdx.x;
    const int m = (s < S && ids[base + s] != pad) ? 1 : 0;
    int x = m;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_total[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int t = warp_total[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += y;
      }
      warp_total[lane] = t;   // inclusive over warps 0..lane
    }
    __syncthreads();
    const int count = carry + (warp > 0 ? warp_total[warp - 1] : 0) + x;
    if (s < S) pos[base + s] = m ? count + pad : pad;
    carry += warp_total[POS_THREADS / 32 - 1];
    __syncthreads();   // every warp has read warp_total before the next chunk rewrites it
  }
}

// BERT embeddings: word[ids] + position[t % S] + type[type_ids] -> LayerNorm -> h16 hidden.
// (transformers/models/bert/modeling_bert.py:72-112)
// pos_ids (nullable): position row of each [B,S] token (RoBERTa's rule, roberta_positions_kernel) instead of t % S.
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
embed_layernorm_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ type_ids,
                       const float* __restrict__ word, const float* __restrict__ pos,
                       const float* __restrict__ type, const float* __restrict__ gamma,
                       const float* __restrict__ beta, h16* __restrict__ out, int rows, int S,
                       float eps, const int* __restrict__ n_dev, const int* __restrict__ tok_src,
                       const int* __restrict__ pos_ids = nullptr) {
  // n_dev / tok_src (nullable, pack.cuh): rows in use and the [B,S] position each packed row comes from
  constexpr int NV = row_passes(H);
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
  if (n_dev != nullptr) rows = __ldg(n_dev);
  if (row >= rows) return;
  const int src = tok_src != nullptr ? __ldg(tok_src + row) : row;
  const int64_t id = ids[src];
  const int64_t tt = type_ids ? type_ids[src] : 0;
  const int p = pos_ids != nullptr ? __ldg(pos_ids + src) : src % S;
  float x[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) { zero8(x[v]); continue; }
    const int c = v * 256 + lane * 8;
    float w[8], q[8], t[8];
    load8(word + static_cast<size_t>(id) * H + c, w);
    load8(pos + static_cast<size_t>(p) * H + c, q);
    load8(type + static_cast<size_t>(tt) * H + c, t);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[v][e] = (w[e] + t[e]) + q[e];  // HF order: (word + type) + pos
  }
  warp_layernorm<H>(x, gamma, beta, lane, eps);
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) store8(out + static_cast<size_t>(row) * H + v * 256 + lane * 8, x[v]);
}

// x = in (+ resid when given): the residual add of the transformer block rides on the LayerNorm's
// coalesced row reads instead of the GEMM epilogue's one-row-per-lane accesses.
__device__ __forceinline__ void load8_residual(const h16* in, const h16* resid, float (&x)[8]) {
  load8(in, x);
  if (resid != nullptr) {
    float r[8];
    load8(resid, r);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] += r[e];
  }
}

// LayerNorm over rows of a h16 matrix, optionally of (in + resid).  `out` may alias `resid`
// (each warp reads its whole row before writing it).
template <int H, typename OutT>
__global__ void __launch_bounds__(ROW_THREADS)
layernorm_kernel(const h16* __restrict__ in, const h16* resid, const float* __restrict__ gamma,
                 const float* __restrict__ beta, OutT* out, int rows, float eps,
                 const int* __restrict__ n_dev = nullptr, const int* __restrict__ out_row = nullptr) {
  // n_dev: device-resident row count; out_row: where each row goes in `out` (scatter back to [B,S])
  constexpr int NV = row_passes(H);
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
  if (n_dev != nullptr) rows = __ldg(n_dev);
  if (row >= rows) return;
  float x[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) { zero8(x[v]); continue; }
    const size_t off = static_cast<size_t>(row) * H + v * 256 + lane * 8;
    load8_residual(in + off, resid ? resid + off : nullptr, x[v]);
  }
  warp_layernorm<H>(x, gamma, beta, lane, eps);
  const size_t orow = out_row != nullptr ? static_cast<size_t>(__ldg(out_row + row)) : static_cast<size_t>(row);
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) store8(out + orow * H + v * 256 + lane * 8, x[v]);
}

// LayerNorm of selected rows only: out[b] = LN(in[b*S + idx[b]])  (last-token pooling).
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
layernorm_gather_kernel(const h16* __restrict__ in, const h16* __restrict__ resid,
                        const int* __restrict__ idx, const float* __restrict__ gamma,
                        const float* __restrict__ beta, float* __restrict__ out, int B, int S,
                        float eps, const int* __restrict__ cu = nullptr) {
  constexpr int NV = row_passes(H);
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
  if (b >= B) return;
  const size_t row = (cu != nullptr ? static_cast<size_t>(__ldg(cu + b)) : static_cast<size_t>(b) * S) + idx[b];
  float x[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) { zero8(x[v]); continue; }
    const size_t off = row * H + v * 256 + lane * 8;
    load8_residual(in + off, resid ? resid + off : nullptr, x[v]);
  }
  warp_layernorm<H>(x, gamma, beta, lane, eps);
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) store8(out + static_cast<size_t>(b) * H + v * 256 + lane * 8, x[v]);
}

// ------------------------------------------------------------------ pooling weights
// seq_len[b] = sum_s mask[b,s]  (distllm/embed/poolers/mean.py:32), one warp per sequence.
__global__ void seq_len_kernel(const int64_t* __restrict__ mask, int* __restrict__ seq_len, int B,
                               int S) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  long long acc = 0;
  for (int s = lane; s < S; s += 32) acc += mask[static_cast<size_t>(b) * S + s];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) seq_len[b] = static_cast<int>(acc);
}

// kill[s] = 1 for every column some sequence ends on.  mean.py:36 writes
// `attention_mask[:, seq_lengths - 1] = 0`, i.e. it zeroes column len_j-1 of EVERY row for every j
// in the batch (index -1 wraps to the last column, as in torch).
__global__ void kill_columns_kernel(const int* __restrict__ seq_len, int* __restrict__ kill, int B,
                                    int S) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int c = seq_len[b] - 1;
  if (c < 0) c += S;
  kill[c] = 1;
}

// w[b,s] = mask[b,s] with column 0 and the killed columns cleared; count[b] = sum_s w[b,s].
// quirk != 0: reference semantics (cross-row kill set); quirk == 0: only the row's own last token.
// When `mutate` is set the int64 mask is rewritten in place exactly as mean.py:35-36 does.
__global__ void pool_weights_kernel(int64_t* __restrict__ mask, const int* __restrict__ seq_len,
                                    const int* __restrict__ kill, float* __restrict__ w,
                                    float* __restrict__ count, int B, int S, int quirk,
                                    int mutate) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  int own = seq_len[b] - 1;
  if (own < 0) own += S;
  float acc = 0.0f;
  for (int s = lane; s < S; s += 32) {
    const size_t i = static_cast<size_t>(b) * S + s;
    const bool dead = (s == 0) || (quirk ? kill[s] != 0 : s == own);
    const int64_t mv = dead ? 0 : mask[i];
    if (mutate && dead) mask[i] = 0;
    const float wv = static_cast<float>(mv);
    w[i] = wv;
    acc += wv;
  }
  acc = warp_sum(acc);
  if (lane == 0) count[b] = acc;
}

// last_token.py:30-39: if every row's final mask entry is set use column S-1, else len_b - 1.
__global__ void last_token_index_kernel(const int64_t* __restrict__ mask,
                                        const int* __restrict__ seq_len, int* __restrict__ idx,
                                        int B, int S) {
  // single block
  __shared__ int all_set;
  if (threadIdx.x == 0) all_set = 1;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x)
    if (mask[static_cast<size_t>(b) * S + (S - 1)] != 1) atomicAnd(&all_set, 0);
  __syncthreads();
  // the reference tests `mask[:, -1].sum() == B`; with 0/1 masks that is "all ones"
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    int i = S - 1;
    if (!all_set) {
      i = seq_len[b] - 1;
      if (i < 0) i += S;
    }
    idx[b] = i;
  }
}

// ------------------------------------------------------------------ masked-sum pooling
// Shared tail: combine the ROW_WARPS per-warp partial column sums and write them to part[b,split,:].
template <int H>
__device__ __forceinline__ void block_store_partial(float (&acc)[row_passes(H)][8], float* red,
                                                    float* __restrict__ part_row, int warp,
                                                    int lane) {
  constexpr int NV = row_passes(H);
  for (int w = 0; w < ROW_WARPS; ++w) {
    if (warp == w) {
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        if (!row_lane_on<H>(v, lane)) continue;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int c = v * 256 + lane * 8 + e;
          red[c] = (w == 0) ? acc[v][e] : red[c] + acc[v][e];
        }
      }
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < H; c += ROW_THREADS) part_row[c] = red[c];
}

// Final-layer LayerNorm fused with masked-sum pooling: the [B,S,H] final hidden state is never
// written.  grid = (B, nsplit); each warp walks rows s = split*rows_per + warp, += ROW_WARPS.
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
layernorm_pool_kernel(const h16* __restrict__ in, const h16* __restrict__ resid,
                      const float* __restrict__ gamma, const float* __restrict__ beta,
                      const float* __restrict__ w,
                      float* __restrict__ part, int S, int rows_per, float eps,
                      const int* __restrict__ cu = nullptr) {
  constexpr int NV = row_passes(H);
  __shared__ float red[H];
  const int b = blockIdx.x, split = blockIdx.y, nsplit = gridDim.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[v][e] = 0.0f;
  const int s_end = min(S, (split + 1) * rows_per);
  for (int s = split * rows_per + warp; s < s_end; s += ROW_WARPS) {
    const float wv = w[static_cast<size_t>(b) * S + s];
    if (wv == 0.0f) continue;  // warp-uniform
    float x[NV][8];
    // (a row with a non-zero weight is an attended row: it exists in the packed layout too)
    const size_t row = (cu != nullptr ? static_cast<size_t>(__ldg(cu + b)) : static_cast<size_t>(b) * S) + s;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      if (!row_lane_on<H>(v, lane)) { zero8(x[v]); continue; }
      const size_t off = row * H + v * 256 + lane * 8;
      load8_residual(in + off, resid ? resid + off : nullptr, x[v]);
    }
    warp_layernorm<H>(x, gamma, beta, lane, eps);
#pragma unroll
    for (int v = 0; v < NV; ++v)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[v][e] = fmaf(x[v][e], wv, acc[v][e]);
  }
  block_store_partial<H>(acc, red, part + (static_cast<size_t>(b) * nsplit + split) * H, warp,
                          lane);
}

// Standalone masked-sum over a materialised hidden state (Pooler.pool API path).
template <int H, typename T>
__global__ void __launch_bounds__(ROW_THREADS)
pool_sum_kernel(const T* __restrict__ in, const float* __restrict__ w, float* __restrict__ part,
                int S, int rows_per) {
  constexpr int NV = row_passes(H);
  __shared__ float red[H];
  const int b = blockIdx.x, split = blockIdx.y, nsplit = gridDim.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[v][e] = 0.0f;
  const int s_end = min(S, (split + 1) * rows_per);
  for (int s = split * rows_per + warp; s < s_end; s += ROW_WARPS) {
    const float wv = w[static_cast<size_t>(b) * S + s];
    if (wv == 0.0f) continue;
    const size_t row = static_cast<size_t>(b) * S + s;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      if (!row_lane_on<H>(v, lane)) continue;
      float x[8];
      load8(in + row * H + v * 256 + lane * 8, x);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[v][e] = fmaf(x[e], wv, acc[v][e]);
    }
  }
  block_store_partial<H>(acc, red, part + (static_cast<size_t>(b) * nsplit + split) * H, warp,
                          lane);
}

// out[b,:] = (sum_split part[b,split,:]) / max(count[b], 1e-9), optionally L2-normalised
// (mean.py:45-49; F.normalize(p=2, dim=-1, eps=1e-12) from full_sequence.py:68-69).
// round_mode: 0 none, 1 round the summed numerator through bf16, 2 through fp16 -- torch sums
// `embeddings * mask` in the embedding dtype before the fp32 division.
__global__ void pool_finalize_kernel(const float* __restrict__ part, const float* __restrict__ count,
                                     float* __restrict__ out, int H, int nsplit, int l2_normalize,
                                     int round_mode) {
  extern __shared__ float row[];  // H floats + 32
  float* red = row + H;
  const int b = blockIdx.x;
  const float denom = fmaxf(count[b], 1e-9f);
  float ss = 0.0f;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float s = 0.0f;
    for (int k = 0; k < nsplit; ++k) s += part[(static_cast<size_t>(b) * nsplit + k) * H + c];
    if (round_mode == 1) s = __bfloat162float(__float2bfloat16_rn(s));
    if (round_mode == 2) s = __half2float(__float2half_rn(s));
    const float v = s / denom;
    row[c] = v;
    ss = fmaf(v, v, ss);
  }
  float norm = 1.0f;
  if (l2_normalize) {
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.0f;
    for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) tot += red[i];
    norm = fmaxf(sqrtf(tot), 1e-12f);
  }
  // a division, as F.normalize does: x * (1 / norm) differs from x / norm by one ulp in about a third of elements
  for (int c = threadIdx.x; c < H; c += blockDim.x)
    out[static_cast<size_t>(b) * H + c] = l2_normalize ? row[c] / norm : row[c];
}

// out[b,:] = in[b, idx[b], :] as fp32 (last_token.py:33-39), optional L2 normalise done separately.
template <typename T>
__global__ void gather_rows_kernel(const T* __restrict__ in, const int* __restrict__ idx,
                                   float* __restrict__ out, int B, int S, int H) {
  const int b = blockIdx.x;
  const size_t row = static_cast<size_t>(b) * S + idx[b];
  for (int c = threadIdx.x * 8; c < H; c += blockDim.x * 8) {
    float x[8];
    load8(in + row * H + c, x);
    store8(out + static_cast<size_t>(b) * H + c, x);
  }
}

// In-place row-wise x / max(||x||_2, 1e-12), one warp per row.
__global__ void l2_normalize_kernel(float* __restrict__ x, int N, int H) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= N) return;
  const int lane = threadIdx.x & 31;
  float* p = x + static_cast<size_t>(row) * H;
  float ss = 0.0f;
  for (int c = lane * 4; c < H; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(p + c);
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  const float norm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);   // divided by, as F.normalize does (pool_finalize_kernel)
  for (int c = lane * 4; c < H; c += 128) {
    float4 v = *reinterpret_cast<float4*>(p + c);
    v.x /= norm; v.y /= norm; v.z /= norm; v.w /= norm;
    *reinterpret_cast<float4*>(p + c) = v;
  }
}

// Semantic splitter distance (distllm/embed/embedders/semantic_chunk.py:41-53), fused
// normalise + dot: out[i] = 1 - <e_i, e_{i+1}> / (||e_i|| ||e_{i+1}||), one warp per adjacent pair.
// Rows are read once from HBM (the neighbour read hits L1/L2).  Pairs that straddle a document
// boundary (doc_id differs) are written as NaN and skipped by the host.
template <typename T>
__global__ void adjacent_cosine_kernel(const T* __restrict__ emb, const int* __restrict__ doc_id,
                                       float* __restrict__ out, int N, int H) {
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= N - 1) return;
  const int lane = threadIdx.x & 31;
  if (doc_id != nullptr && doc_id[i] != doc_id[i + 1]) {
    if (lane == 0) out[i] = __int_as_float(0x7fc00000);
    return;
  }
  const T* a = emb + static_cast<size_t>(i) * H;
  const T* b = a + H;
  float dot = 0.0f, na = 0.0f, nb = 0.0f;
  for (int c = lane * 8; c < H; c += 256) {
    float x[8], y[8];
    load8(a + c, x);
    load8(b + c, y);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      dot = fmaf(x[e], y[e], dot);
      na = fmaf(x[e], x[e], na);
      nb = fmaf(y[e], y[e], nb);
    }
  }
  dot = warp_sum(dot);
  na = warp_sum(na);
  nb = warp_sum(nb);
  if (lane == 0) out[i] = 1.0f - dot / (sqrtf(na) * sqrtf(nb));
}

}  // namespace b2e

// ====================================================================== ESM-2 (pre-LayerNorm) pieces
namespace b2e {

// scale[b] = (1 - 0.12) / (1 - n_mask_tokens / n_attended): ESM's "token dropout" compensation
// (transformers/models/esm/modeling_esm.py:217-224).  mask_token < 0 disables it (scale 1).
__global__ void esm_token_scale_kernel(const int64_t* __restrict__ ids,
                                       const int64_t* __restrict__ mask, float* __restrict__ scale,
                                       int B, int S, int mask_token) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  float n_mask = 0.0f, n_att = 0.0f;
  for (int s = lane; s < S; s += 32) {
    const size_t i = static_cast<size_t>(b) * S + s;
    n_att += static_cast<float>(mask[i]);
    n_mask += (mask_token >= 0 && ids[i] == mask_token) ? 1.0f : 0.0f;
  }
  n_mask = warp_sum(n_mask);
  n_att = warp_sum(n_att);
  if (lane == 0) scale[b] = mask_token >= 0 ? (1.0f - 0.15f * 0.8f) / (1.0f - n_mask / n_att) : 1.0f;
}

// x[t,:] = word[ids[t]] (zero for <mask> tokens) * scale[b] * attention_mask[t]  -> fp32 residual stream
// (modeling_esm.py:189-234 with rotary positions: no position table, no embedding LayerNorm)
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
esm_embed_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ mask,
                 const float* __restrict__ word, const float* __restrict__ scale,
                 float* __restrict__ xres, int rows, int S, int mask_token,
                 const int* __restrict__ n_dev = nullptr, const int* __restrict__ tok_src = nullptr) {
  constexpr int NV = row_passes(H);
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
  if (n_dev != nullptr) rows = __ldg(n_dev);
  if (row >= rows) return;
  const int src = tok_src != nullptr ? __ldg(tok_src + row) : row;
  const int64_t id = ids[src];
  float f = scale[src / S] * static_cast<float>(mask[src]);
  if (mask_token >= 0 && id == mask_token) f = 0.0f;
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) continue;
    const int c = v * 256 + lane * 8;
    float w[8];
    load8(word + static_cast<size_t>(id) * H + c, w);
#pragma unroll
    for (int e = 0; e < 8; ++e) w[e] *= f;
    store8(xres + static_cast<size_t>(row) * H + c, w);
  }
}

// ModernBERT embeddings (transformers/models/modernbert/modeling_modernbert.py:52-71): x = LayerNorm(tok[ids]);
// x is the fp32 residual stream AND (layer 0 has no attn_norm: :318-320) the first attention input.
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
modernbert_embed_kernel(const int64_t* __restrict__ ids, const float* __restrict__ table,
                        const float* __restrict__ gamma, const float* __restrict__ beta,
                        float* __restrict__ xres, h16* __restrict__ hidden, int rows, float eps,
                        const int* __restrict__ n_dev = nullptr, const int* __restrict__ tok_src = nullptr) {
  constexpr int NV = row_passes(H);
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
  if (n_dev != nullptr) rows = __ldg(n_dev);
  if (row >= rows) return;
  const int64_t id = ids[tok_src != nullptr ? __ldg(tok_src + row) : row];
  float x[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) load8(table + static_cast<size_t>(id) * H + v * 256 + lane * 8, x[v]);
    else zero8(x[v]);
  warp_layernorm<H>(x, gamma, beta, lane, eps);
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) continue;
    const size_t off = static_cast<size_t>(row) * H + v * 256 + lane * 8;
    store8(xres + off, x[v]);
    store8(hidden + off, x[v]);
  }
}

// Residual stream update fused with the next LayerNorm (pre-LN blocks):
//   xres += add (h16 GEMM output; nullptr on the very first call);  out = LayerNorm(xres)
// The fp32 residual stream keeps 33 layers of accumulation out of h16.
template <int H, typename OutT>
__global__ void __launch_bounds__(ROW_THREADS)
add_layernorm_kernel(float* __restrict__ xres, const h16* __restrict__ add,
                     const float* __restrict__ gamma, const float* __restrict__ beta,
                     OutT* __restrict__ out, int rows, float eps, const int* __restrict__ n_dev = nullptr) {
  constexpr int NV = row_passes(H);
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
  if (n_dev != nullptr) rows = __ldg(n_dev);
  if (row >= rows) return;
  float x[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) { zero8(x[v]); continue; }
    const size_t off = static_cast<size_t>(row) * H + v * 256 + lane * 8;
    load8(xres + off, x[v]);
    if (add != nullptr) {
      float a[8];
      load8(add + off, a);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[v][e] += a[e];
      store8(xres + off, x[v]);
    }
  }
  warp_layernorm<H>(x, gamma, beta, lane, eps);
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) store8(out + static_cast<size_t>(row) * H + v * 256 + lane * 8, x[v]);
}

// cos/sin tables for rotary embeddings, [max_pos, 32] each: angle(p, i) = p * 10000^(-2i/64)
// (modeling_esm.py:81-123, head_dim 64)
__global__ void rope_table_kernel(float* __restrict__ cos_t, float* __restrict__ sin_t, int max_pos) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= max_pos * 32) return;
  const int p = i / 32, k = i % 32;
  const float inv_freq = powf(10000.0f, -static_cast<float>(2 * k) / 64.0f);
  float s, c;
  sincosf(static_cast<float>(p) * inv_freq, &s, &c);
  cos_t[i] = c;
  sin_t[i] = s;
}

// In-place rotary embedding of the first `n_rot` heads of every row of qkv [T, ld], head_dim 2 * HALF in the
// "halves" convention (rotate_half):
//   out[i] = x[i] cos_i - x[i+HALF] sin_i ;  out[i+HALF] = x[i+HALF] cos_i + x[i] sin_i
// with the position of a row inside its sequence = tok_src[t] % S (packed layout) or t % S.  The rotated heads
// start at column 0: Q heads directly followed by the K heads in every layout this library uses.
// A thread owns 8 consecutive frequencies (one 16-byte vector from each half), HALF / 8 threads share a head,
// so a warp moves 1 KiB (HALF = 32) or 2 x 512 B (HALF = 64) of contiguous bytes per access: the kernel is a plain
// HBM stream (one 2-byte element per lane would leave most of each 32-byte sector transfer unused).
template <int HALF>
__global__ void __launch_bounds__(256)
rope_halves_kernel(h16* __restrict__ qkv, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                   int T, int S, int n_rot, int ld, const int* __restrict__ n_dev = nullptr,
                   const int* __restrict__ tok_src = nullptr) {
  constexpr int TPH = HALF / 8;   // threads per head
  if (n_dev != nullptr) T = __ldg(n_dev);
  const long long gtid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long unit = gtid / TPH;
  const int g = static_cast<int>(gtid % TPH);
  if (unit >= static_cast<long long>(T) * n_rot) return;
  const int t = static_cast<int>(unit / n_rot);
  const int hd = static_cast<int>(unit % n_rot);
  h16* p = qkv + static_cast<size_t>(t) * ld + hd * (2 * HALF) + g * 8;
  const int pos = (tok_src != nullptr ? __ldg(tok_src + t) : t) % S;
  float c[8], sn[8], x1[8], x2[8];
  load8(cos_t + static_cast<size_t>(pos) * HALF + g * 8, c);
  load8(sin_t + static_cast<size_t>(pos) * HALF + g * 8, sn);
  load8(p, x1);
  load8(p + HALF, x2);
  float o1[8], o2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    o1[i] = x1[i] * c[i] - x2[i] * sn[i];
    o2[i] = x2[i] * c[i] + x1[i] * sn[i];
  }
  store8(p, o1);
  store8(p + HALF, o2);
}

}  // namespace b2e
