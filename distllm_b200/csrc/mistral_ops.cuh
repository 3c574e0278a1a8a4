// Row kernels of the Mistral-family forward pass (pre-norm decoder blocks used as an encoder):
// embedding gather, RMSNorm fused with the fp32 residual update, rotary tables and the in-place
// rotation of the q and k heads.  Semantics: transformers/models/mistral/modeling_mistral.py
// :181-200 (RMSNorm), :51-80 and :262-326 (rotary, halves convention), :202-242 (pre-norm blocks),
// :328-400 (embed_tokens, final norm), reached from distllm/embed/encoders/auto.py:135.
#pragma once

#include "rowops.cuh"

namespace b2e {

// xres[row] = embed_tokens[ids[row]]   (fp32 residual stream; padding rows are embedded like any other
// token, exactly as HF does -- they are only ever masked as KEYS)
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
mistral_embed_kernel(const int64_t* __restrict__ ids, const float* __restrict__ table,
                     float* __restrict__ xres, int rows, const int* __restrict__ n_dev = nullptr,
                     const int* __restrict__ tok_src = nullptr) {
  constexpr int NV = row_passes(H);
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
  if (n_dev != nullptr) rows = __ldg(n_dev);
  if (row >= rows) return;
  const int64_t id = ids[tok_src != nullptr ? __ldg(tok_src + row) : row];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) continue;
    const int c = v * 256 + lane * 8;
    float w[8];
    load8(table + static_cast<size_t>(id) * H + c, w);
    store8(xres + static_cast<size_t>(row) * H + c, w);
  }
}

template <int H>
__device__ __forceinline__ void warp_rmsnorm(float (&x)[row_passes(H)][8], const float* __restrict__ gamma,
                                             int lane, float eps) {
  constexpr int NV = row_passes(H);
  float ss = 0.0f;
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int e = 0; e < 8; ++e) ss = fmaf(x[v][e], x[v][e], ss);
  ss = warp_sum(ss);
  const float r = rsqrtf(ss * (1.0f / H) + eps);
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    if (!row_lane_on<H>(v, lane)) continue;
    float g[8];
    load8(gamma + v * 256 + lane * 8, g);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[v][e] = g[e] * (x[v][e] * r);
  }
}

// Residual stream update fused with the next RMSNorm:
//   xres += add (h16 GEMM output; nullptr on the very first call);  out = RMSNorm(xres) * gamma
template <int H, typename OutT>
__global__ void __launch_bounds__(ROW_THREADS)
add_rmsnorm_kernel(float* __restrict__ xres, const h16* __restrict__ add,
                   const float* __restrict__ gamma, OutT* __restrict__ out, int rows, float eps,
                   const int* __restrict__ n_dev = nullptr) {
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
  warp_rmsnorm<H>(x, gamma, lane, eps);
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) store8(out + static_cast<size_t>(row) * H + v * 256 + lane * 8, x[v]);
}

// Final norm for the last-token pooler: only the B selected rows are normalised.
//   out[b] = RMSNorm(xres[b*S + idx[b]] + add[b*S + idx[b]]) * gamma        (fp32 [B,H])
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
rmsnorm_gather_kernel(const float* __restrict__ xres, const h16* __restrict__ add,
                      const float* __restrict__ gamma, const int* __restrict__ idx,
                      float* __restrict__ out, int B, int S, float eps, const int* __restrict__ cu = nullptr) {
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
    float a[8];
    load8(xres + off, x[v]);
    load8(add + off, a);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[v][e] += a[e];
  }
  warp_rmsnorm<H>(x, gamma, lane, eps);
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) store8(out + static_cast<size_t>(b) * H + v * 256 + lane * 8, x[v]);
}

// ESM-2 last-token pooling: out[b] = LayerNorm(xres[row] + add[row]) for the B selected rows (fp32 [B,H]).
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
addnorm_gather_kernel(const float* __restrict__ xres, const h16* __restrict__ add,
                      const float* __restrict__ gamma, const float* __restrict__ beta,
                      const int* __restrict__ idx, float* __restrict__ out, int B, int S, float eps,
                      const int* __restrict__ cu = nullptr) {
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
    float a[8];
    load8(xres + off, x[v]);
    load8(add + off, a);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[v][e] += a[e];
  }
  warp_layernorm<H>(x, gamma, beta, lane, eps);
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) store8(out + static_cast<size_t>(b) * H + v * 256 + lane * 8, x[v]);
}

// Final norm of the pre-norm families fused with the masked-sum pooling (the [B,S,H] final hidden state is
// never written): x = xres + add, then LayerNorm (RMS == false: ESM-2's emb_layer_norm_after) or RMSNorm
// (RMS == true: Mistral's final norm), weighted by the pooling weights and summed per block.
// grid = (B, nsplit); each warp walks rows s = split*rows_per + warp, += ROW_WARPS (as layernorm_pool_kernel).
template <int H, bool RMS>
__global__ void __launch_bounds__(ROW_THREADS)
addnorm_pool_kernel(const float* __restrict__ xres, const h16* __restrict__ add,
                    const float* __restrict__ gamma, const float* __restrict__ beta,
                    const float* __restrict__ w, float* __restrict__ part, int S, int rows_per, float eps,
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
    const size_t row = (cu != nullptr ? static_cast<size_t>(__ldg(cu + b)) : static_cast<size_t>(b) * S) + s;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      if (!row_lane_on<H>(v, lane)) { zero8(x[v]); continue; }
      const size_t off = row * H + v * 256 + lane * 8;
      float a[8];
      load8(xres + off, x[v]);
      load8(add + off, a);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[v][e] += a[e];
    }
    if (RMS) warp_rmsnorm<H>(x, gamma, lane, eps);
    else warp_layernorm<H>(x, gamma, beta, lane, eps);
#pragma unroll
    for (int v = 0; v < NV; ++v)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[v][e] = fmaf(x[v][e], wv, acc[v][e]);
  }
  block_store_partial<H>(acc, red, part + (static_cast<size_t>(b) * nsplit + split) * H, warp, lane);
}

// cos/sin tables [max_pos, half]: angle(p, i) = p * theta^(-2i / (2*half))
__global__ void rope_table_theta_kernel(float* __restrict__ cos_t, float* __restrict__ sin_t,
                                        int max_pos, int half, float theta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= max_pos * half) return;
  const int p = i / half, k = i % half;
  const float inv_freq = 1.0f / powf(theta, static_cast<float>(2 * k) / static_cast<float>(2 * half));
  float s, c;
  sincosf(static_cast<float>(p) * inv_freq, &s, &c);
  cos_t[i] = c;
  sin_t[i] = s;
}

// Qwen3 (transformers/models/qwen3/modeling_qwen3.py:248-249, :263-264): every q head and every k head of qkv
// [T, ld] goes through its own RMSNorm over head_dim 128 BEFORE the rotary embedding, in place, one pass:
//   y[i] = gamma[i] * (x[i] * rsqrt(mean(x^2) + eps)),   gamma = q_gamma for heads [0, heads), k_gamma for
//   heads [heads, heads + kv_heads);  then the halves rotation of y at position tok_src[t] % S (or t % S).
// Layout of rope_halves_kernel<64>: 8 threads per head, each owning frequencies [8g, 8g + 8) of both halves as
// two 16-byte vectors; the head's sum of squares is reduced over its 8 lanes (8-aligned in the warp, since the
// block size is a multiple of 8, and all 8 leave together past the last row).  One rounding to 16 bits, at the
// store; the V heads behind the k heads are not touched.
__global__ void __launch_bounds__(256)
qk_rmsnorm_rope_kernel(h16* __restrict__ qkv, const float* __restrict__ q_gamma, const float* __restrict__ k_gamma,
                       const float* __restrict__ cos_t, const float* __restrict__ sin_t, int T, int S, int heads,
                       int kv_heads, int ld, float eps, const int* __restrict__ n_dev = nullptr,
                       const int* __restrict__ tok_src = nullptr) {
  constexpr int HALF = 64, TPH = HALF / 8;
  if (n_dev != nullptr) T = __ldg(n_dev);
  const int n_rot = heads + kv_heads;
  const long long gtid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long unit = gtid / TPH;
  const int g = static_cast<int>(gtid % TPH);
  if (unit >= static_cast<long long>(T) * n_rot) return;
  const int t = static_cast<int>(unit / n_rot);
  const int hd = static_cast<int>(unit % n_rot);
  h16* p = qkv + static_cast<size_t>(t) * ld + hd * (2 * HALF) + g * 8;
  float x1[8], x2[8];
  load8(p, x1);
  load8(p + HALF, x2);
  float ss = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss = fmaf(x2[i], x2[i], fmaf(x1[i], x1[i], ss));
  const unsigned group = 0xffu << (threadIdx.x & 24);
#pragma unroll
  for (int o = TPH / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(group, ss, o);
  const float r = rsqrtf(ss * (1.0f / (2 * HALF)) + eps);
  const float* gamma = (hd < heads ? q_gamma : k_gamma) + g * 8;
  float g1[8], g2[8];
  load8(gamma, g1);
  load8(gamma + HALF, g2);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    x1[i] = g1[i] * (x1[i] * r);
    x2[i] = g2[i] * (x2[i] * r);
  }
  const int pos = (tok_src != nullptr ? __ldg(tok_src + t) : t) % S;
  float c[8], sn[8];
  load8(cos_t + static_cast<size_t>(pos) * HALF + g * 8, c);
  load8(sin_t + static_cast<size_t>(pos) * HALF + g * 8, sn);
  float o1[8], o2[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    o1[i] = x1[i] * c[i] - x2[i] * sn[i];
    o2[i] = x2[i] * c[i] + x1[i] * sn[i];
  }
  store8(p, o1);
  store8(p + HALF, o2);
}

// ESM C (esm/layers/attention.py, esm/layers/rotary.py of the esm package): the whole H-wide q row and the whole k row
// of qkv [T, 3H] each go through a LayerNorm without bias (q_ln / k_ln, statistics over H in fp32), and then every
// 64-wide head of the result is rotated in the halves convention at position tok_src[t] % S (or t % S), in place:
//   y = gamma * ((x - mean) * rstd);  out[i] = y[i] cos_i - y[i+32] sin_i,  out[i+32] = y[i+32] cos_i + y[i] sin_i
// One warp per (token, q or k) row in the row layout of rowops.cuh (warp_layernorm): lane owns 8 consecutive columns
// of each 256-column pass, so a head is 8 lanes of one pass and the partner of a lane's columns is lane ^ 4 (the same
// 8 frequencies (lane & 3) * 8 .. +8 of the other half).  Heads never straddle a pass, and the off lanes of a partial
// pass (row_lane_on) hold whole heads, so an on lane never partners an off lane.  One rounding to 16 bits, at the
// store; V and rows from T on (T = *n_dev when given) are not touched.
template <int H>
__global__ void __launch_bounds__(ROW_THREADS)
qk_layernorm_rope_kernel(h16* __restrict__ qkv, const float* __restrict__ q_gamma, const float* __restrict__ k_gamma,
                         const float* __restrict__ cos_t, const float* __restrict__ sin_t, int T, int S, float eps,
                         const int* __restrict__ n_dev = nullptr, const int* __restrict__ tok_src = nullptr) {
  constexpr int NV = row_passes(H), HALF = 32;
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);   // 2 t + (0: q, 1: k)
  if (n_dev != nullptr) T = __ldg(n_dev);
  const int t = r >> 1;
  if (t >= T) return;   // warp-uniform
  h16* row = qkv + static_cast<size_t>(t) * (3 * H) + (r & 1) * H;
  float x[NV][8];
#pragma unroll
  for (int v = 0; v < NV; ++v)
    if (row_lane_on<H>(v, lane)) load8(row + v * 256 + lane * 8, x[v]);
    else zero8(x[v]);
  warp_layernorm<H, false>(x, (r & 1) ? k_gamma : q_gamma, nullptr, lane, eps);
  const int pos = (tok_src != nullptr ? __ldg(tok_src + t) : t) % S;
  float c[8], sn[8];
  load8(cos_t + static_cast<size_t>(pos) * HALF + (lane & 3) * 8, c);
  load8(sin_t + static_cast<size_t>(pos) * HALF + (lane & 3) * 8, sn);
  const bool upper = (lane & 4) != 0;   // columns i + 32 of the head
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float p = __shfl_xor_sync(0xffffffffu, x[v][e], 4);
      o[e] = upper ? x[v][e] * c[e] + p * sn[e] : x[v][e] * c[e] - p * sn[e];
    }
    if (row_lane_on<H>(v, lane)) store8(row + v * 256 + lane * 8, o);
  }
}

}  // namespace b2e
