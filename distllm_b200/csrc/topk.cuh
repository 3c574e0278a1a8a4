// Exact inner-product top-k over a device-resident embedding matrix (SURVEY 8(f) rank 2: the retrieval
// query path that consumes the all-gathered [N,H] matrix).  Replaces faiss.IndexFlatIP.search as called
// from distllm/rag/search.py:280-336 (semantic_search_faiss, exact float32 branch): scores are fp32 dot
// products, the k best per query come back sorted by descending score.
//
// The scan is HBM-bound for small query batches: every corpus row is read once for up to TOPK_QT
// queries.  A warp holds TOPK_ROWS rows in registers, streams the query tile from shared memory (one
// load feeds TOPK_ROWS rows) and keeps one partial dot product per (query, row); candidates that beat the
// CTA's current k-th row -- higher score, or an equal score and a lower row id -- enter a small
// shared-memory set under a per-query lock (rare after the first few thousand rows).  A second kernel
// merges the per-CTA sets of one query and sorts the survivors.  Equal scores are resolved by row id at
// every step, so the result does not depend on the order in which warps and CTAs reach the rows.
//
// The L2 instantiation (float32 corpus only: faiss.IndexFlatL2 of distllm/rag/search.py:402-666, FaissIndexV1
// with metric='l2') accumulates (q_i - x_i)^2 instead of q_i * x_i and offers -D to the same sets, so "higher
// score, then lower row id" orders rows by ascending squared distance, ties by ascending row id; the merge writes
// D = -score back out (an empty slot's -inf becomes +inf).
#pragma once

#include "common.cuh"

namespace b2e {

constexpr int TOPK_QT = 16;        // queries per pass over the corpus (wide variant)
// Two shapes of the scan: <QT=16, ROWS=4> shares one pass among up to 16 queries; <QT=4, ROWS=8> serves
// the usual one-to-four-query search with twice the rows (bytes) in flight per warp and a 32-value
// reduction instead of a 64-value one.  QT * ROWS is 32 or 64: the transposing butterfly needs it.
constexpr int TOPK_THREADS = 256;
constexpr int TOPK_MAX_K = 256;

// ---- a k-slot candidate set in shared memory: replace-the-worst insertion by a whole warp
// The set keeps the k best rows in a strict total order: higher score first, then lower row id (the
// contract's "ties by ascending index").  Which rows it ends up with is therefore independent of the
// order the rows are offered in: of the lanes' value layout, of warp scheduling, of the merge's walk.
struct TopkSet {
  float* score;    // [k]
  int64_t* index;  // [k]; -1 = empty slot (score -inf), worse than any row
  float* kth;      // score of the set's worst slot (threshold for new candidates)
  int* kth_pos;    // position of the worst slot
  int* lock;
};

// row id of a slot as an ordering key: an empty slot's -1 sorts above every row id
__device__ __forceinline__ int64_t topk_id_key(const TopkSet& s, int slot) {
  const int64_t idx = reinterpret_cast<volatile int64_t*>(s.index)[slot];
  return idx < 0 ? INT64_MAX : idx;
}

__device__ __forceinline__ void topk_insert_inline(const TopkSet& s, int k, float score, int64_t idx, int lane) {
  // all 32 lanes call this together with the same (score, idx); every decision below is taken on lane
  // 0's reading of the threshold so that the warp never diverges around the __syncwarp()s.  The worst
  // slot only ever gets better, so a score strictly below any reading of the threshold can be rejected
  // without the lock; an equal score is decided under the lock by the row ids.
  float th = *reinterpret_cast<volatile float*>(s.kth);
  th = __shfl_sync(0xffffffffu, th, 0);
  if (!(score >= th)) return;
  if (lane == 0) {
    while (atomicCAS(s.lock, 0, 1) != 0) {
    }
  }
  __syncwarp();
  __threadfence_block();
  int take = 0, pos = 0;
  if (lane == 0) {
    th = *reinterpret_cast<volatile float*>(s.kth);
    pos = *reinterpret_cast<volatile int*>(s.kth_pos);
    take = score > th || (score == th && idx < topk_id_key(s, pos));
  }
  if (__shfl_sync(0xffffffffu, take, 0)) {
    if (lane == 0) {
      s.score[pos] = score;
      s.index[pos] = idx;
    }
    __syncwarp();
    __threadfence_block();
    // new worst slot (lowest score, then highest id): every lane scans a strided part of the set for the
    // lowest score and notes whether it holds that score twice
    float m = INFINITY;
    int mp = 0;
    bool twice = false;
    for (int i = lane; i < k; i += 32) {
      const float v = reinterpret_cast<volatile float*>(s.score)[i];
      if (v < m) { m = v; mp = i; twice = false; } else if (v == m) { twice = true; }
    }
    const float lane_min = m;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o);
      const int op = __shfl_xor_sync(0xffffffffu, mp, o);
      if (om < m || (om == m && op < mp)) { m = om; mp = op; }
    }
    // several slots at the lowest score (duplicate rows, or the empty slots while the set fills): the
    // worst of them is the highest row id, found in a second pass that only such ties pay for
    const bool at_min = lane_min == m;
    if (__popc(__ballot_sync(0xffffffffu, at_min)) > 1 || __any_sync(0xffffffffu, at_min && twice)) {
      uint64_t key = 0;   // id + 1 of the lane's worst slot at score m (empty slot: all ones); 0 = none
      int wp = k;
      for (int i = lane; i < k; i += 32) {
        if (reinterpret_cast<volatile float*>(s.score)[i] == m) {
          const uint64_t ki = static_cast<uint64_t>(topk_id_key(s, i)) + 1u;   // INT64_MAX + 1: empty
          if (ki > key) { key = ki; wp = i; }
        }
      }
      const unsigned hi = __reduce_max_sync(0xffffffffu, static_cast<unsigned>(key >> 32));
      const unsigned lo = __reduce_max_sync(0xffffffffu, static_cast<unsigned>(key >> 32) == hi
                                                             ? static_cast<unsigned>(key) : 0u);
      const bool worst = static_cast<unsigned>(key >> 32) == hi && static_cast<unsigned>(key) == lo;
      mp = static_cast<int>(__reduce_min_sync(0xffffffffu, worst ? static_cast<unsigned>(wp) : 0xffffffffu));
    }
    if (lane == 0) {
      *reinterpret_cast<volatile int*>(s.kth_pos) = mp;
      *reinterpret_cast<volatile float*>(s.kth) = m;
    }
  }
  __syncwarp();
  __threadfence_block();
  if (lane == 0) atomicExch(s.lock, 0);
  __syncwarp();
}

// the scan's copy: one out-of-line body shared by all its call sites (see the candidate loop below)
__device__ __noinline__ void topk_insert(const TopkSet& s, int k, float score, int64_t idx, int lane) {
  topk_insert_inline(s, k, score, idx, lane);
}

// One 16-byte vector of a corpus row per lane: 4 fp32 or 8 bf16 elements.
template <typename T> struct TopkVec;
template <> struct TopkVec<float> {
  static constexpr int E = 4;
  float4 raw;
  __device__ __forceinline__ void load(const float* p) { raw = *reinterpret_cast<const float4*>(p); }
  __device__ __forceinline__ void zero() { raw = make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ __forceinline__ float dot(const float* q, float acc) const {
    const float4 w = *reinterpret_cast<const float4*>(q);
    return fmaf(raw.x, w.x, fmaf(raw.y, w.y, fmaf(raw.z, w.z, fmaf(raw.w, w.w, acc))));
  }
  // acc + sum (q_i - x_i)^2, in the order dot() sums the products
  __device__ __forceinline__ float sqdist(const float* q, float acc) const {
    const float4 w = *reinterpret_cast<const float4*>(q);
    const float dx = w.x - raw.x, dy = w.y - raw.y, dz = w.z - raw.z, dw = w.w - raw.w;
    return fmaf(dx, dx, fmaf(dy, dy, fmaf(dz, dz, fmaf(dw, dw, acc))));
  }
};
template <> struct TopkVec<bf16> {
  static constexpr int E = 8;
  uint4 raw;
  __device__ __forceinline__ void load(const bf16* p) { raw = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void zero() { raw = make_uint4(0u, 0u, 0u, 0u); }
  __device__ __forceinline__ float dot(const float* q, float acc) const {
    const float4 w0 = *reinterpret_cast<const float4*>(q), w1 = *reinterpret_cast<const float4*>(q + 4);
    const float2 a = unpack_bf16x2(raw.x), b = unpack_bf16x2(raw.y), c = unpack_bf16x2(raw.z),
                 d = unpack_bf16x2(raw.w);
    acc = fmaf(a.x, w0.x, fmaf(a.y, w0.y, fmaf(b.x, w0.z, fmaf(b.y, w0.w, acc))));
    return fmaf(c.x, w1.x, fmaf(c.y, w1.y, fmaf(d.x, w1.z, fmaf(d.y, w1.w, acc))));
  }
};

// shared memory: queries [nq][H] f32 | sets: score [nq][k] f32, index [nq][k] i64, kth/kth_pos/lock [nq]
// L2: the sets hold -D (squared Euclidean distance), see the file header.
template <typename T, int QT, int ROWS, int VMAX, bool L2 = false>
__global__ void __launch_bounds__(TOPK_THREADS)
topk_scan_kernel(const float* __restrict__ queries,   // [nq, H] (this pass's query tile)
                 const T* __restrict__ corpus,        // [N, H]
                 int nq, long long N, int H, int k,
                 float* __restrict__ part_score,      // [gridDim.x, nq, k]
                 int64_t* __restrict__ part_index,
                 const int* __restrict__ run_flag = nullptr) {   // non-null: do nothing unless *run_flag != 0
  if (run_flag != nullptr && *run_flag == 0) return;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float* qs = reinterpret_cast<float*>(smem_raw);
  float* set_score = qs + static_cast<size_t>(nq) * H;
  int64_t* set_index = reinterpret_cast<int64_t*>(set_score + nq * k + ((nq * k) & 1));
  float* kth = reinterpret_cast<float*>(set_index + nq * k);
  int* kth_pos = reinterpret_cast<int*>(kth + nq);
  int* lock = kth_pos + nq;

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < nq * H; i += TOPK_THREADS) qs[i] = queries[i];
  for (int i = threadIdx.x; i < nq * k; i += TOPK_THREADS) {
    set_score[i] = -INFINITY;
    set_index[i] = -1;
  }
  for (int i = threadIdx.x; i < nq; i += TOPK_THREADS) {
    kth[i] = -INFINITY;
    kth_pos[i] = 0;
    lock[i] = 0;
  }
  __syncthreads();

  constexpr int E = TopkVec<T>::E;
  constexpr int TOPK_VMAX = VMAX;     // 16-byte vectors per lane and row held in registers at a time
  constexpr int TOPK_ROWS = ROWS;
  constexpr int VALS = QT * ROWS;
  constexpr int PER = VALS / 32;      // totals a lane ends up with
  static_assert(VALS == 32 || VALS == 64, "the butterfly reduces 32 or 64 values per lane");
  const int nv = H / (32 * E);                 // 16-byte vectors per lane and row
  const long long warps_total = static_cast<long long>(gridDim.x) * (TOPK_THREADS / 32);
  const long long gwarp = static_cast<long long>(blockIdx.x) * (TOPK_THREADS / 32) + warp;
  for (long long row0 = gwarp * TOPK_ROWS; row0 < N; row0 += warps_total * TOPK_ROWS) {
    float acc[QT][TOPK_ROWS];
#pragma unroll
    for (int q = 0; q < QT; ++q)
#pragma unroll
      for (int r = 0; r < TOPK_ROWS; ++r) acc[q][r] = 0.0f;
    for (int v0 = 0; v0 < nv; v0 += TOPK_VMAX) {
      TopkVec<T> x[TOPK_ROWS][TOPK_VMAX];
#pragma unroll
      for (int r = 0; r < TOPK_ROWS; ++r) {
        const long long row = row0 + r;
#pragma unroll
        for (int v = 0; v < TOPK_VMAX; ++v) {
          x[r][v].zero();
          if (row < N && v0 + v < nv)
            x[r][v].load(corpus + static_cast<size_t>(row) * H + ((v0 + v) * 32 + lane) * E);
        }
      }
#pragma unroll
      for (int q = 0; q < QT; ++q) {
        if (q < nq) {
#pragma unroll
          for (int v = 0; v < TOPK_VMAX; ++v) {
            if (v0 + v < nv) {
              const float* w = qs + static_cast<size_t>(q) * H + ((v0 + v) * 32 + lane) * E;
#pragma unroll
              for (int r = 0; r < TOPK_ROWS; ++r) {
                if constexpr (L2) acc[q][r] = x[r][v].sqdist(w, acc[q][r]);
                else acc[q][r] = x[r][v].dot(w, acc[q][r]);
              }
            }
          }
        }
      }
    }
    // VALS partial sums per lane -> totals by a transposing butterfly (VALS - PER shuffles instead of
    // 5 * VALS): lane l ends up with the totals of value indices l * PER + j, index = query * ROWS + row
    float v[VALS];
#pragma unroll
    for (int q = 0; q < QT; ++q)
#pragma unroll
      for (int r = 0; r < TOPK_ROWS; ++r) v[q * TOPK_ROWS + r] = acc[q][r];
#pragma unroll
    for (int half = VALS / 2, bit = 16; half >= PER; half >>= 1, bit >>= 1) {
      const bool upper = (lane & bit) != 0;
#pragma unroll
      for (int i = 0; i < half; ++i) {
        const float keep = upper ? v[i + half] : v[i];
        const float send = upper ? v[i] : v[i + half];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, bit);
      }
    }
    if constexpr (L2) {
#pragma unroll
      for (int j = 0; j < PER; ++j) v[j] = -v[j];
    }
    // the few candidates that reach their query's current k-th score are inserted one by one (a score
    // equal to it may still win on the row id: topk_insert decides); the loop body exists once (64 inlined
    // copies of it used to push the kernel out of the instruction cache)
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int my_i = lane * PER + j;
      const int my_q = my_i / TOPK_ROWS, my_r = my_i % TOPK_ROWS;
      const float th = (my_q < nq) ? *reinterpret_cast<volatile float*>(kth + my_q) : INFINITY;
      const bool cand = (my_q < nq) && (row0 + my_r < N) && (v[j] >= th);
      unsigned todo = __ballot_sync(0xffffffffu, cand);
      while (todo != 0) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const float sc = __shfl_sync(0xffffffffu, v[j], src);
        const int i = src * PER + j;
        const int q = i / TOPK_ROWS, r = i % TOPK_ROWS;
        const TopkSet set{set_score + q * k, set_index + q * k, kth + q, kth_pos + q, lock + q};
        topk_insert(set, k, sc, row0 + r, lane);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nq * k; i += TOPK_THREADS) {
    part_score[static_cast<size_t>(blockIdx.x) * nq * k + i] = set_score[i];
    part_index[static_cast<size_t>(blockIdx.x) * nq * k + i] = set_index[i];
  }
}

// One CTA per query: merge `parts` candidate sets of k entries, sort the k survivors by descending
// score (ties: ascending index), write them out (L2: negated, i.e. D ascending).  Empty slots (index -1) sort last.
template <bool L2 = false>
__global__ void __launch_bounds__(TOPK_THREADS)
topk_merge_kernel(const float* __restrict__ part_score, const int64_t* __restrict__ part_index, int parts,
                  int nq, int k, float* __restrict__ out_score, int64_t* __restrict__ out_index,
                  int out_stride, const int* __restrict__ run_flag = nullptr) {
  if (run_flag != nullptr && *run_flag == 0) return;
  __shared__ float s_score[TOPK_MAX_K];
  __shared__ int64_t s_index[TOPK_MAX_K];
  __shared__ float s_kth;
  __shared__ int s_kth_pos, s_lock;
  const int q = blockIdx.x;
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < TOPK_MAX_K; i += TOPK_THREADS) {
    s_score[i] = -INFINITY;
    s_index[i] = -1;
  }
  if (threadIdx.x == 0) {
    s_kth = -INFINITY;
    s_kth_pos = 0;
    s_lock = 0;
  }
  __syncthreads();
  const TopkSet set{s_score, s_index, &s_kth, &s_kth_pos, &s_lock};
  const int total = parts * k;
  // warp-uniform candidate per iteration: each warp walks its own slice (in any order: topk_insert keeps
  // the k best by (score, row id))
  const int warp = threadIdx.x >> 5;
  for (int c = warp; c < total; c += TOPK_THREADS / 32) {
    const int part = c / k, slot = c % k;
    const size_t off = (static_cast<size_t>(part) * nq + q) * k + slot;
    const int64_t idx = part_index[off];
    if (idx >= 0) topk_insert_inline(set, k, part_score[off], idx, lane);
  }
  __syncthreads();
  // bitonic sort of TOPK_MAX_K slots (slots >= k hold -inf / -1)
  for (int size = 2; size <= TOPK_MAX_K; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < TOPK_MAX_K; i += TOPK_THREADS) {
        const int j = i ^ stride;
        if (j > i) {
          const bool desc = (i & size) == 0;
          const float a = s_score[i], b = s_score[j];
          const int64_t ia = s_index[i], ib = s_index[j];
          // "a before b": higher score first, empty slots last, then lower index
          const bool a_first = (a > b) || (a == b && ((ia >= 0 && ib < 0) || ((ia >= 0) == (ib >= 0) && ia < ib)));
          if (desc ? !a_first : a_first) {
            s_score[i] = b; s_score[j] = a;
            s_index[i] = ib; s_index[j] = ia;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < k; i += TOPK_THREADS) {
    out_score[static_cast<size_t>(q) * out_stride + i] = L2 ? -s_score[i] : s_score[i];
    out_index[static_cast<size_t>(q) * out_stride + i] = s_index[i];
  }
}

}  // namespace b2e
