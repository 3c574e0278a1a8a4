// libb2e.so -- C ABI (include/b2e.h) over the sm_90a kernels.  Host runtime only: handle,
// lazily grown workspace, TMA descriptors and launches.  No CPU fallback: without an sm_90 device
// every compute entry point fails with B2E_ERR_NO_DEVICE.
#include "../../include/b2e.h"
#include "../../include/b2e_debug.h"

#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "attention.cuh"
#include "binsearch.cuh"
#include "common.cuh"
#include "gemm.cuh"
#include "mistral_ops.cuh"
#include "pack.cuh"
#include "rowops.cuh"
#include "topk.cuh"
#include "topk_tc.cuh"

using namespace b2e;

// the 16-bit storage type of this build (common.cuh): tensor-map element type and its ABI dtype code
#ifdef B2E_STORAGE_BF16
#define B2E_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
constexpr int kStorageDtype = B2E_DTYPE_BF16;
#else
#define B2E_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_FLOAT16
constexpr int kStorageDtype = B2E_DTYPE_F16;
#endif

namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define CUDA_TRY(expr)                                                                    \
  do {                                                                                    \
    cudaError_t e_ = (expr);                                                              \
    if (e_ != cudaSuccess)                                                                \
      return fail(B2E_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_),   \
                  __FILE__, __LINE__);                                                    \
  } while (0)

// ---- driver entry point for tensor-map encoding (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// 2-D half row-major [rows, cols] tensor, box = 64 columns (128 B, swizzle-128B) x box_rows, or with box_cols = 32
// 32 columns (64 B, swizzle-64B: the head_dim-32 attention boxes).  ld: the row stride in elements (0: cols).
int make_tmap_h16(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols,
                   uint32_t box_rows, uint32_t box_cols = 64, uint64_t ld = 0) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(B2E_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {(ld ? ld : cols) * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, B2E_TMAP_DTYPE, 2, const_cast<void*>(base), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B2E_ERR_CUDA, "cuTensorMapEncodeTiled(rows=%llu, cols=%llu, box_rows=%u) -> %d",
                (unsigned long long)rows, (unsigned long long)cols, box_rows, (int)r);
  return B2E_OK;
}

// NF4 codes, uint8 row-major [rows, cols] (cols = K/2), box = 32 bytes (one k-block) x GEMM_BN rows, no swizzle
int make_tmap_codes(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(B2E_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols};
  cuuint32_t box[2] = {GEMM_BK / 2, GEMM_BN};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B2E_ERR_CUDA, "cuTensorMapEncodeTiled codes(rows=%llu, cols=%llu) -> %d", (unsigned long long)rows,
                (unsigned long long)cols, (int)r);
  return B2E_OK;
}

// 2-D float32 row-major tensor, box = 32 columns (128 bytes) x box_rows, 128-byte swizzle; rows beyond the
// tensor read as zeros
int make_tmap_f32(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(B2E_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 4};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B2E_ERR_CUDA, "cuTensorMapEncodeTiled f32(rows=%llu, cols=%llu, box_rows=%u) -> %d",
                (unsigned long long)rows, (unsigned long long)cols, box_rows, (int)r);
  return B2E_OK;
}

struct DeviceInfo {
  int sms = 0;
  int cc_major = 0;
  bool ok = false;
};

int device_info(int device, DeviceInfo* info) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(B2E_ERR_NO_DEVICE, "no CUDA device visible; libb2e has no CPU fallback");
  }
  if (device < 0 || device >= n) return fail(B2E_ERR_INVALID, "device %d out of range", device);
  cudaDeviceProp p;
  CUDA_TRY(cudaGetDeviceProperties(&p, device));
  if (p.major != 9 || p.minor != 0)
    return fail(B2E_ERR_NO_DEVICE, "device %d is sm_%d%d; libb2e is built for sm_90a only", device,
                p.major, p.minor);
  info->sms = p.multiProcessorCount;
  info->cc_major = p.major;
  info->ok = true;
  return B2E_OK;
}

int current_device_info(DeviceInfo* info) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    cudaGetLastError();
    return fail(B2E_ERR_NO_DEVICE, "no CUDA device visible; libb2e has no CPU fallback");
  }
  static DeviceInfo cache[64];
  if (dev < 64 && cache[dev].ok) {
    *info = cache[dev];
    return B2E_OK;
  }
  int rc = device_info(dev, info);
  if (rc == B2E_OK && dev < 64) cache[dev] = *info;
  return rc;
}

// Opt a kernel in to `bytes` of dynamic shared memory, once per (kernel, device): the attribute belongs
// to the device's context, and a process may drive more than one device over its lifetime.
template <typename Kern>
int ensure_smem_attr(Kern kern, int bytes) {
  // keyed by the kernel's ADDRESS (kernels with equal signatures share one C++ type) and the device
  static std::vector<std::pair<const void*, int>> done;
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  const void* key = reinterpret_cast<const void*>(kern);
  for (const auto& d : done)
    if (d.first == key && d.second == dev) return B2E_OK;
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.emplace_back(key, dev);
  return B2E_OK;
}

// ---------------------------------------------------------------- launches
int check_gemm_shape(int M, int N, int K) {
  if (M <= 0 || N <= 0 || K <= 0) return fail(B2E_ERR_INVALID, "gemm: empty shape %dx%dx%d", M, N, K);
  if (N % 128 != 0) return fail(B2E_ERR_INVALID, "gemm: N=%d must be a multiple of 128", N);
  if (K % 64 != 0) return fail(B2E_ERR_INVALID, "gemm: K=%d must be a multiple of 64", K);
  return B2E_OK;
}

bool g_gemm_profiling = false;   // b2e_debug_set_clock_buffer: the bias and bias + GELU GEMMs run their timeline instantiations

// B2E_GEMM_BN=128 | 192 or b2e_debug_set_gemm_bn forces the GEMM tile width of the W maps built from then on (A/B
// measurements, the equality tests); 0: the rule of gemm_bn
int g_gemm_bn = -1;   // -1: not decided yet (B2E_GEMM_BN)
inline int gemm_bn_override() {
  if (g_gemm_bn < 0) {
    const char* e = getenv("B2E_GEMM_BN");
    const int v = e ? atoi(e) : 0;
    g_gemm_bn = (v == 128 || v == 192) ? v : 0;
  }
  return g_gemm_bn;
}

// The tile width of the GEMM whose W has N rows (gemm.cuh): 192 wherever that kernel exists (16-bit weights, not a
// gated epilogue) and divides N, else 128.
int gemm_bn(int N, int epi, bool nf4) {
  const bool wide_ok = !nf4 && epi != B2E_EPI_SWIGLU && epi != B2E_EPI_GEGLU && N % 192 == 0;
  if (!wide_ok) return 128;
  const int forced = gemm_bn_override();
  return forced ? forced : 192;
}

// The W operand of a GEMM: a 16-bit [N,K] map (box 64 x bn), or with absmax set the NF4 code map
// (make_tmap_codes) and the block scales [K/64, N] it is dequantised with.  `bn` is the tile width the map was
// built for; the launch runs the kernel of that width.
struct GemmLora;
struct GemmW {
  CUtensorMap tm;
  const float* absmax = nullptr;
  int bn = GEMM_BN;
  const GemmLora* lora = nullptr;   // NF4 only: the slot's low-rank term, run as extra k-blocks (gemm_nf4_lora_kernel)
};

// The low-rank term U . B_cat^T of an NF4 slot, U = X . A_cat^T (embed/encoders/weights.py: lora_slot_factors).
// With u_ws set, launch_gemm first runs U's 16-bit GEMM from the slot's A operand into the handle's U workspace
// [rows, r128] (*u_ws: the workspace moves when it grows); without, U is given (b2e_gemm_nf4_lora).
struct GemmLora {
  GemmW a;                       // A_cat [r128, K]: the W operand of U's GEMM
  CUtensorMap tm_b;              // B_cat [N, 64 r_blocks], box 64 x 128
  int r_blocks = 0, r128 = 0;    // R / 64; R rounded up to 128 (the rows of A_cat, the columns of U)
  h16* const* u_ws = nullptr;
  const void* u = nullptr;
  int ldu = 0;
};

// epi: the B2E_EPI_* epilogue the GEMM will run with (it decides the tile width with N and the storage)
int make_gemm_w(GemmW* w, const void* base, const float* absmax, uint64_t rows, uint64_t cols, int epi) {
  w->absmax = absmax;
  w->bn = gemm_bn((int)rows, epi, absmax != nullptr);
  return absmax ? make_tmap_codes(&w->tm, base, rows, cols / 2) : make_tmap_h16(&w->tm, base, rows, cols, w->bn);
}

// The LoRA factors of an [N, K] NF4 slot: A_cat 16-bit [round_up(R, 128), K], B_cat 16-bit [N, R], R % 64 == 0
int make_gemm_lora(GemmLora* lo, const void* a_cat, const void* b_cat, int R, int N, int K) {
  if (R <= 0 || R % GEMM_BK != 0) return fail(B2E_ERR_INVALID, "LoRA rank %d must be a positive multiple of 64", R);
  lo->r_blocks = R / GEMM_BK;
  lo->r128 = (R + 127) / 128 * 128;
  int rc;
  if ((rc = make_gemm_w(&lo->a, a_cat, nullptr, lo->r128, K, B2E_EPI_BIAS))) return rc;
  return make_tmap_h16(&lo->tm_b, b_cat, N, R, GEMM_BN);
}

template <int EPI>
int launch_gemm_epi(const CUtensorMap& ta, const GemmW& wb, void* out, const float* bias,
                    const h16* resid, int M, int N, int K, cudaStream_t st, const int* m_dev,
                    const CUtensorMap* tm_u = nullptr) {
  auto kern = gemm_h16_wgmma_kernel<EPI>;
  int smem = GemmPlan<false>::SMEM_BYTES;
  if (N % wb.bn != 0) return fail(B2E_ERR_INVALID, "gemm: N=%d is not a multiple of its W map's tile width %d", N, wb.bn);
  if (wb.lora) {
    int rc = ensure_smem_attr(gemm_nf4_lora_kernel<EPI>, GemmPlan<true>::SMEM_BYTES);
    if (rc) return rc;
    DeviceInfo dev;
    if ((rc = current_device_info(&dev))) return rc;
    const long long tiles = (long long)(N / GEMM_BN) * ((M + GEMM_BM - 1) / GEMM_BM);
    if (tiles > 0x7fffffffLL) return fail(B2E_ERR_INVALID, "gemm: %lld output tiles exceed one grid", tiles);
    CUtensorMap tm_out;
    if ((rc = make_tmap_h16(&tm_out, out, M, epi_is_glu(EPI) ? N / 2 : N, GEMM_BM))) return rc;
    const unsigned grid = (unsigned)(tiles < dev.sms ? tiles : dev.sms);
    gemm_nf4_lora_kernel<EPI><<<grid, GEMM_THREADS, GemmPlan<true>::SMEM_BYTES, st>>>(
        ta, wb.tm, tm_out, static_cast<h16*>(out), bias, resid, M, N, K, m_dev, wb.absmax, *tm_u, wb.lora->tm_b,
        wb.lora->r_blocks);
    CUDA_TRY(cudaGetLastError());
    return B2E_OK;
  }
  if (wb.absmax) {
    kern = gemm_h16_wgmma_kernel<EPI, false, true>;
    smem = GemmPlan<true>::SMEM_BYTES;
  } else if (wb.bn == 192) {
    if constexpr (epi_is_glu(EPI)) {
      return fail(B2E_ERR_INVALID, "gemm: the gated epilogues run 128-wide tiles only");
    } else {
      kern = gemm_h16_wgmma_kernel<EPI, false, false, 192>;
      smem = GemmPlan<false, 192>::SMEM_BYTES;
      if constexpr (EPI == EPI_BIAS || EPI == EPI_BIAS_GELU)
        if (g_gemm_profiling) kern = gemm_h16_wgmma_kernel<EPI, true, false, 192>;
    }
  } else if constexpr (EPI == EPI_BIAS || EPI == EPI_BIAS_GELU) {
    if (g_gemm_profiling) kern = gemm_h16_wgmma_kernel<EPI, true>;
  }
  int rc = ensure_smem_attr(kern, smem);
  if (rc) return rc;
  DeviceInfo dev;
  if ((rc = current_device_info(&dev))) return rc;
  const long long tiles = (long long)(N / wb.bn) * ((M + GEMM_BM - 1) / GEMM_BM);
  if (tiles > 0x7fffffffLL) return fail(B2E_ERR_INVALID, "gemm: %lld output tiles exceed one grid", tiles);
  CUtensorMap tm_out;   // the epilogue's TMA stores: 64-column boxes of 128 rows
  if ((rc = make_tmap_h16(&tm_out, out, M, epi_is_glu(EPI) ? N / 2 : N, GEMM_BM))) return rc;
  // persistent: one CTA per SM (fewer for small problems), each walking its share of the tiles
  const unsigned grid = (unsigned)(tiles < dev.sms ? tiles : dev.sms);
  kern<<<grid, GEMM_THREADS, smem, st>>>(ta, wb.tm, tm_out, static_cast<h16*>(out), bias, resid, M, N, K, m_dev,
                                         wb.absmax);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// A map: [M,K] box 128 rows; W: see GemmW.
// m_dev (nullable): device-resident row count <= M (packed token layout); M sizes the grid and the tensor maps.
// A slot with a low-rank term (tb.lora) launches U's GEMM (when U lives in the handle's workspace) and then the
// NF4 kernel with the tail k-blocks over U.
int launch_gemm(const CUtensorMap& ta, const GemmW& tb, void* out, const float* bias,
                const void* resid, int M, int N, int K, int epi, cudaStream_t st, const int* m_dev = nullptr) {
  const h16* r = static_cast<const h16*>(resid);
  CUtensorMap tm_u;
  if (tb.lora) {
    const GemmLora& lo = *tb.lora;
    const void* u = lo.u;
    int ldu = lo.ldu, rc;
    if (lo.u_ws) {
      u = *lo.u_ws;
      ldu = lo.r128;
      if ((rc = launch_gemm_epi<EPI_BIAS>(ta, lo.a, const_cast<void*>(u), nullptr, nullptr, M, lo.r128, K, st, m_dev)))
        return rc;
    }
    if ((rc = make_tmap_h16(&tm_u, u, M, (uint64_t)lo.r_blocks * GEMM_BK, GEMM_BM, 64, ldu))) return rc;
  }
  switch (epi) {
    case B2E_EPI_BIAS: return launch_gemm_epi<EPI_BIAS>(ta, tb, out, bias, r, M, N, K, st, m_dev, &tm_u);
    case B2E_EPI_BIAS_GELU: return launch_gemm_epi<EPI_BIAS_GELU>(ta, tb, out, bias, r, M, N, K, st, m_dev, &tm_u);
    case B2E_EPI_BIAS_RESID: return launch_gemm_epi<EPI_BIAS_RESID>(ta, tb, out, bias, r, M, N, K, st, m_dev, &tm_u);
    case B2E_EPI_SWIGLU: return launch_gemm_epi<EPI_SWIGLU>(ta, tb, out, bias, r, M, N, K, st, m_dev, &tm_u);
    case B2E_EPI_GEGLU: return launch_gemm_epi<EPI_GEGLU>(ta, tb, out, bias, r, M, N, K, st, m_dev, &tm_u);
  }
  return fail(B2E_ERR_INVALID, "unknown epilogue %d", epi);
}

// A device buffer of n T that only grows.  grow() frees the old one, nulls the pointer and zeroes the capacity
// BEFORE the new cudaMalloc: a failed allocation leaves "nothing allocated", never a dangling pointer behind a
// non-zero capacity that a smaller later call would reuse.  Every reallocation bumps the owner's `gen`: captured
// CUDA graphs hold these pointers (B2EEncoder::buffer_stamp).  Converts to T* wherever a pointer is expected.
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  operator T*() const { return p; }
  // zero: fill a new allocation with zeros (buffers that are read before anything writes them)
  int grow(size_t n, uint64_t& gen, bool zero = false) {
    if (n <= cap) return B2E_OK;
    ++gen;
    release();
    CUDA_TRY(cudaMalloc(&p, n * sizeof(T)));
    if (zero) CUDA_TRY(cudaMemset(p, 0, n * sizeof(T)));
    cap = n;
    return B2E_OK;
  }
  void release() {
    cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

// Scratch that lives on the calling thread's current device: the encoder's per-pass scratch and the thread-local
// scratch of the handle-less entry points, which a process may call on more than one device.
struct DeviceScratch {
  int device = -1;    // the buffers live on this device
  uint64_t gen = 0;   // bumped on every reallocation or device change
};

// A call from another device than the buffers' frees them (Scratch::release) and starts over on this one.
template <typename Scratch>
int follow_device(Scratch& s) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  if (dev != s.device) {
    s.release();
    s.device = dev;
    ++s.gen;
  }
  return B2E_OK;
}

// Per-forward attention inputs derived from the mask (attention3.cuh): additive key bias rows and
// the number of 64-key chunks that hold an attended key.
struct AttnScratch : DeviceScratch {
  DevBuf<float> bias;          // [B, S_pad]
  DevBuf<int> kv_chunks;       // [B]
  DevBuf<int> plain_chunks;    // [B]  leading fully-attended chunks
  int ensure(int B, int S_pad) {
    int rc;
    if ((rc = follow_device(*this)) || (rc = bias.grow((size_t)B * S_pad, gen)) || (rc = kv_chunks.grow(B, gen)) ||
        (rc = plain_chunks.grow(B, gen)))
      return rc;
    return B2E_OK;
  }
  void release() {
    bias.release();
    kv_chunks.release();
    plain_chunks.release();
  }
};

inline int attn_s_pad(int S) { return (S + AT_KC - 1) / AT_KC * AT_KC; }

int attention_prepare(AttnScratch& sc, const int64_t* mask, int B, int S, cudaStream_t st) {
  int rc;
  const int S_pad = attn_s_pad(S);
  if ((rc = sc.ensure(B, S_pad))) return rc;
  attn_prep_kernel<<<(B + 7) / 8, 256, 0, st>>>(mask, sc.bias, sc.kv_chunks, sc.plain_chunks, B, S, S_pad);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// Token layout of a forward pass (pack.cuh): null pointers = the padded [B, S] layout.
struct SeqLayout {
  const int* cu = nullptr;       // [B + 1]
  const int* len = nullptr;      // [B]
  const int* t_real = nullptr;   // [2]: rows in use, packed flag
  const int* tok_src = nullptr;  // [B * S]
};

// Device buffers behind a packed SeqLayout (pack_prepare): per-sequence lengths and prefix flags, cu, t_real, and
// the packed-row -> padded-position map.
struct PackBuffers : DeviceScratch {
  DevBuf<int> len_raw, ok, len;   // [B]
  DevBuf<int> cu;                 // [B + 1]
  DevBuf<int> t_real;             // [2]
  DevBuf<int> src;                // [tokens]
  int ensure(int B, size_t tokens) {
    int rc;
    if ((rc = follow_device(*this)) || (rc = len_raw.grow(B, gen)) || (rc = ok.grow(B, gen)) ||
        (rc = len.grow(B, gen)) || (rc = cu.grow((size_t)B + 1, gen)) || (rc = t_real.grow(2, gen)) ||
        (rc = src.grow(tokens, gen)))
      return rc;
    return B2E_OK;
  }
  void release() {
    len_raw.release(); ok.release(); len.release(); cu.release(); t_real.release(); src.release();
  }
};

template <int D, int MODE, int V>
int launch_attention_kernel(const CUtensorMap& tm, const AttnScratch& sc, void* ctx, int B, int S, int heads,
                            int kv_heads, int window, cudaStream_t st, const SeqLayout& lay) {
  using Cfg = AtCfg<D, V>;
  auto kern = attention_kernel<D, MODE, V>;
  int rc = ensure_smem_attr(kern, Cfg::SMEM_BYTES);
  if (rc) return rc;
  CUtensorMap tm_ctx = {};   // [B*S, heads*D], box 64 x Cfg::COLS: the epilogue role's TMA stores
  if ((V & 128) && (rc = make_tmap_h16(&tm_ctx, ctx, (uint64_t)B * S, (uint64_t)heads * D, 64, Cfg::COLS))) return rc;
  const float scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(D));
  const long long ctas = (long long)heads * B * ((S + Cfg::QT - 1) / Cfg::QT);
  if (ctas > 0x7fffffffLL)
    return fail(B2E_ERR_INVALID, "attention: %lld CTAs (heads=%d B=%d S=%d) exceed one grid", ctas, heads, B, S);
  kern<<<(unsigned)ctas, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(tm, tm_ctx, sc.bias, sc.kv_chunks, sc.plain_chunks, B, S,
                                                    attn_s_pad(S), heads, kv_heads, window, scale_log2e, lay.cu,
                                                    lay.len, static_cast<h16*>(ctx));
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// Variant of the head_dim-64 kernel (attention.cuh: bit 0 plain chunks from attn_prep, bits 2-3 polynomial
// exponentials per four, bit 6 four consumer warpgroups, bit 7 epilogue role, bit 8 timeline stamps);
// B2E_ATT3=<n> or b2e_debug_set_att3_variant picks one of the instantiated ones for A/B measurements.
// 193 (four warpgroups, plain chunks from attn_prep, TMA-store epilogue role) measured fastest of these at the C2
// shape (B=512, S=512, 12 heads) on an H100 SXM, all variants side by side in one process: about 6 % ahead of
// variant 1 (two warpgroups) and 17 % ahead of variant 0; within 3 % of variant 1 at S = 1026.
constexpr int AT_DEFAULT_VARIANT = 193;
int g_att3_variant = -1;
inline int att3_variant() {
  if (g_att3_variant < 0) {
    const char* e = getenv("B2E_ATT3");
    g_att3_variant = e ? atoi(e) : AT_DEFAULT_VARIANT;
  }
  return g_att3_variant;
}

// tkv: [T,3H] box 64x64.  `sc` must have been prepared for this batch's mask.
// window > 0: bidirectional sliding window |q - k| <= window (ModernBERT's local layers), else full attention;
// the windowed kernel takes the variant's warpgroup count and epilogue role.
int launch_attention(const CUtensorMap& tkv, const AttnScratch& sc, void* ctx, int B, int S, int heads,
                     cudaStream_t st, int window = 0, const SeqLayout& lay = SeqLayout()) {
  const int v = att3_variant();
#define B2E_ATT(MODE, V) launch_attention_kernel<64, MODE, V>(tkv, sc, ctx, B, S, heads, heads, window, st, lay)
  if (window > 0) {
    switch (v & 192) {
      case 0: return B2E_ATT(1, 0);
      case 64: return B2E_ATT(1, 64);
      case 128: return B2E_ATT(1, 128);
      case 192: return B2E_ATT(1, 192);
    }
    return fail(B2E_ERR_INVALID, "windowed attention: variant %d has no instantiation (bits 6-7 of the variant pick "
                "0, 64, 128 or 192)", v);
  }
  switch (v) {
    case 0: return B2E_ATT(0, 0);
    case 1: return B2E_ATT(0, 1);
    case 5: return B2E_ATT(0, 5);
    case 64: return B2E_ATT(0, 64);
    case 65: return B2E_ATT(0, 65);
    case 69: return B2E_ATT(0, 69);
    case 193: return B2E_ATT(0, 193);
    case 261: return B2E_ATT(0, 261);   // 5 + timeline stamps
    case 321: return B2E_ATT(0, 321);   // 65 + timeline stamps
  }
#undef B2E_ATT
  return fail(B2E_ERR_INVALID, "attention variant %d is not instantiated (0,1,5,64,65,69,193,261,321)", v);
}

// Causal grouped-query attention, head_dim 128.  qkv is [B*S, (heads + 2 kv_heads)*128]
// with columns  q heads | k heads | v heads;  sc must have been prepared for (mask, B, S).
int launch_attention_causal_d128(const void* qkv, AttnScratch& sc, void* ctx, int B, int S, int heads,
                                 int kv_heads, int window, cudaStream_t st, const SeqLayout& lay = SeqLayout()) {
  CUtensorMap tm;
  const int rc = make_tmap_h16(&tm, qkv, (uint64_t)B * S, (uint64_t)(heads + 2 * kv_heads) * 128, AT_KC);
  if (rc) return rc;
  return launch_attention_kernel<128, 2, 0>(tm, sc, ctx, B, S, heads, kv_heads, window, st, lay);
}

// The one head_dim-32 instantiation (bidirectional, key-padding bias: MiniLM / BGE-small / E5-small, ESM-2 150M),
// outside the variant switch: two consumer warpgroups, plain chunks from attn_prep, every thread storing its own
// output pairs.  Measured on an H100 80GB HBM3 at a 700 W power limit, attn_prep + kernel, the eight combinations of
// warpgroups x plain chunks x epilogue role side by side in one process (three runs each), bfloat16:
//   MiniLM shape B=512 S=512, 12 heads, all rows full:  1.04-1.05 ms (variant 1) | 1.05-1.06 (129) | 1.09-1.10 (0,
//                                                       193) | 1.26-1.32 (64, 192)
//   the same, ragged lengths S/8..S:                    0.769-0.772 (1, 129) | 0.776 (128) | 0.78 (0) | 0.82 (193)
//   ESM2-150M shape B=64 S=1026, 20 heads, ragged:      0.58-0.61 (0, 1, 128, 129) | 0.66-0.69 (193)
// Four warpgroups lose here: with 32-column heads a chunk is too little work per CTA to pay for the wider CTA.
constexpr int AT_D32_VARIANT = 1;

// Bidirectional attention of the BERT and ESM-2 trunks by head_dim: the head_dim-64 kernel of the variant switch or
// the head_dim-32 one.  tqkv: [T, 3H] with box 64 x head_dim (make_tmap_h16(..., AT_KC, head_dim)).
int launch_attention_bidir(const CUtensorMap& tqkv, const AttnScratch& sc, void* ctx, int B, int S, int heads,
                           int head_dim, cudaStream_t st, const SeqLayout& lay = SeqLayout()) {
  if (head_dim == 32)
    return launch_attention_kernel<32, 0, AT_D32_VARIANT>(tqkv, sc, ctx, B, S, heads, heads, 0, st, lay);
  return launch_attention(tqkv, sc, ctx, B, S, heads, st, 0, lay);
}

// Row kernels are instantiated per hidden width HW (rowops.cuh: row_passes / row_lane_on); check_h accepts exactly
// these widths.
#define DISPATCH_H(H, CALL)                                         \
  switch (H) {                                                      \
    case 256: { constexpr int HW = 256; CALL; break; }              \
    case 384: { constexpr int HW = 384; CALL; break; }              \
    case 512: { constexpr int HW = 512; CALL; break; }              \
    case 640: { constexpr int HW = 640; CALL; break; }              \
    case 768: { constexpr int HW = 768; CALL; break; }              \
    case 1024: { constexpr int HW = 1024; CALL; break; }            \
    case 1280: { constexpr int HW = 1280; CALL; break; }            \
    case 2048: { constexpr int HW = 2048; CALL; break; }            \
    case 2560: { constexpr int HW = 2560; CALL; break; }            \
    case 4096: { constexpr int HW = 4096; CALL; break; }            \
    default: return fail(B2E_ERR_INVALID, "hidden size %d not supported (need 256*{1,2,3,4,5,8,10,16}, 384 or 640)", (H)); \
  }

inline int row_blocks(int rows) { return (rows + ROW_WARPS - 1) / ROW_WARPS; }

// The row kernels are instantiated per width (DISPATCH_H): reject every other width up front, i.e.
// at b2e_encoder_create, before any weight is touched, not at the first forward pass.
int check_h(int H) {
  if (H == 384 || H == 640) return B2E_OK;   // the two widths that end on a 128-column half pass
  if (H % 256 != 0) return fail(B2E_ERR_INVALID, "hidden size %d must be a multiple of 256, or 384 or 640", H);
  switch (H / 256) {
    case 1: case 2: case 3: case 4: case 5: case 8: case 10: case 16: return B2E_OK;
  }
  return fail(B2E_ERR_UNSUPPORTED, "hidden size %d not supported (built: 256 x {1,2,3,4,5,8,10,16}, 384, 640)", H);
}

// Pool-weight scratch shared by the fused and the standalone poolers.
struct PoolScratch : DeviceScratch {
  DevBuf<int> seq_len;    // [B]
  DevBuf<int> kill;       // [S]
  DevBuf<int> idx;        // [B]
  DevBuf<float> w;        // [B,S]
  DevBuf<float> count;    // [B]
  DevBuf<float> part;     // [B,nsplit,H]
  int ensure(int B, int S, size_t part_elems) {
    int rc;
    if ((rc = follow_device(*this)) || (rc = seq_len.grow(B, gen)) || (rc = kill.grow(S, gen)) ||
        (rc = idx.grow(B, gen)) || (rc = w.grow((size_t)B * S, gen)) || (rc = count.grow(B, gen)) ||
        (rc = part.grow(part_elems, gen)))
      return rc;
    return B2E_OK;
  }
  void release() {
    seq_len.release(); kill.release(); idx.release(); w.release(); count.release(); part.release();
  }
};

inline int pool_nsplit(int S) {
  int n = (S + 63) / 64;  // ~64 rows per block keeps every SM busy at B >= 32
  return n < 1 ? 1 : (n > 16 ? 16 : n);
}

int launch_pool_weights(PoolScratch& ps, int64_t* mask, int B, int S, int pool_kind, int mutate,
                        cudaStream_t st) {
  seq_len_kernel<<<(B + 7) / 8, 256, 0, st>>>(mask, ps.seq_len, B, S);
  CUDA_TRY(cudaMemsetAsync(ps.kill, 0, sizeof(int) * S, st));
  kill_columns_kernel<<<(B + 255) / 256, 256, 0, st>>>(ps.seq_len, ps.kill, B, S);
  pool_weights_kernel<<<(B + 7) / 8, 256, 0, st>>>(mask, ps.seq_len, ps.kill, ps.w, ps.count, B, S,
                                                    pool_kind == B2E_POOL_MEAN_REF ? 1 : 0, mutate);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

int launch_finalize(PoolScratch& ps, float* out, int B, int H, int nsplit, int l2, int round_mode,
                    cudaStream_t st) {
  pool_finalize_kernel<<<B, 256, (H + 32) * sizeof(float), st>>>(ps.part, ps.count, out, H, nsplit,
                                                                 l2, round_mode);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// Restores the caller's current device on scope exit: create / destroy / embed_host switch to the
// encoder's device and must not leave torch's notion of the current device changed behind its back.
struct DeviceGuard {
  int prev = -1;
  DeviceGuard() {
    if (cudaGetDevice(&prev) != cudaSuccess) {
      cudaGetLastError();
      prev = -1;
    }
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

thread_local PoolScratch g_pool_scratch;  // for the handle-less standalone poolers
thread_local AttnScratch g_attn_scratch;  // for the standalone attention op
thread_local PackBuffers g_pack_scratch;  // for b2e_debug_attention_packed

}  // namespace

// The decoder family (Mistral, Qwen3): pre-RMSNorm blocks, head_dim-128 grouped-query causal attention, SwiGLU.
// Qwen3 adds a per-head RMSNorm of q and k before the rotary embedding: two more weight slots per layer.
inline bool is_decoder(int arch) { return arch == B2E_ARCH_MISTRAL || arch == B2E_ARCH_QWEN3; }

namespace {
// The final norm of a family and the tensors it reads
enum FinalNorm {
  NORM_POST_LN,   // post-LayerNorm over tmp + hidden (BERT): the last ACTIVE layer's LayerNorm
  NORM_ADD_LN,    // LayerNorm over the fp32 residual stream xres + tmp (ESM-2, ModernBERT)
  NORM_ADD_RMS,   // RMSNorm over xres + tmp (Mistral, Qwen3)
};

// Layers 0..num_layers-1 of a family; leaves what its FinalNorm reads.  `types` is BERT's alone.
using TrunkFn = int (*)(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t* types, int B, int S,
                        cudaStream_t st, const SeqLayout& lay);

// One row per B2E_ARCH_*: the weight-slot layout of the ABI (embed/encoders/weights.py), what its linear layers
// run and its trunk.  Slot of (layer l, offset k) = lead + stride * l + k.
struct Family {
  int lead, stride;              // fixed leading slots; slots per layer
  int wqkv, wo, w1, w2;          // per-layer offsets of the four GEMM weights
  bool w1_gated;                 // W1 holds 2I rows: two halves interleaved in blocks of 64 (B2E_EPI_SWIGLU/GEGLU)
  int w1_epi;                    // the epilogue W1's GEMM runs with
  FinalNorm norm;
  int norm_g, norm_b;            // the final norm's gain / bias: leading slots, or per-layer offsets of the last
                                 // active layer (NORM_POST_LN); -1: none
  TrunkFn trunk;
};
const Family* family(int arch);   // null: unknown architecture
}  // namespace

// ================================================================== encoder handle
struct B2EEncoder {
  B2EModelDesc desc;
  const Family* fam = nullptr;
  int full_layers = 0;   // desc.num_layers as created (b2e_debug_set_layers may lower desc.num_layers)
  std::vector<const void*> w;
  int device = 0;
  int sms = 0;
  // activations (h16); the pre-norm families' fp32 residual stream; ESM-2's token-dropout scales
  DevBuf<h16> hidden, qkv, ctx, tmp, ffn;
  DevBuf<float> xres, tok_scale;
  PoolScratch pool;
  AttnScratch attn;
  // padding-free token layout of the pooled forward pass (pack.cuh)
  PackBuffers pack;
  // weight operands, one per layer: 16-bit maps, or (b2e_encoder_create_nf4) code maps with their block scales
  std::vector<GemmW> tm_wqkv, tm_wo, tm_w1, tm_w2;
  // (b2e_encoder_create_nf4_lora) the low-rank terms, 4 per layer in the absmax order (r_blocks 0: none; sized
  // once, the GemmW point into it), and U's workspace [tokens, lora_r128]
  std::vector<GemmLora> lora;
  int lora_r128 = 0;
  DevBuf<h16> lora_u;
  // host-loop staging
  DevBuf<int64_t> stage_in;
  DevBuf<float> stage_out;
  cudaStream_t own_stream = nullptr;
  // rotary tables (make_rope_tables); ModernBERT: rope_cos/sin = full-attention layers' table, rope_cos2/sin2 =
  // sliding-attention layers'
  float *rope_cos = nullptr, *rope_sin = nullptr;
  float *rope_cos2 = nullptr, *rope_sin2 = nullptr;

  // weight slot k of layer l (Family)
  const void* slot(int l, int k) const { return w[fam->lead + fam->stride * l + k]; }
  // The final norm's gain (k = 0) and bias (k = 1; null for RMSNorm).  BERT's live in the last active layer, which
  // b2e_debug_set_layers moves.
  const float* final_norm(int k) const {
    const int s = k ? fam->norm_b : fam->norm_g;
    if (s < 0) return nullptr;
    return (const float*)(fam->norm == NORM_POST_LN ? slot(desc.num_layers - 1, s) : w[s]);
  }
  // b2e_embed_host replays one CUDA graph per (batch shape, pooling, staging slot) instead of ~90
  // launches per batch; every graph is dropped when a buffer it points into is reallocated
  struct StepGraph {
    int B, S, pool_kind, l2, has_types, slot;
    cudaGraphExec_t exec;
  };
  std::vector<StepGraph> graphs;
  uint64_t ws_gen = 0;        // bumped when the workspace or a staging buffer is reallocated
  uint64_t graphs_stamp = 0;  // buffer_stamp() at the time the cached graphs were captured
  uint64_t buffer_stamp() const { return ws_gen + pool.gen + attn.gen + pack.gen; }
  void drop_graphs() {
    for (auto& g : graphs) cudaGraphExecDestroy(g.exec);
    graphs.clear();
  }

  int qkv_cols() const {
    return is_decoder(desc.arch) ? (desc.heads + 2 * desc.kv_heads) * desc.head_dim : 3 * desc.hidden;
  }
  int ctx_cols() const { return is_decoder(desc.arch) ? desc.heads * desc.head_dim : desc.hidden; }
  bool has_xres() const { return desc.arch != B2E_ARCH_BERT; }
};

namespace {

size_t tokens_bytes(const B2EModelDesc& d, size_t tokens) {
  if (is_decoder(d.arch))
    return tokens * (size_t)(2 * d.hidden + (2 * d.heads + 2 * d.kv_heads) * d.head_dim + d.intermediate) * 2;
  return tokens * (size_t)(6 * d.hidden + d.intermediate) * 2;
}

int ensure_workspace(B2EEncoder* e, int B, int S) {
  const size_t tokens = (size_t)B * S, H = e->desc.hidden, I = e->desc.intermediate;
  uint64_t& gen = e->ws_gen;
  // zero-filled on allocation: with the packed token layout rows behind the last attended token are never written
  // by a forward pass but ARE read (partial GEMM tiles, the last key chunk of the last sequence) -- they must
  // hold finite values, never whatever the allocator left there
  int rc;
  if ((rc = e->hidden.grow(tokens * H, gen, true)) || (rc = e->tmp.grow(tokens * H, gen, true)) ||
      (rc = e->qkv.grow(tokens * e->qkv_cols(), gen, true)) || (rc = e->ctx.grow(tokens * e->ctx_cols(), gen, true)) ||
      (rc = e->ffn.grow(tokens * I, gen, true)))
    return rc;
  if (e->has_xres() && (rc = e->xres.grow(tokens * H, gen, true))) return rc;
  if (e->desc.arch == B2E_ARCH_ESM2 && (rc = e->tok_scale.grow(B, gen))) return rc;
  if (e->lora_r128 && (rc = e->lora_u.grow(tokens * e->lora_r128, gen, true))) return rc;
  if ((rc = e->pack.ensure(B, tokens))) return rc;
  return e->pool.ensure(B, S, (size_t)B * pool_nsplit(S) * e->desc.hidden);
}

// B2E_PACKED=0 keeps the padded [B, S] layout on every path (A/B measurements, debugging)
int g_packing = -1;   // -1: not decided yet (B2E_PACKED), 0 / 1: b2e_debug_set_packing or the environment
inline bool packing_enabled() {
  if (g_packing < 0) {
    const char* e = getenv("B2E_PACKED");
    g_packing = (e && e[0] == '0') ? 0 : 1;
  }
  return g_packing == 1;
}

// Token layout of this forward pass (pack.cuh), decided and built ON DEVICE from the mask: attended tokens
// back to back when every mask row is a non-empty prefix and `enable`, else the identity ([B, S]) layout
// expressed through the same descriptors.
int pack_prepare(PackBuffers& pk, const int64_t* mask, int B, int S, bool enable, cudaStream_t st, SeqLayout* lay) {
  pack_lengths_kernel<<<(B + 7) / 8, 256, 0, st>>>(mask, pk.len_raw, pk.ok, B, S);
  pack_scan_kernel<<<1, 256, 0, st>>>(pk.len_raw, pk.ok, pk.len, pk.cu, pk.t_real, B, S, enable ? 1 : 0);
  pack_fill_kernel<<<dim3((S + 255) / 256, B), 256, 0, st>>>(pk.len, pk.cu, pk.src, B, S);
  CUDA_TRY(cudaGetLastError());
  lay->cu = pk.cu;
  lay->len = pk.len;
  lay->t_real = pk.t_real;
  lay->tok_src = pk.src;
  return B2E_OK;
}

int validate_batch(const B2EEncoder* e, int B, int S) {
  if (!e) return fail(B2E_ERR_INVALID, "null encoder handle");
  if (B <= 0 || S <= 0) return fail(B2E_ERR_INVALID, "empty batch B=%d S=%d", B, S);
  int cur = -1;
  if (cudaGetDevice(&cur) == cudaSuccess && cur != e->device)
    return fail(B2E_ERR_INVALID, "encoder lives on device %d but device %d is current", e->device, cur);
  if (S > e->desc.max_pos)
    return fail(B2E_ERR_INVALID, "S=%d exceeds max_position_embeddings=%d", S, e->desc.max_pos);
  return B2E_OK;
}

// The GEMM A operands over the activations of a [B*S] pass (box 128 rows) and, for the bidirectional trunks, the
// attention operand qkv (box AT_KC x head_dim; the decoders' launch_attention_causal_d128 maps qkv itself).
struct TrunkMaps {
  CUtensorMap hidden, ctx, ffn, qkv;
};

// Every trunk's step after its embedding: attention_prepare for this batch's mask, then the tensor maps.
int trunk_prologue(B2EEncoder* e, const int64_t* mask, int B, int S, cudaStream_t st, TrunkMaps* tm) {
  const B2EModelDesc& d = e->desc;
  const int M = B * S;
  int rc;
  if ((rc = attention_prepare(e->attn, mask, B, S, st))) return rc;
  if ((rc = make_tmap_h16(&tm->hidden, e->hidden, M, d.hidden, 128))) return rc;
  if ((rc = make_tmap_h16(&tm->ctx, e->ctx, M, e->ctx_cols(), 128))) return rc;
  if ((rc = make_tmap_h16(&tm->ffn, e->ffn, M, d.intermediate, 128))) return rc;
  if (is_decoder(d.arch)) return B2E_OK;
  return make_tmap_h16(&tm->qkv, e->qkv, M, e->qkv_cols(), AT_KC, d.head_dim);
}

// The rotary step of layer l, in place on qkv [M, qkv_cols()] in the token layout `lay` (rows from lay.t_real on are
// not touched): ESM-2 rope_halves<16> (head_dim 32) or <32> over its q and k heads, ModernBERT rope_halves<32> with the
// full-attention (l % global_every == 0) or the sliding-attention table, Mistral rope_halves<64>, Qwen3 the per-head
// q / k RMSNorm fused with the rotation.  The trunks and b2e_debug_rotary launch it.
void launch_rotary(B2EEncoder* e, int l, h16* qkv, int M, int S, cudaStream_t st, const SeqLayout& lay) {
  const B2EModelDesc& d = e->desc;
  if (is_decoder(d.arch)) {
    const int n_rot = d.heads + d.kv_heads;   // q heads and k heads are adjacent columns of qkv
    const unsigned grid = (unsigned)(((long long)M * n_rot * 8 + 255) / 256);
    if (d.arch == B2E_ARCH_QWEN3)
      qk_rmsnorm_rope_kernel<<<grid, 256, 0, st>>>(qkv, (const float*)e->slot(l, 6), (const float*)e->slot(l, 7),
                                                   e->rope_cos, e->rope_sin, M, S, d.heads, d.kv_heads, e->qkv_cols(),
                                                   d.eps, lay.t_real, lay.tok_src);
    else
      rope_halves_kernel<64><<<grid, 256, 0, st>>>(qkv, e->rope_cos, e->rope_sin, M, S, n_rot, e->qkv_cols(),
                                                   lay.t_real, lay.tok_src);
    return;
  }
  const long long rope_work = (long long)M * d.heads * 2;
  const bool global = d.arch != B2E_ARCH_MODERNBERT || (l % d.global_every) == 0;
  const float* cos_t = global ? e->rope_cos : e->rope_cos2;
  const float* sin_t = global ? e->rope_sin : e->rope_sin2;
  if (d.head_dim == 32)   // two threads per head of 2 x 16 frequencies
    rope_halves_kernel<16><<<(unsigned)((rope_work * 2 + 255) / 256), 256, 0, st>>>(
        qkv, cos_t, sin_t, M, S, 2 * d.heads, 3 * d.hidden, lay.t_real, lay.tok_src);
  else
    rope_halves_kernel<32><<<(unsigned)((rope_work * 4 + 255) / 256), 256, 0, st>>>(
        qkv, cos_t, sin_t, M, S, 2 * d.heads, 3 * d.hidden, lay.t_real, lay.tok_src);
}

// The embedding step of a family over M = B*S rows in the token layout `lay`: BERT embed_layernorm into hidden, ESM-2
// the token-dropout scales (into e->tok_scale) and esm_embed into xres, Mistral / Qwen3 the gather into xres,
// ModernBERT the gather into xres and its LayerNorm into hidden.  The trunks and b2e_debug_embed launch it.
int launch_embed(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t* types, int B, int S,
                 h16* hidden, float* xres, cudaStream_t st, const SeqLayout& lay) {
  const B2EModelDesc& d = e->desc;
  const int M = B * S, H = d.hidden;
  switch (d.arch) {
    case B2E_ARCH_BERT:   // leading slots: word, position, token-type embeddings, embedding LayerNorm g/b
      DISPATCH_H(H, (embed_layernorm_kernel<HW><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                         ids, types, (const float*)e->w[0], (const float*)e->w[1], (const float*)e->w[2],
                         (const float*)e->w[3], (const float*)e->w[4], hidden, M, S, d.eps, lay.t_real,
                         lay.tok_src)));
      break;
    case B2E_ARCH_ESM2: {
      const int mask_token = d.reserved - 1;  // reserved = mask_token_id + 1, 0 = token dropout off
      esm_token_scale_kernel<<<(B + 7) / 8, 256, 0, st>>>(ids, mask, e->tok_scale, B, S, mask_token);
      DISPATCH_H(H, (esm_embed_kernel<HW><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                         ids, mask, (const float*)e->w[0], e->tok_scale, xres, M, S, mask_token, lay.t_real,
                         lay.tok_src)));
      break;
    }
    case B2E_ARCH_MODERNBERT:
      DISPATCH_H(H, (modernbert_embed_kernel<HW><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                         ids, (const float*)e->w[0], (const float*)e->w[1], (const float*)e->w[2], xres, hidden, M,
                         d.eps, lay.t_real, lay.tok_src)));
      break;
    default:   // Mistral, Qwen3
      DISPATCH_H(H, (mistral_embed_kernel<HW><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                         ids, (const float*)e->w[0], xres, M, lay.t_real, lay.tok_src)));
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// Layers 0..L-1 up to (and including) the last FFN-down GEMM: leaves the pre-LayerNorm residual sum
// of the final layer split as e->tmp (FFN-down output + bias) and e->hidden (the residual it still has
// to be added to); every earlier LayerNorm output lives in e->hidden.
int run_bert_trunk(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t* types,
                   int B, int S, cudaStream_t st, const SeqLayout& lay) {
  const B2EModelDesc& d = e->desc;
  const int M = B * S, H = d.hidden, I = d.intermediate;
  int rc;
  if ((rc = launch_embed(e, ids, mask, types, B, S, e->hidden, nullptr, st, lay))) return rc;

  TrunkMaps tm;
  if ((rc = trunk_prologue(e, mask, B, S, st, &tm))) return rc;

  for (int l = 0; l < d.num_layers; ++l) {
    if ((rc = launch_gemm(tm.hidden, e->tm_wqkv[l], e->qkv, (const float*)e->slot(l, 1), nullptr, M,
                          3 * H, H, B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    if ((rc = launch_attention_bidir(tm.qkv, e->attn, e->ctx, B, S, d.heads, d.head_dim, st, lay)))
      return rc;
    // the residual add rides on the LayerNorm's coalesced reads, not on the GEMM epilogue
    if ((rc = launch_gemm(tm.ctx, e->tm_wo[l], e->tmp, (const float*)e->slot(l, 3), nullptr, M, H, H,
                          B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    DISPATCH_H(H, (layernorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                       e->tmp, e->hidden, (const float*)e->slot(l, 4), (const float*)e->slot(l, 5),
                       e->hidden, M, d.eps, lay.t_real)));
    if ((rc = launch_gemm(tm.hidden, e->tm_w1[l], e->ffn, (const float*)e->slot(l, 7), nullptr, M, I,
                          H, B2E_EPI_BIAS_GELU, st, lay.t_real)))
      return rc;
    if ((rc = launch_gemm(tm.ffn, e->tm_w2[l], e->tmp, (const float*)e->slot(l, 9), nullptr, M, H, I,
                          B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    if (l + 1 < d.num_layers) {
      DISPATCH_H(H, (layernorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                         e->tmp, e->hidden, (const float*)e->slot(l, 10), (const float*)e->slot(l, 11),
                         e->hidden, M, d.eps, lay.t_real)));
    }
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// ESM-2 (pre-LayerNorm, rotary): transformers/models/esm/modeling_esm.py:189-234 (embeddings with
// token dropout), :318-362 (attention, rotary on q/k), :386-404 / :446-483 (pre-LN blocks).  The
// residual stream e->xres stays fp32; each add_layernorm call folds the previous GEMM output into it
// and emits the next GEMM's h16 input.  Leaves xres (before the last FFN output is added) and e->tmp
// (that FFN-down output): the caller applies emb_layer_norm_after to xres + tmp.
int run_esm_trunk(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t*, int B, int S,
                  cudaStream_t st, const SeqLayout& lay) {
  const B2EModelDesc& d = e->desc;
  const int M = B * S, H = d.hidden, I = d.intermediate, L = d.num_layers;
  int rc;
  if ((rc = launch_embed(e, ids, mask, nullptr, B, S, nullptr, e->xres, st, lay))) return rc;
  TrunkMaps tm;
  if ((rc = trunk_prologue(e, mask, B, S, st, &tm))) return rc;

  DISPATCH_H(H, (add_layernorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                     e->xres, nullptr, (const float*)e->slot(0, 0), (const float*)e->slot(0, 1), e->hidden,
                     M, d.eps, lay.t_real)));
  for (int l = 0; l < L; ++l) {
    if ((rc = launch_gemm(tm.hidden, e->tm_wqkv[l], e->qkv, (const float*)e->slot(l, 3), nullptr, M,
                          3 * H, H, B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    launch_rotary(e, l, e->qkv, M, S, st, lay);
    if ((rc = launch_attention_bidir(tm.qkv, e->attn, e->ctx, B, S, d.heads, d.head_dim, st, lay)))
      return rc;
    if ((rc = launch_gemm(tm.ctx, e->tm_wo[l], e->tmp, (const float*)e->slot(l, 5), nullptr, M, H, H,
                          B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    DISPATCH_H(H, (add_layernorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                       e->xres, e->tmp, (const float*)e->slot(l, 6), (const float*)e->slot(l, 7), e->hidden,
                       M, d.eps, lay.t_real)));
    if ((rc = launch_gemm(tm.hidden, e->tm_w1[l], e->ffn, (const float*)e->slot(l, 9), nullptr, M, I, H,
                          B2E_EPI_BIAS_GELU, st, lay.t_real)))
      return rc;
    if ((rc = launch_gemm(tm.ffn, e->tm_w2[l], e->tmp, (const float*)e->slot(l, 11), nullptr, M, H, I,
                          B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    if (l + 1 < L) {
      DISPATCH_H(H, (add_layernorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                         e->xres, e->tmp, (const float*)e->slot(l + 1, 0), (const float*)e->slot(l + 1, 1),
                         e->hidden, M, d.eps, lay.t_real)));
    }
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// Mistral family (pre-RMSNorm decoder blocks, rotary, grouped-query causal attention, SwiGLU):
// transformers/models/mistral/modeling_mistral.py:328-400 (model), :202-242 (block), :122-180
// (attention), :35-48 (MLP).  Like the ESM-2 trunk it leaves xres (before the last MLP output is
// added) and e->tmp (that down_proj output); the caller applies the final norm to xres + tmp.
// Qwen3 (transformers/models/qwen3/modeling_qwen3.py) is the same block with q_norm / k_norm applied to every q
// and k head before the rotary embedding: qk_rmsnorm_rope_kernel takes rope_halves_kernel<64>'s place.
int run_mistral_trunk(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t*, int B, int S,
                      cudaStream_t st, const SeqLayout& lay) {
  const B2EModelDesc& d = e->desc;
  const int M = B * S, H = d.hidden, I = d.intermediate, L = d.num_layers;
  const int QC = e->qkv_cols(), CC = e->ctx_cols();
  int rc;
  if ((rc = launch_embed(e, ids, mask, nullptr, B, S, nullptr, e->xres, st, lay))) return rc;
  TrunkMaps tm;
  if ((rc = trunk_prologue(e, mask, B, S, st, &tm))) return rc;

  DISPATCH_H(H, (add_rmsnorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                     e->xres, nullptr, (const float*)e->slot(0, 0), e->hidden, M, d.eps, lay.t_real)));
  for (int l = 0; l < L; ++l) {
    if ((rc = launch_gemm(tm.hidden, e->tm_wqkv[l], e->qkv, nullptr, nullptr, M, QC, H, B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    launch_rotary(e, l, e->qkv, M, S, st, lay);
    if ((rc = launch_attention_causal_d128(e->qkv, e->attn, e->ctx, B, S, d.heads, d.kv_heads,
                                           d.sliding_window, st, lay)))
      return rc;
    if ((rc = launch_gemm(tm.ctx, e->tm_wo[l], e->tmp, nullptr, nullptr, M, H, CC, B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    DISPATCH_H(H, (add_rmsnorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                       e->xres, e->tmp, (const float*)e->slot(l, 3), e->hidden, M, d.eps, lay.t_real)));
    // gate and up in one GEMM (interleaved rows), silu(gate) * up in its epilogue: [M, I]
    if ((rc = launch_gemm(tm.hidden, e->tm_w1[l], e->ffn, nullptr, nullptr, M, 2 * I, H,
                          B2E_EPI_SWIGLU, st, lay.t_real)))
      return rc;
    if ((rc = launch_gemm(tm.ffn, e->tm_w2[l], e->tmp, nullptr, nullptr, M, H, I, B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    if (l + 1 < L) {
      DISPATCH_H(H, (add_rmsnorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                         e->xres, e->tmp, (const float*)e->slot(l + 1, 0), e->hidden, M, d.eps, lay.t_real)));
    }
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// ModernBERT (pre-LayerNorm blocks, rotary with one base per layer type, alternating full / sliding-window
// bidirectional attention, GeGLU MLP, no Linear biases): transformers/models/modernbert/modeling_modernbert.py
// :52-71 (embeddings), :232-310 (attention), :74-91 (MLP), :313-343 (block; layer 0 has no attn_norm),
// :424-490 (model).  Leaves xres (before the last MLP output is added) and e->tmp (that output): the caller
// applies final_norm to xres + tmp.
int run_modernbert_trunk(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t*, int B, int S,
                         cudaStream_t st, const SeqLayout& lay) {
  const B2EModelDesc& d = e->desc;
  const int M = B * S, H = d.hidden, I = d.intermediate, L = d.num_layers;
  int rc;
  if ((rc = launch_embed(e, ids, mask, nullptr, B, S, e->hidden, e->xres, st, lay))) return rc;
  TrunkMaps tm;
  if ((rc = trunk_prologue(e, mask, B, S, st, &tm))) return rc;
  for (int l = 0; l < L; ++l) {
    const bool global = (l % d.global_every) == 0;
    if (l > 0) {
      DISPATCH_H(H, (add_layernorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                         e->xres, e->tmp, (const float*)e->slot(l, 0), (const float*)e->slot(l, 1), e->hidden, M,
                         d.eps, lay.t_real)));
    }
    if ((rc = launch_gemm(tm.hidden, e->tm_wqkv[l], e->qkv, nullptr, nullptr, M, 3 * H, H, B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    launch_rotary(e, l, e->qkv, M, S, st, lay);
    if ((rc = launch_attention(tm.qkv, e->attn, e->ctx, B, S, d.heads, st,
                               global ? 0 : d.sliding_window, lay)))
      return rc;
    if ((rc = launch_gemm(tm.ctx, e->tm_wo[l], e->tmp, nullptr, nullptr, M, H, H, B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
    DISPATCH_H(H, (add_layernorm_kernel<HW, h16><<<row_blocks(M), ROW_THREADS, 0, st>>>(
                       e->xres, e->tmp, (const float*)e->slot(l, 4), (const float*)e->slot(l, 5), e->hidden, M,
                       d.eps, lay.t_real)));
    // Wi with its input / gate halves interleaved: gelu(input) * gate in the epilogue -> [M, I]
    if ((rc = launch_gemm(tm.hidden, e->tm_w1[l], e->ffn, nullptr, nullptr, M, 2 * I, H, B2E_EPI_GEGLU, st, lay.t_real)))
      return rc;
    if ((rc = launch_gemm(tm.ffn, e->tm_w2[l], e->tmp, nullptr, nullptr, M, H, I, B2E_EPI_BIAS, st, lay.t_real)))
      return rc;
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// Weight slots (embed/encoders/weights.py):
//   BERT        0 word, 1 position, 2 token-type embeddings, 3/4 embedding LayerNorm g/b; per layer (5 + 12 l):
//               Wqkv, bqkv, Wo, bo, attention LayerNorm g/b, W1, b1, W2, b2, output LayerNorm g/b
//   ESM-2       0 word emb, 1/2 final LayerNorm; per layer (3 + 12 l): ln1 g/b, Wqkv, bqkv, Wo, bo, ln2 g/b, W1, b1,
//               W2, b2
//   Mistral     0 embed_tokens, 1 final norm; per layer (2 + 6 l): input norm, Wqkv, Wo, post-attention norm, Wgu
//               (gate/up interleaved), Wd
//   ModernBERT  0 tok_embeddings, 1/2 embeddings.norm g/b, 3/4 final_norm g/b; per layer (5 + 8 l): attn_norm g/b,
//               Wqkv, Wo, mlp_norm g/b, Wi (input/gate interleaved), mlp.Wo
//   Qwen3       Mistral's, with q_norm, k_norm (fp32 [128]) after the six of each layer (2 + 8 l)
// Indexed by B2E_ARCH_*.
constexpr Family kFamilies[] = {
    {5, 12, 0, 2, 6, 8, false, B2E_EPI_BIAS_GELU, NORM_POST_LN, 10, 11, run_bert_trunk},        // B2E_ARCH_BERT
    {3, 12, 2, 4, 8, 10, false, B2E_EPI_BIAS_GELU, NORM_ADD_LN, 1, 2, run_esm_trunk},           // B2E_ARCH_ESM2
    {2, 6, 1, 2, 4, 5, true, B2E_EPI_SWIGLU, NORM_ADD_RMS, 1, -1, run_mistral_trunk},          // B2E_ARCH_MISTRAL
    {5, 8, 2, 3, 6, 7, true, B2E_EPI_GEGLU, NORM_ADD_LN, 3, 4, run_modernbert_trunk},          // B2E_ARCH_MODERNBERT
    {2, 8, 1, 2, 4, 5, true, B2E_EPI_SWIGLU, NORM_ADD_RMS, 1, -1, run_mistral_trunk},          // B2E_ARCH_QWEN3
};

const Family* family(int arch) {
  return arch >= 0 && arch < (int)(sizeof kFamilies / sizeof kFamilies[0]) ? &kFamilies[arch] : nullptr;
}

// Rotary cos / sin tables [max_pos, cols] of the families that rotate q and k, built once.  Each table's kernel and
// arguments decide results bit for bit: ESM-2 at head_dim 64 keeps rope_table_kernel, ESM-2 at head_dim 32 builds
// angle(p, i) = p * 10000^(-2i/32) over 16 columns, ModernBERT one table per layer type (rope_theta for the
// full-attention layers, rope_theta_local for the sliding ones), Mistral / Qwen3 64 columns of rope_theta.
int make_rope_tables(B2EEncoder* e) {
  const B2EModelDesc& d = e->desc;
  if (d.arch == B2E_ARCH_BERT) return B2E_OK;
  const bool esm = d.arch == B2E_ARCH_ESM2, two = d.arch == B2E_ARCH_MODERNBERT;
  const int cols = is_decoder(d.arch) ? 64 : (esm && d.head_dim == 32) ? 16 : 32;
  const size_t n = (size_t)d.max_pos * cols;
  const unsigned grid = (unsigned)((n + 255) / 256);
  if (cudaMalloc(&e->rope_cos, n * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&e->rope_sin, n * sizeof(float)) != cudaSuccess ||
      (two && (cudaMalloc(&e->rope_cos2, n * sizeof(float)) != cudaSuccess ||
               cudaMalloc(&e->rope_sin2, n * sizeof(float)) != cudaSuccess)))
    return fail(B2E_ERR_CUDA, "cudaMalloc of the rotary tables failed");
  if (esm && d.head_dim == 64)
    rope_table_kernel<<<grid, 256>>>(e->rope_cos, e->rope_sin, d.max_pos);
  else
    rope_table_theta_kernel<<<grid, 256>>>(e->rope_cos, e->rope_sin, d.max_pos, cols, esm ? 10000.0f : d.rope_theta);
  if (two) rope_table_theta_kernel<<<grid, 256>>>(e->rope_cos2, e->rope_sin2, d.max_pos, cols, d.rope_theta_local);
  if (cudaDeviceSynchronize() != cudaSuccess)
    return fail(B2E_ERR_CUDA, "rotary table kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
  return B2E_OK;
}

// One norm step over `rows` rows of width H into float or the storage type (n_dev: device row count, or null):
// NORM_POST_LN LayerNorm(add + resid) of two 16-bit inputs (resid may be null), NORM_ADD_LN / NORM_ADD_RMS
// xres += add (add may be null) in the fp32 residual stream, then LayerNorm / RMSNorm of xres (beta unused).
template <typename OutT>
int launch_norm(FinalNorm kind, int H, float* xres, const h16* add, const h16* resid, const float* g,
                const float* b, OutT* out, int rows, float eps, cudaStream_t st, const int* n_dev = nullptr) {
  switch (kind) {
    case NORM_POST_LN:
      DISPATCH_H(H, (layernorm_kernel<HW, OutT><<<row_blocks(rows), ROW_THREADS, 0, st>>>(
                        add, resid, g, b, out, rows, eps, n_dev)));
      break;
    case NORM_ADD_LN:
      DISPATCH_H(H, (add_layernorm_kernel<HW, OutT><<<row_blocks(rows), ROW_THREADS, 0, st>>>(
                        xres, add, g, b, out, rows, eps, n_dev)));
      break;
    case NORM_ADD_RMS:
      DISPATCH_H(H, (add_rmsnorm_kernel<HW, OutT><<<row_blocks(rows), ROW_THREADS, 0, st>>>(
                        xres, add, g, out, rows, eps, n_dev)));
      break;
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// The final norm of b2e_encode over the padded [B*S] rows, into float or the storage type: BERT's last LayerNorm over
// tmp + hidden, or emb_layer_norm_after / final_norm / the final RMSNorm over (residual stream + last FFN output).
template <typename OutT>
int launch_final_norm(B2EEncoder* e, int M, OutT* out, cudaStream_t st) {
  const B2EModelDesc& d = e->desc;
  const float *g = e->final_norm(0), *b = e->final_norm(1);
  const h16* resid = e->fam->norm == NORM_POST_LN ? e->hidden.p : nullptr;
  return launch_norm(e->fam->norm, d.hidden, e->xres, e->tmp, resid, g, b, out, M, d.eps, st);
}

}  // namespace

// ================================================================== C ABI
extern "C" {

int b2e_version(void) { return B2E_ABI_VERSION; }
int b2e_storage_dtype(void) { return kStorageDtype; }

// Profiling hooks (include/b2e_debug.h, not part of the reference-facing ABI).
int b2e_debug_set_att3_clock(void* device_buffer) {
  long long* p = static_cast<long long*>(device_buffer);
  CUDA_TRY(cudaMemcpyToSymbol(g_att_clock, &p, sizeof(p)));
  return B2E_OK;
}

int b2e_debug_set_att3_variant(int variant) {
  g_att3_variant = variant;
  return B2E_OK;
}

int b2e_debug_set_clock_buffer(void* device_buffer) {
  long long* p = static_cast<long long*>(device_buffer);
  g_gemm_profiling = p != nullptr;
  CUDA_TRY(cudaMemcpyToSymbol(g_gemm_clock, &p, sizeof(p)));
  return B2E_OK;
}

int b2e_debug_set_gemm_bn(int bn) {
  if (bn != 0 && bn != 128 && bn != 192) return fail(B2E_ERR_INVALID, "gemm tile width %d: 0, 128 or 192", bn);
  g_gemm_bn = bn;
  return B2E_OK;
}

int b2e_debug_gemm_bn(int n, int epi, int nf4, int* out) {
  if (!out) return fail(B2E_ERR_INVALID, "null argument");
  *out = gemm_bn(n, epi, nf4 != 0);
  return B2E_OK;
}

// 0: every forward pass keeps the padded [B, S] token layout; 1: pooled passes pack attended tokens (default)
int b2e_debug_set_packing(int on) {
  g_packing = on ? 1 : 0;
  return B2E_OK;
}

// Run only the first n layers from now on (1 <= n <= the model's depth; 0 restores the full depth).  The
// output is what a checkpoint truncated to n layers would give: BERT's hidden_states[n]; for the pre-norm
// families the final norm applied to the residual stream after n layers.  Used by tools/drift_report.py.
int b2e_debug_set_layers(B2EEncoder* e, int n) {
  if (!e) return fail(B2E_ERR_INVALID, "null encoder handle");
  if (n == 0) n = e->full_layers;
  if (n < 1 || n > e->full_layers)
    return fail(B2E_ERR_INVALID, "layer count %d outside [1, %d]", n, e->full_layers);
  if (n != e->desc.num_layers) e->drop_graphs();
  e->desc.num_layers = n;
  return B2E_OK;
}
const char* b2e_last_error(void) { return g_err.c_str(); }

int b2e_num_weights(const B2EModelDesc* desc) {
  const Family* f = desc ? family(desc->arch) : nullptr;
  return f ? f->lead + f->stride * desc->num_layers : -1;
}

// Everything b2e_encoder_create would reject about the SHAPE of a model, without touching a device or
// a weight: callers run it before they upload gigabytes of parameters.
int b2e_check_model(const B2EModelDesc* desc) {
  if (!desc) return fail(B2E_ERR_INVALID, "null model description");
  if (desc->num_layers <= 0 || desc->hidden <= 0 || desc->heads <= 0 || desc->intermediate <= 0)
    return fail(B2E_ERR_INVALID, "model description has a non-positive size");
  int rc;
  if (is_decoder(desc->arch)) {
    const char* fam = desc->arch == B2E_ARCH_QWEN3 ? "Qwen3" : "Mistral";
    if (desc->head_dim != 128 || desc->kv_heads <= 0 || desc->heads % desc->kv_heads != 0)
      return fail(B2E_ERR_UNSUPPORTED, "%s: need head_dim 128 and heads %% kv_heads == 0 (got %d/%d x %d)",
                  fam, desc->heads, desc->kv_heads, desc->head_dim);
    if (desc->intermediate % 128 != 0)
      return fail(B2E_ERR_UNSUPPORTED, "%s: intermediate size %d must be a multiple of 128", fam,
                  desc->intermediate);
    if (desc->sliding_window < 0) return fail(B2E_ERR_INVALID, "negative sliding_window");
    if (desc->arch == B2E_ARCH_QWEN3 && desc->sliding_window != 0)
      return fail(B2E_ERR_UNSUPPORTED, "Qwen3: sliding-window layers are not built (got sliding_window %d; built: "
                  "full causal attention in every layer)", desc->sliding_window);
    const int H = desc->hidden, I = desc->intermediate;
    const int QC = (desc->heads + 2 * desc->kv_heads) * 128, CC = desc->heads * 128;
    if (H % 256 != 0) return fail(B2E_ERR_UNSUPPORTED, "%s: hidden size %d must be a multiple of 256", fam, H);
    if ((rc = check_h(H))) return rc;
    if ((rc = check_gemm_shape(128, QC, H))) return rc;
    if ((rc = check_gemm_shape(128, H, CC))) return rc;
    if ((rc = check_gemm_shape(128, 2 * I, H))) return rc;
    return check_gemm_shape(128, H, I);
  }
  if (desc->arch != B2E_ARCH_BERT && desc->arch != B2E_ARCH_ESM2 && desc->arch != B2E_ARCH_MODERNBERT)
    return fail(B2E_ERR_UNSUPPORTED, "arch %d: unknown architecture", desc->arch);
  if (desc->arch == B2E_ARCH_MODERNBERT) {
    if (desc->head_dim != 64)
      return fail(B2E_ERR_UNSUPPORTED, "ModernBERT: need head_dim 64 (got %d)", desc->head_dim);
    if (desc->hidden % 256 != 0)
      return fail(B2E_ERR_UNSUPPORTED, "ModernBERT: hidden size %d must be a multiple of 256", desc->hidden);
    if (desc->global_every <= 0) return fail(B2E_ERR_INVALID, "ModernBERT: global_every must be positive");
    if (desc->sliding_window <= 0) return fail(B2E_ERR_INVALID, "ModernBERT: sliding_window must be positive");
    if ((2 * desc->intermediate) % 256 != 0)
      return fail(B2E_ERR_UNSUPPORTED, "ModernBERT: 2 * intermediate_size = %d must be a multiple of 256 (the gated "
                  "epilogue pairs 128 input with 128 gate columns)", 2 * desc->intermediate);
  }
  if ((desc->head_dim != 64 && desc->head_dim != 32) || desc->heads * desc->head_dim != desc->hidden)
    return fail(B2E_ERR_UNSUPPORTED,
                "need head_dim 64 or 32 and heads*head_dim == hidden (got %d heads x %d, H=%d); built: H in 256 x "
                "{1,2,3,4,5,8,10,16}, 384 and 640 (MiniLM / BGE-small / E5-small: 384 = 12 x 32); of the ESM-2 family "
                "that is esm2_t30_150M (H=640), esm2_t33_650M (H=1280) and esm2_t36_3B (H=2560)",
                desc->heads, desc->head_dim, desc->hidden);
  if ((rc = check_h(desc->hidden))) return rc;
  if ((rc = check_gemm_shape(128, 3 * desc->hidden, desc->hidden))) return rc;
  if ((rc = check_gemm_shape(128, desc->intermediate, desc->hidden))) return rc;
  return check_gemm_shape(128, desc->hidden, desc->intermediate);
}

namespace {
// absmax: nullptr (16-bit matrices) or 4 * num_layers NF4 scale pointers (b2e_encoder_create_nf4); lora_*: nullptr
// or 4 * num_layers LoRA factors in the same order (b2e_encoder_create_nf4_lora)
int create_encoder(const B2EModelDesc* desc, const void* const* weights, int n_weights, const float* const* absmax,
                   int device, B2EEncoder** out, const void* const* lora_a = nullptr,
                   const void* const* lora_b = nullptr, const int* lora_rank = nullptr) {
  if (!desc || !weights || !out) return fail(B2E_ERR_INVALID, "null argument");
  *out = nullptr;
  int rc;
  if ((rc = b2e_check_model(desc))) return rc;
  if (n_weights != b2e_num_weights(desc))
    return fail(B2E_ERR_INVALID, "expected %d weight pointers, got %d", b2e_num_weights(desc), n_weights);
  for (int i = 0; i < n_weights; ++i)
    if (!weights[i]) return fail(B2E_ERR_INVALID, "weight pointer %d is null", i);
  DeviceInfo info;
  if ((rc = device_info(device, &info))) return rc;
  DeviceGuard guard;
  CUDA_TRY(cudaSetDevice(device));

  B2EEncoder* e = new B2EEncoder();
  e->desc = *desc;
  e->fam = family(desc->arch);   // b2e_check_model accepted the architecture
  e->full_layers = desc->num_layers;
  e->w.assign(weights, weights + n_weights);
  e->device = device;
  e->sms = info.sms;
  const Family& f = *e->fam;
  const int L = desc->num_layers, H = desc->hidden, I = desc->intermediate;
  const int QC = e->qkv_cols(), CC = e->ctx_cols();
  e->tm_wqkv.resize(L); e->tm_wo.resize(L); e->tm_w1.resize(L); e->tm_w2.resize(L);
  if (lora_rank) e->lora.resize(4 * (size_t)L);
  for (int l = 0; l < L; ++l) {
    const float* const* s = absmax ? absmax + 4 * l : nullptr;
    if ((rc = make_gemm_w(&e->tm_wqkv[l], e->slot(l, f.wqkv), s ? s[0] : nullptr, QC, H, B2E_EPI_BIAS)) ||
        (rc = make_gemm_w(&e->tm_wo[l], e->slot(l, f.wo), s ? s[1] : nullptr, H, CC, B2E_EPI_BIAS)) ||
        (rc = make_gemm_w(&e->tm_w1[l], e->slot(l, f.w1), s ? s[2] : nullptr, f.w1_gated ? 2 * I : I, H, f.w1_epi)) ||
        (rc = make_gemm_w(&e->tm_w2[l], e->slot(l, f.w2), s ? s[3] : nullptr, H, I, B2E_EPI_BIAS))) {
      b2e_encoder_destroy(e);
      return rc;
    }
    if (!lora_rank) continue;
    GemmW* slots[4] = {&e->tm_wqkv[l], &e->tm_wo[l], &e->tm_w1[l], &e->tm_w2[l]};
    const int rows[4] = {QC, H, f.w1_gated ? 2 * I : I, H}, cols[4] = {H, CC, H, I};
    for (int j = 0; j < 4; ++j) {
      const int i = 4 * l + j;
      if (lora_rank[i] == 0 || !lora_a[i] || !lora_b[i]) continue;
      GemmLora& lo = e->lora[i];
      if ((rc = make_gemm_lora(&lo, lora_a[i], lora_b[i], lora_rank[i], rows[j], cols[j]))) {
        b2e_encoder_destroy(e);
        return rc;
      }
      lo.u_ws = &e->lora_u.p;
      e->lora_r128 = std::max(e->lora_r128, lo.r128);
      slots[j]->lora = &lo;
    }
  }
  if ((rc = make_rope_tables(e))) {
    b2e_encoder_destroy(e);
    return rc;
  }
  *out = e;
  return B2E_OK;
}
}  // namespace

int b2e_encoder_create(const B2EModelDesc* desc, const void* const* weights, int n_weights,
                       int device, B2EEncoder** out) {
  return create_encoder(desc, weights, n_weights, nullptr, device, out);
}

int b2e_encoder_create_nf4(const B2EModelDesc* desc, const void* const* weights, int n_weights,
                           const float* const* absmax, int n_absmax, int device, B2EEncoder** out) {
  if (!desc || !weights || !absmax || !out) return fail(B2E_ERR_INVALID, "null argument");
  *out = nullptr;
  if (n_absmax != 4 * desc->num_layers)
    return fail(B2E_ERR_INVALID, "expected %d NF4 scale pointers (4 per layer), got %d", 4 * desc->num_layers,
                n_absmax);
  // the scales of a tile's k-block are one 512-byte bulk copy: 16-byte aligned
  for (int i = 0; i < n_absmax; ++i)
    if (!absmax[i] || reinterpret_cast<uintptr_t>(absmax[i]) % 16 != 0)
      return fail(B2E_ERR_INVALID, "NF4 scale pointer %d is null or not 16-byte aligned", i);
  return create_encoder(desc, weights, n_weights, absmax, device, out);
}

int b2e_encoder_create_nf4_lora(const B2EModelDesc* desc, const void* const* weights, int n_weights,
                                const float* const* absmax, int n_absmax, const void* const* lora_a,
                                const void* const* lora_b, const int* lora_rank, int n_lora, int device,
                                B2EEncoder** out) {
  if (!desc || !weights || !absmax || !lora_a || !lora_b || !lora_rank || !out)
    return fail(B2E_ERR_INVALID, "null argument");
  *out = nullptr;
  if (n_absmax != 4 * desc->num_layers || n_lora != 4 * desc->num_layers)
    return fail(B2E_ERR_INVALID, "expected %d NF4 scale pointers and LoRA slots (4 per layer), got %d and %d",
                4 * desc->num_layers, n_absmax, n_lora);
  for (int i = 0; i < n_absmax; ++i)
    if (!absmax[i] || reinterpret_cast<uintptr_t>(absmax[i]) % 16 != 0)
      return fail(B2E_ERR_INVALID, "NF4 scale pointer %d is null or not 16-byte aligned", i);
  for (int i = 0; i < n_lora; ++i) {
    if (lora_rank[i] < 0 || lora_rank[i] % 64 != 0)
      return fail(B2E_ERR_INVALID, "LoRA slot %d: rank %d must be a non-negative multiple of 64", i, lora_rank[i]);
    if (lora_rank[i] == 0 || !lora_a[i] || !lora_b[i]) continue;
    if (reinterpret_cast<uintptr_t>(lora_a[i]) % 16 != 0 || reinterpret_cast<uintptr_t>(lora_b[i]) % 16 != 0)
      return fail(B2E_ERR_INVALID, "LoRA slot %d: factor pointers must be 16-byte aligned", i);
  }
  return create_encoder(desc, weights, n_weights, absmax, device, out, lora_a, lora_b, lora_rank);
}

void b2e_encoder_destroy(B2EEncoder* e) {
  if (!e) return;
  DeviceGuard guard;
  cudaSetDevice(e->device);
  for (DevBuf<h16>* b : {&e->hidden, &e->qkv, &e->ctx, &e->tmp, &e->ffn}) b->release();
  e->xres.release(); e->tok_scale.release(); e->stage_in.release(); e->stage_out.release(); e->lora_u.release();
  cudaFree(e->rope_cos); cudaFree(e->rope_sin); cudaFree(e->rope_cos2); cudaFree(e->rope_sin2);
  e->pack.release();
  e->drop_graphs();
  e->pool.release();
  e->attn.release();
  if (e->own_stream) cudaStreamDestroy(e->own_stream);
  delete e;
}

int64_t b2e_workspace_bytes(const B2EEncoder* e, int B, int S) {
  if (!e || B <= 0 || S <= 0) return -1;
  const size_t tokens = (size_t)B * S;
  size_t bytes = tokens_bytes(e->desc, tokens);
  if (e->has_xres()) bytes += tokens * e->desc.hidden * 4 + (size_t)B * sizeof(float);
  bytes += tokens * sizeof(float) + (size_t)S * sizeof(int) + (size_t)B * (2 * sizeof(int) + sizeof(float));
  bytes += (size_t)B * pool_nsplit(S) * e->desc.hidden * sizeof(float);
  bytes += tokens * e->lora_r128 * 2;
  return (int64_t)bytes;
}

int b2e_encode(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t* types, int B,
               int S, void* out_hidden, int out_dtype, void* stream) {
  int rc;
  if ((rc = validate_batch(e, B, S))) return rc;
  if (!ids || !mask || !out_hidden) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (out_dtype != B2E_DTYPE_F32 && out_dtype != kStorageDtype)
    return fail(B2E_ERR_INVALID, "encode: out_dtype must be F32 or this build's storage type (%d)", kStorageDtype);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = ensure_workspace(e, B, S))) return rc;
  if ((rc = e->fam->trunk(e, ids, mask, types, B, S, st, SeqLayout()))) return rc;
  if (out_dtype == B2E_DTYPE_F32) return launch_final_norm(e, B * S, (float*)out_hidden, st);
  return launch_final_norm(e, B * S, (h16*)out_hidden, st);
}

int b2e_encode_pooled(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t* types,
                      int B, int S, int pool_kind, int l2, float* out, void* stream) {
  int rc;
  if ((rc = validate_batch(e, B, S))) return rc;
  if (!ids || !mask || !out) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (pool_kind < B2E_POOL_MEAN_REF || pool_kind > B2E_POOL_LAST_TOKEN)
    return fail(B2E_ERR_INVALID, "unknown pool_kind %d", pool_kind);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = ensure_workspace(e, B, S))) return rc;
  const B2EModelDesc& d = e->desc;
  const int H = d.hidden;
  PoolScratch& ps = e->pool;
  // Pooled paths run on the padding-free token layout (pack.cuh): only attended tokens go through the GEMMs, norms
  // and attention query tiles; nothing here can observe a padded position.
  SeqLayout lay;
  if ((rc = pack_prepare(e->pack, mask, B, S, packing_enabled(), st, &lay))) return rc;
  if ((rc = e->fam->trunk(e, ids, mask, types, B, S, st, lay))) return rc;
  const FinalNorm norm = e->fam->norm;
  const float *g = e->final_norm(0), *bt = e->final_norm(1);
  if (pool_kind == B2E_POOL_LAST_TOKEN) {
    // only the B selected rows go through the final norm (fp32 end to end)
    seq_len_kernel<<<(B + 7) / 8, 256, 0, st>>>(mask, ps.seq_len, B, S);
    last_token_index_kernel<<<1, 256, 0, st>>>(mask, ps.seq_len, ps.idx, B, S);
    switch (norm) {
      case NORM_POST_LN:
        DISPATCH_H(H, (layernorm_gather_kernel<HW><<<row_blocks(B), ROW_THREADS, 0, st>>>(
                           e->tmp, e->hidden, ps.idx, g, bt, out, B, S, d.eps, lay.cu)));
        break;
      case NORM_ADD_LN:
        DISPATCH_H(H, (addnorm_gather_kernel<HW><<<row_blocks(B), ROW_THREADS, 0, st>>>(
                           e->xres, e->tmp, g, bt, ps.idx, out, B, S, d.eps, lay.cu)));
        break;
      case NORM_ADD_RMS:
        DISPATCH_H(H, (rmsnorm_gather_kernel<HW><<<row_blocks(B), ROW_THREADS, 0, st>>>(
                           e->xres, e->tmp, g, ps.idx, out, B, S, d.eps, lay.cu)));
        break;
    }
    if (l2) l2_normalize_kernel<<<(B + 7) / 8, 256, 0, st>>>(out, B, H);
    CUDA_TRY(cudaGetLastError());
    return B2E_OK;
  }
  // mean poolers: the final norm fused with the masked sum, fp32 end to end, [B,S,H] never written.  The fused path
  // never edits the caller's mask: weights are built from a read-only view.
  if ((rc = launch_pool_weights(ps, const_cast<int64_t*>(mask), B, S, pool_kind, /*mutate=*/0, st)))
    return rc;
  const int nsplit = pool_nsplit(S);
  const int rows_per = (S + nsplit - 1) / nsplit;
  dim3 grid(B, nsplit);
  switch (norm) {
    case NORM_POST_LN:
      DISPATCH_H(H, (layernorm_pool_kernel<HW><<<grid, ROW_THREADS, 0, st>>>(
                         e->tmp, e->hidden, g, bt, ps.w, ps.part, S, rows_per, d.eps, lay.cu)));
      break;
    case NORM_ADD_LN:
      DISPATCH_H(H, (addnorm_pool_kernel<HW, false><<<grid, ROW_THREADS, 0, st>>>(
                         e->xres, e->tmp, g, bt, ps.w, ps.part, S, rows_per, d.eps, lay.cu)));
      break;
    case NORM_ADD_RMS:
      DISPATCH_H(H, (addnorm_pool_kernel<HW, true><<<grid, ROW_THREADS, 0, st>>>(
                         e->xres, e->tmp, g, bt, ps.w, ps.part, S, rows_per, d.eps, lay.cu)));
      break;
  }
  CUDA_TRY(cudaGetLastError());
  return launch_finalize(ps, out, B, H, nsplit, l2, /*round_mode=*/0, st);
}

int b2e_embed_host(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t* types,
                   int64_t n_rows, int S, int batch, int pool_kind, int l2, float* out_host) {
  if (!e) return fail(B2E_ERR_INVALID, "null encoder handle");
  if (n_rows < 0 || batch <= 0) return fail(B2E_ERR_INVALID, "bad n_rows/batch");
  if (n_rows == 0) return B2E_OK;
  if (!ids || !mask || !out_host) return fail(B2E_ERR_INVALID, "null host pointer");
  int rc;
  DeviceGuard guard;
  CUDA_TRY(cudaSetDevice(e->device));   // host entry point: it owns its device context and stream
  if ((rc = validate_batch(e, batch, S))) return rc;
  if (!e->own_stream) CUDA_TRY(cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking));
  cudaStream_t st = e->own_stream;
  const int H = e->desc.hidden;
  // two input slots (ids | mask | types) so batch i+1 uploads while batch i computes
  const size_t slot = (size_t)batch * S * 3;
  if ((rc = e->stage_in.grow(2 * slot, e->ws_gen)) || (rc = e->stage_out.grow((size_t)batch * H * 2, e->ws_gen)))
    return rc;
  static const bool use_graphs = [] {
    const char* v = getenv("B2E_GRAPHS");   // B2E_GRAPHS=0: every batch launches its kernels one by one
    return !(v && v[0] == '0');
  }();
  int which = 0;
  for (int64_t r0 = 0; r0 < n_rows; r0 += batch, which ^= 1) {
    const int B = (int)((n_rows - r0 < batch) ? (n_rows - r0) : batch);
    const size_t n = (size_t)B * S;
    int64_t* d_ids = e->stage_in + which * slot;
    int64_t* d_mask = d_ids + (size_t)batch * S;
    int64_t* d_types = d_mask + (size_t)batch * S;
    float* d_out = e->stage_out + (size_t)which * batch * H;
    CUDA_TRY(cudaMemcpyAsync(d_ids, ids + r0 * S, n * 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(d_mask, mask + r0 * S, n * 8, cudaMemcpyHostToDevice, st));
    if (types) CUDA_TRY(cudaMemcpyAsync(d_types, types + r0 * S, n * 8, cudaMemcpyHostToDevice, st));
    // The first batch runs eagerly (it sizes every buffer and sets the kernels' attributes); later
    // FULL batches replay a graph captured once per (shape, pooling, staging slot): one launch
    // instead of ~90, which is what a small `batch_size` (the reference's default is 8) is bound by.
    const bool eager = !use_graphs || r0 == 0 || B != batch;
    if (eager) {
      if ((rc = b2e_encode_pooled(e, d_ids, d_mask, types ? d_types : nullptr, B, S, pool_kind, l2,
                                  d_out, st)))
        return rc;
    } else {
      if (e->graphs_stamp != e->buffer_stamp()) {
        e->drop_graphs();
        e->graphs_stamp = e->buffer_stamp();
      }
      cudaGraphExec_t exec = nullptr;
      for (const auto& g : e->graphs)
        if (g.B == B && g.S == S && g.pool_kind == pool_kind && g.l2 == l2 &&
            g.has_types == (types != nullptr) && g.slot == which)
          exec = g.exec;
      if (!exec) {
        cudaGraph_t graph = nullptr;
        CUDA_TRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        rc = b2e_encode_pooled(e, d_ids, d_mask, types ? d_types : nullptr, B, S, pool_kind, l2, d_out, st);
        const cudaError_t ce = cudaStreamEndCapture(st, &graph);
        if (rc) {
          if (graph) cudaGraphDestroy(graph);
          return rc;
        }
        if (ce != cudaSuccess) return fail(B2E_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(ce));
        if (e->graphs_stamp != e->buffer_stamp()) {   // a buffer moved during capture: do not keep it
          cudaGraphDestroy(graph);
          return fail(B2E_ERR_CUDA, "workspace reallocated while capturing a step graph");
        }
        const cudaError_t ie = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (ie != cudaSuccess) return fail(B2E_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ie));
        e->graphs.push_back({B, S, pool_kind, l2, types != nullptr, which, exec});
      }
      CUDA_TRY(cudaGraphLaunch(exec, st));
    }
    CUDA_TRY(cudaMemcpyAsync(out_host + r0 * H, d_out, (size_t)B * H * sizeof(float),
                             cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return B2E_OK;
}

int b2e_pool_mean(const void* hidden, int dtype, int64_t* mask, int B, int S, int H, int pool_kind,
                  int quirk_mutate, float* out, void* stream) {
  if (!hidden || !mask || !out) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (B <= 0 || S <= 0) return fail(B2E_ERR_INVALID, "empty batch B=%d S=%d", B, S);
  if (pool_kind != B2E_POOL_MEAN_REF && pool_kind != B2E_POOL_MEAN_PER_ROW)
    return fail(B2E_ERR_INVALID, "pool_mean: pool_kind %d", pool_kind);
  int rc;
  if ((rc = check_h(H))) return rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  PoolScratch& ps = g_pool_scratch;
  const int nsplit = pool_nsplit(S);
  const int rows_per = (S + nsplit - 1) / nsplit;
  if ((rc = ps.ensure(B, S, (size_t)B * nsplit * H))) return rc;
  if ((rc = launch_pool_weights(ps, mask, B, S, pool_kind, quirk_mutate, st))) return rc;
  dim3 grid(B, nsplit);
  int round_mode = 0;
  switch (dtype) {
    case B2E_DTYPE_F32:
      DISPATCH_H(H, (pool_sum_kernel<HW, float><<<grid, ROW_THREADS, 0, st>>>(
                         (const float*)hidden, ps.w, ps.part, S, rows_per)));
      break;
    case B2E_DTYPE_BF16:
      round_mode = 1;
      DISPATCH_H(H, (pool_sum_kernel<HW, bf16><<<grid, ROW_THREADS, 0, st>>>(
                         (const bf16*)hidden, ps.w, ps.part, S, rows_per)));
      break;
    case B2E_DTYPE_F16:
      round_mode = 2;
      DISPATCH_H(H, (pool_sum_kernel<HW, __half><<<grid, ROW_THREADS, 0, st>>>(
                         (const __half*)hidden, ps.w, ps.part, S, rows_per)));
      break;
    default:
      return fail(B2E_ERR_INVALID, "pool_mean: dtype %d", dtype);
  }
  CUDA_TRY(cudaGetLastError());
  return launch_finalize(ps, out, B, H, nsplit, 0, round_mode, st);
}

int b2e_pool_last_token(const void* hidden, int dtype, const int64_t* mask, int B, int S, int H,
                        float* out, void* stream) {
  if (!hidden || !mask || !out) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (B <= 0 || S <= 0) return fail(B2E_ERR_INVALID, "empty batch B=%d S=%d", B, S);
  if (H % 8 != 0) return fail(B2E_ERR_INVALID, "H=%d must be a multiple of 8", H);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  PoolScratch& ps = g_pool_scratch;
  if ((rc = ps.ensure(B, S, 0))) return rc;
  seq_len_kernel<<<(B + 7) / 8, 256, 0, st>>>(mask, ps.seq_len, B, S);
  last_token_index_kernel<<<1, 256, 0, st>>>(mask, ps.seq_len, ps.idx, B, S);
  switch (dtype) {
    case B2E_DTYPE_F32:
      gather_rows_kernel<float><<<B, 128, 0, st>>>((const float*)hidden, ps.idx, out, B, S, H);
      break;
    case B2E_DTYPE_BF16:
      gather_rows_kernel<bf16><<<B, 128, 0, st>>>((const bf16*)hidden, ps.idx, out, B, S, H);
      break;
    case B2E_DTYPE_F16:
      gather_rows_kernel<__half><<<B, 128, 0, st>>>((const __half*)hidden, ps.idx, out, B, S, H);
      break;
    default:
      return fail(B2E_ERR_INVALID, "pool_last_token: dtype %d", dtype);
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

int b2e_l2_normalize(float* x, int64_t n_rows, int H, void* stream) {
  if (!x) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (n_rows <= 0) return B2E_OK;
  if (H % 4 != 0) return fail(B2E_ERR_INVALID, "H=%d must be a multiple of 4", H);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  l2_normalize_kernel<<<(unsigned)((n_rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, (int)n_rows,
                                                                                   H);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

int b2e_adjacent_cosine_dist(const void* emb, int dtype, int64_t n_rows, int H,
                             const int32_t* doc_id, float* out, void* stream) {
  if (n_rows <= 1) return B2E_OK;  // no adjacent pair: nothing to write (semantic_chunk.py:80-81)
  if (!emb || !out) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (H % 8 != 0) return fail(B2E_ERR_INVALID, "H=%d must be a multiple of 8", H);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((n_rows - 1 + 7) / 8);
  switch (dtype) {
    case B2E_DTYPE_F32:
      adjacent_cosine_kernel<float><<<blocks, 256, 0, st>>>((const float*)emb, doc_id, out,
                                                            (int)n_rows, H);
      break;
    case B2E_DTYPE_BF16:
      adjacent_cosine_kernel<bf16><<<blocks, 256, 0, st>>>((const bf16*)emb, doc_id, out,
                                                           (int)n_rows, H);
      break;
    case B2E_DTYPE_F16:
      adjacent_cosine_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)emb, doc_id, out,
                                                             (int)n_rows, H);
      break;
    default:
      return fail(B2E_ERR_INVALID, "adjacent_cosine_dist: dtype %d", dtype);
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

extern "C++" {
namespace {
// b2e_gemm_h16 (absmax null), b2e_gemm_nf4 and b2e_debug_gemm_rows (m_dev set).  An argument the epilogue would not
// read is an error rather than silently dropped: the gated epilogues add no bias, only B2E_EPI_BIAS_RESID adds resid.
int gemm_entry(const void* A, const void* W, const float* absmax, const float* bias, const void* resid, void* out,
               int M, int N, int K, int epi, const int* m_dev, void* stream, const GemmLora* lora = nullptr) {
  if (!A || !W || !out) return fail(B2E_ERR_INVALID, "null tensor pointer");  // bias may be null
  if (absmax && reinterpret_cast<uintptr_t>(absmax) % 16 != 0)
    return fail(B2E_ERR_INVALID, "absmax not 16-byte aligned");
  if (epi == B2E_EPI_BIAS_RESID && !resid) return fail(B2E_ERR_INVALID, "resid epilogue needs resid");
  if (epi != B2E_EPI_BIAS_RESID && resid) return fail(B2E_ERR_INVALID, "gemm: epilogue %d reads no resid", epi);
  if (epi_is_glu(epi) && bias) return fail(B2E_ERR_INVALID, "gemm: the gated epilogues add no bias");
  int rc;
  if ((rc = check_gemm_shape(M, N, K))) return rc;
  if (epi_is_glu(epi) && N % 256 != 0)
    return fail(B2E_ERR_INVALID, "gemm: the gated epilogues need N %% 256 == 0 (got %d)", N);
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  CUtensorMap ta;
  GemmW tb;
  if ((rc = make_tmap_h16(&ta, A, M, K, 128))) return rc;
  if ((rc = make_gemm_w(&tb, W, absmax, N, K, epi))) return rc;
  tb.lora = lora;
  return launch_gemm(ta, tb, out, bias, resid, M, N, K, epi, (cudaStream_t)stream, m_dev);
}
}  // namespace
}  // extern "C++"

int b2e_gemm_h16(const void* A, const void* W, const float* bias, const void* resid, void* out,
                  int M, int N, int K, int epi, void* stream) {
  return gemm_entry(A, W, nullptr, bias, resid, out, M, N, K, epi, nullptr, stream);
}

int b2e_gemm_nf4(const void* A, const void* codes, const float* absmax, const float* bias, const void* resid,
                 void* out, int M, int N, int K, int epi, void* stream) {
  if (!absmax) return fail(B2E_ERR_INVALID, "null tensor pointer");
  return gemm_entry(A, codes, absmax, bias, resid, out, M, N, K, epi, nullptr, stream);
}

int b2e_gemm_nf4_lora(const void* A, const void* codes, const float* absmax, const void* U, int ldu, const void* Bl,
                      int R, const float* bias, const void* resid, void* out, int M, int N, int K, int epi,
                      void* stream) {
  if (!absmax || !U || !Bl) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (R <= 0 || R % GEMM_BK != 0 || ldu < R)
    return fail(B2E_ERR_INVALID, "gemm_nf4_lora: need R a positive multiple of 64 and ldu >= R (got %d, %d)", R, ldu);
  if (reinterpret_cast<uintptr_t>(U) % 16 != 0 || reinterpret_cast<uintptr_t>(Bl) % 16 != 0 || ldu % 8 != 0)
    return fail(B2E_ERR_INVALID, "gemm_nf4_lora: U and Bl must be 16-byte aligned and ldu a multiple of 8");
  GemmLora lo;
  lo.r_blocks = R / GEMM_BK;
  lo.u = U;
  lo.ldu = ldu;
  int rc;
  if ((rc = check_gemm_shape(M, N, K))) return rc;
  if ((rc = make_tmap_h16(&lo.tm_b, Bl, N, R, GEMM_BN))) return rc;
  return gemm_entry(A, codes, absmax, bias, resid, out, M, N, K, epi, nullptr, stream, &lo);
}

int b2e_debug_gemm_rows(const void* A, const void* W, const float* absmax, const float* bias, const void* resid,
                        void* out, int M, int N, int K, int epi, const int* m_dev, void* stream) {
  if (!m_dev) return fail(B2E_ERR_INVALID, "null m_dev");
  return gemm_entry(A, W, absmax, bias, resid, out, M, N, K, epi, m_dev, stream);
}

int b2e_debug_gemm_nf4_lora_rows(const void* A, const void* codes, const float* absmax, const void* A_cat,
                                 const void* B_cat, int R, void* U_ws, const float* bias, const void* resid, void* out,
                                 int M, int N, int K, int epi, const int* m_dev, void* stream) {
  if (!absmax || !A_cat || !B_cat || !U_ws || !m_dev) return fail(B2E_ERR_INVALID, "null tensor pointer");
  int rc;
  if ((rc = check_gemm_shape(M, N, K))) return rc;
  GemmLora lo;
  if ((rc = make_gemm_lora(&lo, A_cat, B_cat, R, N, K))) return rc;
  h16* ws = static_cast<h16*>(U_ws);
  lo.u_ws = &ws;
  return gemm_entry(A, codes, absmax, bias, resid, out, M, N, K, epi, m_dev, stream, &lo);
}

int b2e_attention_d64(const void* qkv, const int64_t* mask, void* ctx, int B, int S, int heads,
                      float* dbg, void* stream) {
  if (!qkv || !mask || !ctx) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (B <= 0 || S <= 0 || heads <= 0) return fail(B2E_ERR_INVALID, "empty attention problem");
  if (dbg) return fail(B2E_ERR_UNSUPPORTED, "the score dump of the first attention kernel is gone: pass NULL");
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CUtensorMap tkv;
  if ((rc = make_tmap_h16(&tkv, qkv, (uint64_t)B * S, (uint64_t)3 * heads * 64, AT_KC))) return rc;
  if ((rc = attention_prepare(g_attn_scratch, mask, B, S, st))) return rc;
  return launch_attention(tkv, g_attn_scratch, ctx, B, S, heads, st);
}

int b2e_attention_d32(const void* qkv, const int64_t* mask, void* ctx, int B, int S, int heads, void* stream) {
  if (!qkv || !mask || !ctx) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (B <= 0 || S <= 0 || heads <= 0) return fail(B2E_ERR_INVALID, "empty attention problem");
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CUtensorMap tkv;
  if ((rc = make_tmap_h16(&tkv, qkv, (uint64_t)B * S, (uint64_t)3 * heads * 32, AT_KC, 32))) return rc;
  if ((rc = attention_prepare(g_attn_scratch, mask, B, S, st))) return rc;
  return launch_attention_bidir(tkv, g_attn_scratch, ctx, B, S, heads, 32, st);
}

int b2e_attention_d64_window(const void* qkv, const int64_t* mask, void* ctx, int B, int S, int heads,
                             int window, void* stream) {
  if (!qkv || !mask || !ctx) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (B <= 0 || S <= 0 || heads <= 0 || window < 0) return fail(B2E_ERR_INVALID, "bad windowed attention problem");
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CUtensorMap tkv;
  if ((rc = make_tmap_h16(&tkv, qkv, (uint64_t)B * S, (uint64_t)3 * heads * 64, AT_KC))) return rc;
  if ((rc = attention_prepare(g_attn_scratch, mask, B, S, st))) return rc;
  return launch_attention(tkv, g_attn_scratch, ctx, B, S, heads, st, window);
}

int b2e_qk_norm_rope(void* qkv, const float* q_gamma, const float* k_gamma, const float* cos_t, const float* sin_t,
                     int T, int S, int heads, int kv_heads, float eps, const int* t_real, const int* tok_src,
                     void* stream) {
  if (!qkv || !q_gamma || !k_gamma || !cos_t || !sin_t) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (T <= 0 || S <= 0 || heads <= 0 || kv_heads <= 0)
    return fail(B2E_ERR_INVALID, "qk_norm_rope: bad problem T=%d S=%d heads=%d/%d", T, S, heads, kv_heads);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  const long long threads = (long long)T * (heads + kv_heads) * 8;
  if ((threads + 255) / 256 > 0x7fffffffLL) return fail(B2E_ERR_INVALID, "qk_norm_rope: %lld threads", threads);
  qk_rmsnorm_rope_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      static_cast<h16*>(qkv), q_gamma, k_gamma, cos_t, sin_t, T, S, heads, kv_heads, (heads + 2 * kv_heads) * 128,
      eps, t_real, tok_src);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

int b2e_attention_causal_d128(const void* qkv, const int64_t* mask, void* ctx, int B, int S, int heads,
                              int kv_heads, int window, void* stream) {
  if (!qkv || !mask || !ctx) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (B <= 0 || S <= 0 || heads <= 0 || kv_heads <= 0 || heads % kv_heads != 0 || window < 0)
    return fail(B2E_ERR_INVALID, "bad causal attention problem B=%d S=%d heads=%d/%d window=%d", B, S,
                heads, kv_heads, window);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = attention_prepare(g_attn_scratch, mask, B, S, st))) return rc;
  return launch_attention_causal_d128(qkv, g_attn_scratch, ctx, B, S, heads, kv_heads, window, st);
}

// The encoder's attention step in its own token layout: pack_prepare decides the layout from the mask (attended
// tokens back to back when every row is a non-empty prefix, else the identity layout), then the same launch as the
// trunks, on tensor maps spanning B*S rows.  qkv / ctx rows are in that layout.
// The handle's rotary step of `layer` (launch_rotary), in place on the caller's qkv [B*S, qkv columns of the
// family], in the token layout the encoder derives from the mask (pack_prepare, b2e_debug_set_packing).
int b2e_debug_rotary(B2EEncoder* e, int layer, void* qkv, const int64_t* mask, int B, int S, void* stream) {
  int rc;
  if ((rc = validate_batch(e, B, S))) return rc;
  if (!qkv || !mask) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (e->desc.arch == B2E_ARCH_BERT) return fail(B2E_ERR_INVALID, "debug_rotary: BERT has no rotary step");
  if (layer < 0 || layer >= e->desc.num_layers)
    return fail(B2E_ERR_INVALID, "debug_rotary: layer %d of %d", layer, e->desc.num_layers);
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = e->pack.ensure(B, (size_t)B * S))) return rc;
  SeqLayout lay;
  if ((rc = pack_prepare(e->pack, mask, B, S, packing_enabled(), st, &lay))) return rc;
  launch_rotary(e, layer, (h16*)qkv, B * S, S, st, lay);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// The handle's embedding step (launch_embed) into the caller's out16 / xres, in the token layout the encoder derives
// from the mask, as b2e_debug_rotary.
int b2e_debug_embed(B2EEncoder* e, const int64_t* ids, const int64_t* mask, const int64_t* types, int B, int S,
                    void* out16, float* xres, void* stream) {
  int rc;
  if ((rc = validate_batch(e, B, S))) return rc;
  const int arch = e->desc.arch;
  const bool wants16 = arch == B2E_ARCH_BERT || arch == B2E_ARCH_MODERNBERT, wants32 = arch != B2E_ARCH_BERT;
  if (!ids || !mask || (wants16 && !out16) || (wants32 && !xres)) return fail(B2E_ERR_INVALID, "null tensor pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = e->pack.ensure(B, (size_t)B * S))) return rc;
  if (arch == B2E_ARCH_ESM2 && (rc = e->tok_scale.grow(B, e->ws_gen))) return rc;
  SeqLayout lay;
  if ((rc = pack_prepare(e->pack, mask, B, S, packing_enabled(), st, &lay))) return rc;
  return launch_embed(e, ids, mask, types, B, S, (h16*)out16, xres, st, lay);
}

int b2e_debug_attention_packed(const void* qkv, const int64_t* mask, void* ctx, int B, int S, int heads,
                               int kv_heads, int head_dim, int window, int causal, void* stream) {
  if (!qkv || !mask || !ctx) return fail(B2E_ERR_INVALID, "null tensor pointer");
  const bool ok = causal ? head_dim == 128 && kv_heads > 0 && heads % kv_heads == 0
                         : (head_dim == 64 || (head_dim == 32 && window == 0)) && kv_heads == heads;
  if (B <= 0 || S <= 0 || heads <= 0 || window < 0 || !ok)
    return fail(B2E_ERR_INVALID, "packed attention: no kernel for B=%d S=%d heads=%d/%d head_dim=%d window=%d "
                "causal=%d", B, S, heads, kv_heads, head_dim, window, causal);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  SeqLayout lay;
  if ((rc = g_pack_scratch.ensure(B, (size_t)B * S))) return rc;
  if ((rc = pack_prepare(g_pack_scratch, mask, B, S, true, st, &lay))) return rc;
  if ((rc = attention_prepare(g_attn_scratch, mask, B, S, st))) return rc;
  if (causal)
    return launch_attention_causal_d128(qkv, g_attn_scratch, ctx, B, S, heads, kv_heads, window, st, lay);
  CUtensorMap tkv;
  if ((rc = make_tmap_h16(&tkv, qkv, (uint64_t)B * S, (uint64_t)3 * heads * head_dim, AT_KC, head_dim))) return rc;
  if (window > 0) return launch_attention(tkv, g_attn_scratch, ctx, B, S, heads, st, window, lay);
  return launch_attention_bidir(tkv, g_attn_scratch, ctx, B, S, heads, head_dim, st, lay);
}

// ---- exact inner-product top-k (retrieval query path)
extern "C++" {
namespace {
struct TopkScratch : DeviceScratch {
  DevBuf<float> score;
  DevBuf<int64_t> index;
  int ensure(size_t elems) {
    int rc;
    if ((rc = follow_device(*this)) || (rc = score.grow(elems, gen)) || (rc = index.grow(elems, gen))) return rc;
    return B2E_OK;
  }
  void release() {
    score.release();
    index.release();
  }
};
thread_local TopkScratch g_topk_scratch;

template <typename T, int QT, int ROWS, int VMAX>
int launch_topk_cfg(const float* queries, int Q, const T* corpus, int64_t N, int H, int k, float* out_score,
                    int64_t* out_index, int sms, cudaStream_t st, const int* run_flag = nullptr) {
  // queries per pass: bounded by QT and by ~160 KiB of shared memory for the query tile
  int qt = QT;
  while (qt > 1 && (size_t)qt * H * 4 > 160 * 1024) qt >>= 1;
  const long long rows_per_cta = (TOPK_THREADS / 32) * ROWS;
  const long long want = (N + rows_per_cta - 1) / rows_per_cta;
  const int grid = (int)(want < (long long)2 * sms ? (want > 0 ? want : 1) : (long long)2 * sms);
  int rc;
  if ((rc = g_topk_scratch.ensure((size_t)grid * qt * k))) return rc;
  auto kern = topk_scan_kernel<T, QT, ROWS, VMAX>;
  const size_t smem_max = (size_t)qt * H * 4 + (size_t)qt * k * 12 + 8 + (size_t)qt * 12;
  // (k varies between calls: always set the attribute to this call's worst case)
  CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max));
  for (int q0 = 0; q0 < Q; q0 += qt) {
    const int nq = (Q - q0 < qt) ? (Q - q0) : qt;
    const size_t smem = (size_t)nq * H * 4 + (size_t)nq * k * 12 + 8 + (size_t)nq * 12;
    kern<<<grid, TOPK_THREADS, smem, st>>>(queries + (size_t)q0 * H, corpus, nq, (long long)N, H, k,
                                           g_topk_scratch.score, g_topk_scratch.index, run_flag);
    topk_merge_kernel<<<nq, TOPK_THREADS, 0, st>>>(g_topk_scratch.score, g_topk_scratch.index, grid, nq,
                                                   k, out_score + (size_t)q0 * k,
                                                   out_index + (size_t)q0 * k, k, run_flag);
  }
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

// one to four queries: the narrow, deeper scan; more: 16 queries per pass
template <typename T, int VWIDE, int VNARROW>
int launch_topk(const float* queries, int Q, const T* corpus, int64_t N, int H, int k, float* out_score,
                int64_t* out_index, int sms, cudaStream_t st, const int* run_flag = nullptr) {
  if (Q <= 4)
    return launch_topk_cfg<T, 4, 8, VNARROW>(queries, Q, corpus, N, H, k, out_score, out_index, sms, st, run_flag);
  return launch_topk_cfg<T, TOPK_QT, 4, VWIDE>(queries, Q, corpus, N, H, k, out_score, out_index, sms, st,
                                               run_flag);
}

// ---- tensor-core fast path (topk_tc.cuh)
struct TcScratch : DeviceScratch {
  DevBuf<float> scores;       // [tiles * 128, 16]
  DevBuf<float> qpad;         // [16, H]
  DevBuf<TcQuery> meta;       // [16]
  DevBuf<unsigned> hist;      // [16, TC_BINS]
  DevBuf<unsigned> cand;      // [16, TC_MAX_CAND]
  DevBuf<unsigned> n_cand;    // [16]
  DevBuf<int> flag;           // [2]: fallback requested; passes that requested it (debug); zeroed on allocation
  DevBuf<float> norm2;        // [1]
  int ensure(size_t rows, size_t h) {
    int rc;
    if ((rc = follow_device(*this)) || (rc = scores.grow(rows * TC_NQ, gen)) || (rc = qpad.grow(TC_NQ * h, gen)) ||
        (rc = meta.grow(TC_NQ, gen)) || (rc = hist.grow((size_t)TC_NQ * TC_BINS, gen)) ||
        (rc = cand.grow((size_t)TC_NQ * TC_MAX_CAND, gen)) || (rc = n_cand.grow(TC_NQ, gen)) ||
        (rc = flag.grow(2, gen, true)) || (rc = norm2.grow(1, gen)))
      return rc;
    return B2E_OK;
  }
  void release() {
    scores.release(); qpad.release(); meta.release(); hist.release(); cand.release(); n_cand.release();
    flag.release(); norm2.release();
  }
};
thread_local TcScratch g_tc_scratch;
}  // namespace
}  // extern "C++"

int b2e_topk_ip(const float* queries, int Q, const void* corpus, int corpus_dtype, int64_t N, int H,
                int k, float* out_scores, int64_t* out_indices, void* stream) {
  if (!queries || !corpus || !out_scores || !out_indices) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (Q <= 0 || N <= 0) return fail(B2E_ERR_INVALID, "topk: empty problem Q=%d N=%lld", Q, (long long)N);
  if (k <= 0 || k > TOPK_MAX_K) return fail(B2E_ERR_INVALID, "topk: k=%d must be in [1, %d]", k, TOPK_MAX_K);
  const int hq = (corpus_dtype == B2E_DTYPE_BF16) ? 256 : 128;   // one 16-byte vector per lane
  if (H % hq != 0 || H > 8192)
    return fail(B2E_ERR_INVALID, "topk: H=%d must be a multiple of %d (<= 8192)", H, hq);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  switch (corpus_dtype) {
    case B2E_DTYPE_F32:
      return launch_topk<float, 6, 3>(queries, Q, (const float*)corpus, N, H, k, out_scores, out_indices, info.sms, st);
    case B2E_DTYPE_BF16:
      return launch_topk<bf16, 3, 2>(queries, Q, (const bf16*)corpus, N, H, k, out_scores, out_indices, info.sms, st);
  }
  return fail(B2E_ERR_INVALID, "topk: corpus dtype %d (F32 or BF16)", corpus_dtype);
}

// largest Euclidean row norm of a float32 matrix (synchronises the stream: an index-build step, not a query step)
int b2e_max_row_norm(const float* x, int64_t N, int H, float* out_host, void* stream) {
  if (!x || !out_host) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (N <= 0 || H <= 0 || H % 4 != 0) return fail(B2E_ERR_INVALID, "max_row_norm: N=%lld H=%d", (long long)N, H);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  TcScratch& sc = g_tc_scratch;
  if ((rc = sc.ensure(TC_ROWS, 128))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(cudaMemsetAsync(sc.norm2, 0, sizeof(float), st));
  max_row_norm2_kernel<<<info.sms * 4, 256, 0, st>>>(x, (long long)N, H, sc.norm2);
  float n2 = 0.0f;
  CUDA_TRY(cudaMemcpyAsync(&n2, sc.norm2, sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  *out_host = sqrtf(n2);
  return B2E_OK;
}

// Exact inner-product top-k with the scan on the tensor cores (topk_tc.cuh).  corpus_max_norm bounds the Euclidean
// norm of every corpus row (b2e_max_row_norm; 1 for normalised embeddings): it sizes the TF32 error margin.
// Same results as b2e_topk_ip; small problems and anything the fast path cannot take go there directly.
int b2e_topk_ip_tc(const float* queries, int Q, const float* corpus, int64_t N, int H, int k,
                   float corpus_max_norm, float* out_scores, int64_t* out_indices, void* stream) {
  if (!queries || !corpus || !out_scores || !out_indices) return fail(B2E_ERR_INVALID, "null tensor pointer");
  const bool fast = N >= 32768 && N < ((int64_t)1 << 31) - TC_ROWS && H % 128 == 0 && H <= 8192 && k > 0 && k <= TOPK_MAX_K &&
                    corpus_max_norm > 0.0f && corpus_max_norm < 1e30f && Q > 0;
  if (!fast) return b2e_topk_ip(queries, Q, corpus, B2E_DTYPE_F32, N, H, k, out_scores, out_indices, stream);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const long long tiles = (N + TC_ROWS - 1) / TC_ROWS;
  TcScratch& sc = g_tc_scratch;
  if ((rc = sc.ensure((size_t)tiles * TC_ROWS, (size_t)H))) return rc;
  CUtensorMap tm_c, tm_q;
  if ((rc = make_tmap_f32(&tm_c, corpus, (uint64_t)N, (uint64_t)H, TC_ROWS))) return rc;
  if ((rc = make_tmap_f32(&tm_q, sc.qpad, TC_NQ, (uint64_t)H, TC_NQ))) return rc;
  if ((rc = ensure_smem_attr(tf32_scan_kernel, TC_SMEM_BYTES))) return rc;
  if ((rc = ensure_smem_attr(score_hist_kernel, TC_NQ * TC_BINS * 4))) return rc;
  if ((rc = ensure_smem_attr(exact_rescore_kernel, TC_MAX_CAND * 8 + 8192 * 4))) return rc;
  CUDA_TRY(cudaMemsetAsync(sc.flag, 0, 2 * sizeof(int), st));
  const int grid_scan = tiles < info.sms ? (int)tiles : info.sms;
  const int grid_rows = info.sms * 2;
  for (int q0 = 0; q0 < Q; q0 += TC_NQ) {
    const int nq = Q - q0 < TC_NQ ? Q - q0 : TC_NQ;
    tc_prepare_queries_kernel<<<TC_NQ, 256, 0, st>>>(queries + (size_t)q0 * H, nq, H, corpus_max_norm, sc.qpad,
                                                     sc.meta);
    CUDA_TRY(cudaMemsetAsync(sc.hist, 0, (size_t)TC_NQ * TC_BINS * sizeof(unsigned), st));
    CUDA_TRY(cudaMemsetAsync(sc.n_cand, 0, TC_NQ * sizeof(unsigned), st));
    tf32_scan_kernel<<<grid_scan, TC_THREADS, TC_SMEM_BYTES, st>>>(tm_c, tm_q, sc.scores, tiles, H);
    score_hist_kernel<<<grid_rows, 512, (size_t)nq * TC_BINS * 4, st>>>(sc.scores, (long long)N, nq, sc.meta,
                                                                        sc.hist);
    score_threshold_kernel<<<1, 32 * TC_NQ, 0, st>>>(sc.hist, nq, (long long)N, k, sc.meta);
    score_select_kernel<<<grid_rows, 512, 0, st>>>(sc.scores, (long long)N, nq, sc.meta, sc.cand, sc.n_cand);
    exact_rescore_kernel<<<nq, 512, (size_t)TC_MAX_CAND * 8 + (size_t)H * 4, st>>>(
        sc.cand, sc.n_cand, sc.meta, queries + (size_t)q0 * H, corpus, H, k, out_scores + (size_t)q0 * k,
        out_indices + (size_t)q0 * k, sc.flag);
  }
  CUDA_TRY(cudaGetLastError());
  // the exact scan redoes the call when a candidate list overflowed; otherwise its kernels return at once
  return launch_topk<float, 6, 3>(queries, Q, corpus, N, H, k, out_scores, out_indices, info.sms, st, sc.flag);
}

// 1 when the last b2e_topk_ip_tc call of this thread had to fall back to the exact scan (synchronises the device)
int b2e_debug_topk_tc_fell_back(int* out) {
  if (!out) return fail(B2E_ERR_INVALID, "null pointer");
  *out = 0;
  if (g_tc_scratch.flag.p == nullptr) return B2E_OK;
  CUDA_TRY(cudaDeviceSynchronize());
  CUDA_TRY(cudaMemcpy(out, g_tc_scratch.flag, sizeof(int), cudaMemcpyDeviceToHost));
  return B2E_OK;
}

// ---- ubinary retrieval: packed bits, Hamming top-K, float rescoring (binsearch.cuh)
extern "C++" {
namespace {
struct BinScratch : DeviceScratch {
  DevBuf<uint32_t> qbits;               // [Q, W]
  DevBuf<unsigned> hist;                // [Q, H+1]
  DevBuf<int> thr;                      // [Q, 2]
  DevBuf<unsigned long long> cand;      // [Q, BIN_MAX_CAND]
  DevBuf<unsigned> n_cand;              // [Q]
  int ensure(int Q, int H) {
    // sized for at least 8 queries of 1024 columns
    const size_t q = (size_t)Q > 8 ? Q : 8, h = (size_t)H > 1024 ? H : 1024;
    int rc;
    if ((rc = follow_device(*this)) || (rc = qbits.grow(q * (h / 32), gen)) || (rc = hist.grow(q * (h + 1), gen)) ||
        (rc = thr.grow(q * 2, gen)) || (rc = cand.grow(q * BIN_MAX_CAND, gen)) || (rc = n_cand.grow(q, gen)))
      return rc;
    return B2E_OK;
  }
  void release() {
    qbits.release(); hist.release(); thr.release(); cand.release(); n_cand.release();
  }
};
thread_local BinScratch g_bin_scratch;

template <int Q>
int launch_bin_pass(const uint32_t* corpus, const uint32_t* qbits, int64_t N, int W, int H, long long K,
                    BinScratch& sc, int q0, int grid, cudaStream_t st) {
  const size_t smem_hist = (size_t)Q * W * 4 + (size_t)Q * (H + 1) * 4;
  const size_t smem_sel = (size_t)Q * W * 4;
  auto hist_k = hamming_hist_kernel<Q>;
  auto sel_k = hamming_select_kernel<Q>;
  int rc;
  // the attribute is set ONCE per kernel and device: to the largest size any call may ask for (Q <= 8 queries of
  // H <= 8192 stay under 160 KiB by the choice of qp in the caller), not to this call's size
  if ((rc = ensure_smem_attr(hist_k, 164 * 1024))) return rc;
  hist_k<<<grid, BIN_THREADS, smem_hist, st>>>(corpus, qbits + (size_t)q0 * W, N, W, H,
                                               sc.hist + (size_t)q0 * (H + 1));
  hamming_threshold_kernel<<<1, 32, 0, st>>>(sc.hist + (size_t)q0 * (H + 1), H, K, Q, sc.thr + 2 * q0);
  sel_k<<<grid, BIN_THREADS, smem_sel, st>>>(corpus, qbits + (size_t)q0 * W, N, W, sc.thr + 2 * q0,
                                             sc.cand + (size_t)q0 * BIN_MAX_CAND, sc.n_cand + q0, BIN_MAX_CAND);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}
}  // namespace
}  // extern "C++"

int b2e_pack_ubinary(const float* emb, int64_t n_rows, int H, uint8_t* out, void* stream) {
  if (n_rows <= 0) return B2E_OK;
  if (!emb || !out) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (H <= 0 || H % 8 != 0) return fail(B2E_ERR_INVALID, "pack_ubinary: H=%d must be a positive multiple of 8", H);
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  const long long total = (long long)n_rows * (H / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)info.sms * 16) blocks = (long long)info.sms * 16;
  pack_ubinary_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(emb, out, n_rows, H);
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

int b2e_search_ubinary(const float* queries, int Q, const uint8_t* corpus_bits, int64_t N, int H, int k,
                       int rescore_multiplier, float* out_scores, int64_t* out_indices, void* stream) {
  if (!queries || !corpus_bits || !out_scores || !out_indices) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (Q <= 0 || N <= 0) return fail(B2E_ERR_INVALID, "search_ubinary: empty problem Q=%d N=%lld", Q, (long long)N);
  if (H <= 0 || H % 32 != 0 || H / 32 > BIN_MAX_WORDS)
    return fail(B2E_ERR_INVALID, "search_ubinary: H=%d must be a multiple of 32 (<= %d)", H, 32 * BIN_MAX_WORDS);
  if (N >= (1ll << 40)) return fail(B2E_ERR_INVALID, "search_ubinary: N=%lld too large", (long long)N);
  if (k <= 0 || rescore_multiplier <= 0) return fail(B2E_ERR_INVALID, "search_ubinary: k and rescore_multiplier must be positive");
  const long long K = (long long)k * rescore_multiplier;
  if (2 * K > BIN_MAX_CAND)
    return fail(B2E_ERR_INVALID, "search_ubinary: k * rescore_multiplier = %lld exceeds %d", K, BIN_MAX_CAND / 2);
  if ((reinterpret_cast<uintptr_t>(corpus_bits) & 15u) != 0)
    return fail(B2E_ERR_INVALID, "search_ubinary: corpus_bits must be 16-byte aligned");
  int rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  BinScratch& sc = g_bin_scratch;
  if ((rc = sc.ensure(Q, H))) return rc;
  const int W = H / 32;
  const uint32_t* corpus = reinterpret_cast<const uint32_t*>(corpus_bits);
  if ((rc = b2e_pack_ubinary(queries, Q, H, reinterpret_cast<uint8_t*>(sc.qbits.p), stream))) return rc;
  CUDA_TRY(cudaMemsetAsync(sc.hist, 0, (size_t)Q * (H + 1) * sizeof(unsigned), st));
  CUDA_TRY(cudaMemsetAsync(sc.n_cand, 0, (size_t)Q * sizeof(unsigned), st));
  long long want = (N + BIN_THREADS - 1) / BIN_THREADS;
  const int grid = (int)(want < (long long)info.sms * 8 ? want : (long long)info.sms * 8);
  // queries per pass over the corpus: as many as the shared-memory histogram allows (<= 8)
  int qp = 8;
  while (qp > 1 && (size_t)qp * (W + H + 1) * 4 > 160 * 1024) qp >>= 1;
  for (int q0 = 0; q0 < Q;) {
    int n = Q - q0 < qp ? Q - q0 : qp;
    if (n >= 8) { n = 8; rc = launch_bin_pass<8>(corpus, sc.qbits, N, W, H, K, sc, q0, grid, st); }
    else if (n >= 4) { n = 4; rc = launch_bin_pass<4>(corpus, sc.qbits, N, W, H, K, sc, q0, grid, st); }
    else if (n >= 2) { n = 2; rc = launch_bin_pass<2>(corpus, sc.qbits, N, W, H, K, sc, q0, grid, st); }
    else { n = 1; rc = launch_bin_pass<1>(corpus, sc.qbits, N, W, H, K, sc, q0, grid, st); }
    if (rc) return rc;
    q0 += n;
  }
  // candidates: the K nearest plus every row tied with the K-th; sort width = next power of two >= 2K
  int n_pow2 = 2;
  while (n_pow2 < 2 * K || n_pow2 < 64) n_pow2 <<= 1;
  if (n_pow2 < BIN_MAX_CAND) n_pow2 = BIN_MAX_CAND;   // ties beyond 2K still fit up to the buffer size
  const size_t smem = (size_t)n_pow2 * 8 + (size_t)H * 4;
  if ((rc = ensure_smem_attr(binary_rescore_kernel, BIN_MAX_CAND * 8 + 32 * BIN_MAX_WORDS * 4))) return rc;
  binary_rescore_kernel<<<Q, BIN_THREADS, smem, st>>>(sc.cand, sc.n_cand, BIN_MAX_CAND, n_pow2, corpus, W, H,
                                                      queries, K, k, out_scores,
                                                      reinterpret_cast<long long*>(out_indices));
  CUDA_TRY(cudaGetLastError());
  return B2E_OK;
}

int b2e_layernorm(const void* in, const float* gamma, const float* beta, void* out, int rows, int H,
                  float eps, int out_dtype, void* stream) {
  if (!in || !gamma || !beta || !out) return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (rows <= 0) return B2E_OK;
  int rc;
  if ((rc = check_h(H))) return rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (out_dtype == B2E_DTYPE_F32)
    return launch_norm(NORM_POST_LN, H, nullptr, (const h16*)in, nullptr, gamma, beta, (float*)out, rows, eps, st);
  if (out_dtype == kStorageDtype)
    return launch_norm(NORM_POST_LN, H, nullptr, (const h16*)in, nullptr, gamma, beta, (h16*)out, rows, eps, st);
  return fail(B2E_ERR_INVALID, "layernorm: out_dtype must be F32 or the storage type");
}

int b2e_debug_norm(int kind, int H, float* xres, const void* add, const void* resid, const float* gamma,
                   const float* beta, void* out, int out_dtype, int rows, float eps, const int* t_real, void* stream) {
  if (kind < NORM_POST_LN || kind > NORM_ADD_RMS) return fail(B2E_ERR_INVALID, "debug_norm: kind %d", kind);
  const FinalNorm k = (FinalNorm)kind;
  if (!gamma || !out || (k == NORM_POST_LN ? !add || !beta : !xres) || (k == NORM_ADD_LN && !beta))
    return fail(B2E_ERR_INVALID, "null tensor pointer");
  if (k != NORM_POST_LN && resid) return fail(B2E_ERR_INVALID, "debug_norm: the fp32-stream norms read no resid");
  if (rows <= 0) return B2E_OK;
  int rc;
  if ((rc = check_h(H))) return rc;
  DeviceInfo info;
  if ((rc = current_device_info(&info))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const h16 *a = (const h16*)add, *r = (const h16*)resid;
  if (out_dtype == B2E_DTYPE_F32) return launch_norm(k, H, xres, a, r, gamma, beta, (float*)out, rows, eps, st, t_real);
  if (out_dtype == kStorageDtype) return launch_norm(k, H, xres, a, r, gamma, beta, (h16*)out, rows, eps, st, t_real);
  return fail(B2E_ERR_INVALID, "debug_norm: out_dtype must be F32 or the storage type");
}

}  // extern "C"
