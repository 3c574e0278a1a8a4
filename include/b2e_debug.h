/* b2e_debug.h -- profiling / experiment hooks of libb2e.so.
 *
 * NOT part of the reference-facing ABI (include/b2e.h): nothing in distllm would bind these.  They
 * exist for the tests and the tools under tools/ and are declared here so that every symbol the shared
 * library exports is declared in a header.  0 on success.
 */
#ifndef B2E_DEBUG_H_
#define B2E_DEBUG_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

struct B2EEncoder;
/* run only the first n layers of an encoder handle from now on (0 = full depth again): the per-layer
 * drift report (tools/drift_report.py) compares every depth with the CPU oracle */
int b2e_debug_set_layers(struct B2EEncoder* enc, int n_layers);

/* device buffer of 4 x 512 int64: CTA (0, 0, 0) of a timeline instantiation of the attention kernel (variant bit 8)
 * records (clock64, event code) pairs of its first consumer warpgroup; NULL switches it off */
int b2e_debug_set_att3_clock(void* device_buffer);
/* which instantiated variant of the head_dim-64 attention kernel the next launches use (also B2E_ATT3; -1 = the
 * environment / built-in default) */
int b2e_debug_set_att3_variant(int variant);
/* device buffer of 4 x 256 int64 filled with clock64() stamps by CTA (0, 0) of the bias and bias + GELU GEMMs while
 * set (the timeline instantiation runs instead of the production one; csrc/gemm.cuh: g_gemm_clock); NULL switches
 * it off */
int b2e_debug_set_clock_buffer(void* device_buffer);
/* tile width of the GEMM (csrc/gemm.cuh) for the W maps built from now on -- encoder handles created and
 * b2e_gemm_h16 calls made after it: 128 or 192 forces it wherever the 192-wide kernel exists (16-bit weights, no
 * gated epilogue, N % 192 == 0), 0 restores the built-in rule.  Also B2E_GEMM_BN=128|192.  A/B measurements only. */
int b2e_debug_set_gemm_bn(int bn);
/* *out = the tile width a W map of n rows for epilogue epi (B2E_EPI_*) gets now, NF4 (nf4 != 0) or 16-bit */
int b2e_debug_gemm_bn(int n, int epi, int nf4, int* out);
/* b2e_gemm_h16 (absmax NULL) or b2e_gemm_nf4 (W = codes, absmax set) with the row count the encoders' packed
 * forward passes use: *m_dev (device int, 0 <= *m_dev <= M) rows are computed, the rows from *m_dev to M are not
 * written.  M sizes the grid and the tensor maps. */
int b2e_debug_gemm_rows(const void* A, const void* W, const float* absmax, const float* bias, const void* resid,
                        void* out, int M, int N, int K, int epi, const int* m_dev, void* stream);
/* b2e_gemm_nf4_lora as an NF4 + LoRA encoder slot runs it, with the device row count *m_dev (as above): U = A . A_cat^T
 * on the 16-bit GEMM into U_ws [M, round_up(R, 128)] (A_cat 16-bit [round_up(R, 128), K]), then the NF4 GEMM with
 * R / 64 tail k-blocks over U and B_cat [N, R].  Rows from *m_dev to M of out are not written. */
int b2e_debug_gemm_nf4_lora_rows(const void* A, const void* codes, const float* absmax, const void* A_cat,
                                 const void* B_cat, int R, void* U_ws, const float* bias, const void* resid, void* out,
                                 int M, int N, int K, int epi, const int* m_dev, void* stream);
/* 0: keep the padded [B, S] token layout on every path; 1 (default, also B2E_PACKED=1): pooled forward passes run
 * on the attended tokens only (csrc/pack.cuh).  Drops the handle's cached CUDA graphs' validity: call it before
 * b2e_embed_host, not between its batches. */
int b2e_debug_set_packing(int on);
/* *out = 1 when this thread's last b2e_topk_ip_tc call had to fall back to the exact scan (synchronises the device) */
int b2e_debug_topk_tc_fell_back(int* out);
/* one attention step as an encoder runs it, in the token layout it derives from the mask (csrc/pack.cuh): with
 * every mask row a non-empty prefix, qkv and ctx hold the attended tokens back to back (row cu[b] + s), else they
 * are [B*S] rows in the padded layout.  Both span B*S rows.  causal = 0: bidirectional, head_dim 32 or 64
 * (kv_heads == heads; window > 0: |q - k| <= window, head_dim 64 only); causal = 1: grouped-query causal,
 * head_dim 128 (window > 0: q - k < window).  The head_dim-64 kernel is b2e_debug_set_att3_variant's. */
int b2e_debug_attention_packed(const void* qkv, const int64_t* mask, void* ctx, int B, int S, int heads,
                               int kv_heads, int head_dim, int window, int causal, void* stream);
/* the encoder's rotary step of `layer`, in place on qkv (B*S rows of the family's q | k | v columns, 16-bit storage)
 * in the token layout it derives from the mask, as b2e_debug_attention_packed: ESM-2 and ModernBERT (its full or
 * sliding table by layer) rotate the q and k heads, Mistral the q and k heads, Qwen3 normalises each q / k head with
 * the layer's q_norm / k_norm before rotating it.  Rows past the last attended token (packed layout) and the v
 * heads are not touched. */
int b2e_debug_rotary(struct B2EEncoder* enc, int layer, void* qkv, const int64_t* mask, int B, int S, void* stream);
/* the encoder's embedding step, in the token layout it derives from the mask (as b2e_debug_rotary), over B*S rows:
 * BERT word + position + token-type embeddings and their LayerNorm into out16 (types may be NULL: type 0); ESM-2
 * the token-dropout scale and the masked gather into xres; Mistral / Qwen3 the gather into xres; ModernBERT the
 * gather and its LayerNorm into xres (fp32) and out16.  out16 is 16-bit storage [B*S, H], xres fp32 [B*S, H]; the
 * one a family does not write may be NULL. */
int b2e_debug_embed(struct B2EEncoder* enc, const int64_t* ids, const int64_t* mask, const int64_t* types, int B,
                    int S, void* out16, float* xres, void* stream);
/* one norm step of the trunks over `rows` rows of width H, with the caller's gamma / beta, into out (out_dtype: F32 or
 * the storage type).  kind 0: LayerNorm(add + resid) over two 16-bit inputs (resid may be NULL); kind 1: xres += add
 * in the fp32 residual stream, then LayerNorm of xres; kind 2: the same with RMSNorm (beta unused).  add may be NULL
 * for kinds 1 and 2 (xres is only read).  t_real: device int whose value replaces rows, or NULL. */
int b2e_debug_norm(int kind, int H, float* xres, const void* add, const void* resid, const float* gamma,
                   const float* beta, void* out, int out_dtype, int rows, float eps, const int* t_real, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2E_DEBUG_H_ */
