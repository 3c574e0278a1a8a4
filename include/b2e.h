/* b2e.h -- C ABI of libb2e.so, the H100-native embedding hot path for distllm.
 *
 * Every entry point is plain C: caller-owned pointers and sizes, no C++/torch types, no exceptions.
 * Functions return 0 on success or a B2E_ERR_* code; b2e_last_error() gives the thread-local
 * message.  Device pointers come from torch.Tensor.data_ptr(); work is enqueued on the supplied
 * cudaStream_t (passed as void*) and never synchronises, except b2e_embed_host which owns its
 * copies and returns with the host output complete.
 *
 * Reference interfaces replaced (paths relative to the distllm tree):
 *   b2e_encoder_create      distllm/embed/encoders/auto.py:37-97   (AutoEncoder.__init__)
 *   b2e_encode              distllm/embed/encoders/auto.py:119-138 (AutoEncoder.encode ->
 *                           HF BertModel.forward, transformers/models/bert/modeling_bert.py:628-690, or
 *                           HF MistralModel.forward, transformers/models/mistral/modeling_mistral.py:328-400, or
 *                           HF ModernBertModel.forward, transformers/models/modernbert/modeling_modernbert.py:424-490, or
 *                           HF Qwen3Model.forward, transformers/models/qwen3/modeling_qwen3.py)
 *                           and distllm/embed/encoders/esm2.py:109-134 (Esm2Encoder.encode -> HF
 *                           EsmForMaskedLM, transformers/models/esm/modeling_esm.py:189-516)
 *                           and distllm/embed/encoders/esmc.py:115-134 (EsmCambrianEncoder.encode -> the esm
 *                           package's ESMC.forward, esm/models/esmc.py)
 *   b2e_encode_pooled       distllm/embed/embedders/full_sequence.py:59-69 (encode + pool + normalize)
 *   b2e_embed_host          distllm/embed/embedders/full_sequence.py:57-78 (the whole batch loop,
 *                           host buffers in / host matrix out)
 *   b2e_pool_mean           distllm/embed/poolers/mean.py:13-49    (average_pool, incl. in-place mask edit)
 *   b2e_pool_last_token     distllm/embed/poolers/last_token.py:12-39
 *   b2e_l2_normalize        distllm/embed/embedders/full_sequence.py:68-69 (F.normalize)
 *   b2e_adjacent_cosine_dist distllm/embed/embedders/semantic_chunk.py:24-55
 *   b2e_topk_ip / b2e_topk_ip_tc / b2e_max_row_norm
 *                           distllm/rag/search.py:280-336 (exact float32 search of the query path)
 *   b2e_topk_l2 / b2e_topk_l2_tc / b2e_row_norms
 *                           distllm/rag/search.py:402-666 (FaissIndexV1, metric='l2': faiss IndexFlatL2)
 *   b2e_gemm_h16 / b2e_attention_d64 / b2e_attention_d32 / b2e_attention_causal_d128 / b2e_qk_norm_rope /
 *   b2e_qk_layernorm_rope / b2e_layernorm:
 *                           the building blocks, exported so the parity tests can pin each kernel separately.
 */
#ifndef B2E_H_
#define B2E_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2E_ABI_VERSION 2   /* 2: the 16-bit storage type is a build property (b2e_storage_dtype); b2e_gemm_h16 */

enum {
  B2E_OK = 0,
  B2E_ERR_INVALID = 1,      /* bad argument / unsupported shape */
  B2E_ERR_CUDA = 2,         /* a CUDA runtime or driver call failed */
  B2E_ERR_UNSUPPORTED = 3,  /* architecture or feature not built yet */
  B2E_ERR_NO_DEVICE = 4     /* no sm_90 device: there is no CPU fallback */
};

enum {
  B2E_ARCH_BERT = 0,
  B2E_ARCH_ESM2 = 1,
  B2E_ARCH_MISTRAL = 2,
  B2E_ARCH_MODERNBERT = 3,
  B2E_ARCH_QWEN3 = 4,
  B2E_ARCH_ESMC = 5
};
enum { B2E_DTYPE_F32 = 0, B2E_DTYPE_BF16 = 1, B2E_DTYPE_F16 = 2 };
enum {
  B2E_POOL_MEAN_REF = 0,     /* mean.py semantics incl. the cross-row end-token quirk (mean.py:36) */
  B2E_POOL_MEAN_PER_ROW = 1, /* drop only each row's own first/last token */
  B2E_POOL_LAST_TOKEN = 2
};
enum {
  B2E_EPI_BIAS = 0,       /* acc (+ bias); resid must be NULL */
  B2E_EPI_BIAS_GELU = 1,  /* erf-GELU(acc (+ bias)); resid must be NULL */
  B2E_EPI_BIAS_RESID = 2, /* acc (+ bias) + resid, summed in fp32 and rounded once; resid required */
  B2E_EPI_SWIGLU = 3, /* W rows = gate/up interleaved in blocks of 64; out = silu(gate)*up [M, N/2]; bias and
                         resid must be NULL */
  B2E_EPI_GEGLU = 4   /* same layout, out = gelu(first half) * second half (ModernBERT's Wi: input | gate); bias
                         and resid must be NULL */
};

typedef struct B2EModelDesc {
  int32_t arch;          /* B2E_ARCH_* */
  int32_t num_layers;
  int32_t hidden;        /* H: see b2e_check_model */
  int32_t heads;
  int32_t kv_heads;
  int32_t head_dim;
  int32_t intermediate;  /* I */
  int32_t vocab;
  int32_t max_pos;
  int32_t type_vocab;
  float eps;             /* LayerNorm / RMSNorm epsilon */
  float rope_theta;      /* unused for BERT */
  int32_t sliding_window; /* Mistral: causal window (0 = none); ModernBERT: |i-j| <= sliding_window on local layers */
  int32_t reserved;       /* BERT: padding_idx + 1 selects RoBERTa / XLM-RoBERTa positions, 0 BERT's; ESM-2: see below */
  float rope_theta_local; /* ModernBERT: rotary base of the sliding-attention layers (rope_theta: full-attention layers) */
  int32_t global_every;   /* ModernBERT: layer l uses full attention iff l % global_every == 0 */
} B2EModelDesc;

typedef struct B2EEncoder B2EEncoder;

int b2e_version(void);
/* B2E_DTYPE_F16 (libb2e.so) or B2E_DTYPE_BF16 (libb2e_bf16.so, the same sources built with
 * -DB2E_STORAGE_BF16): the type of every weight matrix handed to b2e_encoder_create, of every 16-bit
 * activation and of the operands of the building-block entry points.  Both feed the tensor cores at the same
 * rate; half keeps 11 significand bits (a 32-layer Mistral-shaped model stays within 1e-3 cosine of fp32 only
 * with it), bfloat16 suffices for the BERT / ESM-2 depths (bench.py's extra.storage_ab times the same GEMM in both
 * builds).  The
 * reference's own reduced precision is half (distllm/embed/encoders/auto.py:77-79). */
int b2e_storage_dtype(void);
const char* b2e_last_error(void);

/* Number of device weight pointers b2e_encoder_create expects for `desc` (BERT: 5 + 12*L, ESM-2:
 * 3 + 12*L, Mistral: 2 + 6*L, ModernBERT: 5 + 8*L, Qwen3: 2 + 8*L -- Mistral's six per layer, then q_norm and
 * k_norm, fp32 [128] each, at every head_dim and width b2e_check_model accepts; order
 * documented in distllm_b200/embed/encoders/weights.py).  Matrices
 * are of the build's 16-bit storage type (b2e_storage_dtype) [out,in] row-major, vectors and embedding
 * tables fp32.  Half values outside +-65504 saturate.  The pointers stay owned by the
 * caller and must outlive the handle.  For B2E_ARCH_BERT, desc.reserved = padding_idx + 1 (> 0) reads position
 * rows as RoBERTa / XLM-RoBERTa do, from the input ids: m = ids != padding_idx, pos = cumsum(m) * m + padding_idx
 * along each sequence (0: row t % S, BERT's); every other rule of the family is BERT's, and the encode entry points
 * refuse S + padding_idx >= max_pos with B2E_ERR_INVALID (the last row of such a batch would read past the
 * position table).  For B2E_ARCH_ESM2, desc.reserved = mask_token_id + 1 enables
 * ESM's token dropout rescaling (0 = off) and token_type_ids are ignored.  For B2E_ARCH_MISTRAL
 * (head_dim 128, heads % kv_heads == 0, intermediate % 128 == 0) the gate/up projection is ONE matrix
 * with rows interleaved in blocks of 64 (see B2E_EPI_SWIGLU), desc.sliding_window = 0 means none, and
 * token_type_ids are ignored.  For B2E_ARCH_MODERNBERT (head_dim 64, (2*intermediate) % 256 == 0, no Linear
 * biases) Wi is ONE matrix with its input / gate halves interleaved in blocks of 64 rows (B2E_EPI_GEGLU),
 * absent norm biases are passed as zero vectors, token_type_ids are ignored.  B2E_ARCH_QWEN3 is B2E_ARCH_MISTRAL
 * with a per-head RMSNorm of every q and k head (over head_dim 128, epsilon desc.eps) before the rotary embedding;
 * desc.sliding_window must be 0.  B2E_ARCH_ESMC (ESM C: 3 + 10*L): 0 embed, 1/2 final LayerNorm g/b (the bias a
 * zero vector); per layer ln_qkv g/b, Wqkv, q_ln, k_ln (fp32 [H]: a LayerNorm over the whole q / k row, no bias),
 * Wo, ffn LayerNorm g/b, W1 (gate/up interleaved, B2E_EPI_SWIGLU), W2; no Linear biases.  The rotary base is
 * desc.rope_theta; the residual scale of the checkpoint is expected folded into Wo and W2; token_type_ids are
 * ignored. */
int b2e_num_weights(const B2EModelDesc* desc);
/* Shape validation only (no device, no weights): 0 when b2e_encoder_create would accept `desc`,
 * else the error it would fail with.  BERT / ESM-2: head_dim 64 or 32, heads*head_dim == H, H in 256 x
 * {1,2,3,4,5,8,10,16}, 384 or 640 (all-MiniLM-L6-v2, bge-small-en-v1.5, e5-small-v2: 384 = 12 x 32; esm2_t30_150M:
 * 640 = 20 x 32), I % 128 == 0; Mistral and Qwen3: head_dim 128 (see above); Mistral, Qwen3 and ModernBERT: H a
 * multiple of 256 (heads*head_dim may differ from H for Mistral and Qwen3); ESMC: head_dim 64, heads*64 == H, H 960
 * (esmc-300m) or 1152 (esmc-600m), I % 128 == 0.
 * Call it BEFORE uploading weights (distllm/embed/encoders/auto.py:59-63 loads the checkpoint unconditionally). */
int b2e_check_model(const B2EModelDesc* desc);
int b2e_encoder_create(const B2EModelDesc* desc, const void* const* weights, int n_weights,
                       int device, B2EEncoder** out);
/* The same model with every weight matrix held in 4-bit NF4 (distllm/embed/encoders/auto.py:44-56's default
 * quantization; distllm_b200/embed/encoders/nf4.py: nf4_quantize): each matrix slot [N,K] of `weights` points to
 * its codes, uint8 [N, K/2] row-major (byte j of a row: column 2j in the high nibble, 2j+1 in the low one), and
 * `absmax` holds 4 * num_layers pointers to the fp32 block scales [K/64, N] (16-byte aligned), per layer in the
 * order Wqkv, Wo, W1 (Mistral / Qwen3: Wgu, ModernBERT: Wi), W2 (Wd, mlp.Wo).  Every GEMM of the handle
 * dequantises W = round16(code[q] * absmax) into shared memory in front of the tensor cores, so the results equal
 * bit for bit those of b2e_encoder_create on the dequantised 16-bit matrices. */
int b2e_encoder_create_nf4(const B2EModelDesc* desc, const void* const* weights, int n_weights,
                           const float* const* absmax, int n_absmax, int device, B2EEncoder** out);
/* b2e_encoder_create_nf4 with LoRA adapters kept unmerged (distllm_b200/embed/encoders/adapters.py): the layer
 * computes dequant(W) x + B_cat (A_cat x), the adapter outside the quantisation, as peft's LoRA layer does on a
 * 4-bit base.  lora_a / lora_b / lora_rank hold n_lora = 4 * num_layers entries in the absmax order; entry i is
 * R = lora_rank[i] (a multiple of 64; 0 or a NULL factor: no adapter on that slot), A_cat 16-bit
 * [round_up(R, 128), K] and B_cat 16-bit [N, R] with the scaling folded in (weights.py: lora_slot_factors), both
 * 16-byte aligned.  Each such GEMM first computes U = X . A_cat^T into a workspace [tokens, max round_up(R, 128)]
 * and then runs R / 64 extra k-blocks of U . B_cat^T inside the NF4 GEMM, before the epilogue. */
int b2e_encoder_create_nf4_lora(const B2EModelDesc* desc, const void* const* weights, int n_weights,
                                const float* const* absmax, int n_absmax, const void* const* lora_a,
                                const void* const* lora_b, const int* lora_rank, int n_lora, int device,
                                B2EEncoder** out);
void b2e_encoder_destroy(B2EEncoder* enc);

/* Bytes of device workspace the handle holds for a [B,S] batch (grown lazily, never shrunk). */
int64_t b2e_workspace_bytes(const B2EEncoder* enc, int B, int S);

/* Full forward pass; writes the final hidden state [B,S,H] as out_dtype (F32 or the storage type). */
int b2e_encode(B2EEncoder* enc, const int64_t* input_ids, const int64_t* attention_mask,
               const int64_t* token_type_ids /* nullable */, int B, int S, void* out_hidden,
               int out_dtype, void* stream);

/* Forward pass with the pooler fused into the final LayerNorm: writes fp32 [B,H]; the [B,S,H]
 * hidden state never reaches HBM.  attention_mask is NOT modified. */
int b2e_encode_pooled(B2EEncoder* enc, const int64_t* input_ids, const int64_t* attention_mask,
                      const int64_t* token_type_ids /* nullable */, int B, int S, int pool_kind,
                      int l2_normalize, float* out_pooled, void* stream);

/* Host-buffer batch loop: n_rows sequences of S tokens in host memory (pinned for full speed),
 * processed `batch` at a time in order (the batch composition matters for B2E_POOL_MEAN_REF);
 * fp32 [n_rows,H] written to host memory.  Synchronous. */
int b2e_embed_host(B2EEncoder* enc, const int64_t* input_ids, const int64_t* attention_mask,
                   const int64_t* token_type_ids /* nullable */, int64_t n_rows, int S, int batch,
                   int pool_kind, int l2_normalize, float* out_host);

/* Standalone poolers over a materialised hidden state (dtype F32/BF16/F16), fp32 [B,H] out.
 * b2e_pool_mean rewrites attention_mask in place like the reference when quirk_mutate != 0. */
int b2e_pool_mean(const void* hidden, int dtype, int64_t* attention_mask, int B, int S, int H,
                  int pool_kind, int quirk_mutate, float* out, void* stream);
int b2e_pool_last_token(const void* hidden, int dtype, const int64_t* attention_mask, int B, int S,
                        int H, float* out, void* stream);
/* In place, per row: x / max(||x||_2, 1e-12), divided as F.normalize divides (so is l2_normalize of
 * b2e_encode_pooled / b2e_embed_host). */
int b2e_l2_normalize(float* x, int64_t n_rows, int H, void* stream);

/* out[i] = 1 - cos(emb[i], emb[i+1]) for i in [0, n_rows-1); pairs with doc_id[i] != doc_id[i+1]
 * (doc_id nullable) are written as NaN. */
int b2e_adjacent_cosine_dist(const void* emb, int dtype, int64_t n_rows, int H,
                             const int32_t* doc_id, float* out, void* stream);

/* Building blocks (storage type, row-major, fp32 accumulation): out[M,N] = epi(A[M,K] . W[N,K]^T + bias [+ resid]).
 * The fp32 result is rounded to nearest-even once; in the half build values beyond +-65504 saturate to +-65504
 * (bfloat16 has fp32's range).  A bias or resid the epilogue does not read (see B2E_EPI_*) is B2E_ERR_INVALID. */
int b2e_gemm_h16(const void* A, const void* W, const float* bias, const void* resid, void* out,
                  int M, int N, int K, int epilogue, void* stream);
/* The same with W in NF4: codes uint8 [N, K/2] and fp32 scales absmax [K/64, N] (see b2e_encoder_create_nf4). */
int b2e_gemm_nf4(const void* A, const void* codes, const float* absmax, const float* bias, const void* resid,
                 void* out, int M, int N, int K, int epilogue, void* stream);
/* b2e_gemm_nf4 plus a low-rank term: out = epi(A . dequant(W)^T + U[:, :R] . Bl^T + bias [+ resid]), U [M, ldu]
 * (ldu >= R, a multiple of 8), Bl [N, R], R a multiple of 64.  Equal bit for bit to b2e_gemm_h16 on the
 * K-concatenated operands [A | U[:, :R]] and [dequant(W) | Bl]. */
int b2e_gemm_nf4_lora(const void* A, const void* codes, const float* absmax, const void* U, int ldu, const void* Bl,
                      int R, const float* bias, const void* resid, void* out, int M, int N, int K, int epilogue,
                      void* stream);
/* qkv [B*S, 3*heads*64] -> ctx [B*S, heads*64]; `reserved` must be NULL (it was a debug score dump). */
int b2e_attention_d64(const void* qkv, const int64_t* attention_mask, void* ctx, int B, int S,
                      int heads, float* reserved, void* stream);
/* The same at head_dim 32 (MiniLM / BGE-small / E5-small, ESM-2 150M): qkv [B*S, 3*heads*32] -> ctx [B*S, heads*32]. */
int b2e_attention_d32(const void* qkv, const int64_t* attention_mask, void* ctx, int B, int S, int heads,
                      void* stream);
/* Same with a BIDIRECTIONAL sliding window: key j is visible to query i iff |i - j| <= window and
 * attention_mask[b,j] != 0 (window == 0: no window).  ModernBERT's local layers: HF
 * masking_utils.sliding_window_bidirectional_overlay with config.sliding_window = local_attention / 2. */
int b2e_attention_d64_window(const void* qkv, const int64_t* attention_mask, void* ctx, int B, int S,
                             int heads, int window, void* stream);
/* Causal grouped-query attention, head_dim 128 (Mistral family):
 * qkv [B*S, (heads + 2*kv_heads)*128] with columns q heads | k heads | v heads (rotary already
 * applied) -> ctx [B*S, heads*128].  Key j is visible to query i iff j <= i, attention_mask[b,j] != 0
 * and (window == 0 or i - j < window). */
int b2e_attention_causal_d128(const void* qkv, const int64_t* attention_mask, void* ctx, int B, int S,
                              int heads, int kv_heads, int window, void* stream);
/* Qwen3's q/k step, in place on qkv [T, (heads + 2*kv_heads)*128] (columns q heads | k heads | v heads): every q
 * head x becomes rotary(q_gamma * x * rsqrt(mean(x^2) + eps)), every k head the same with k_gamma (fp32 [128]
 * each); v heads are untouched.  cos_t / sin_t are [S, 64] fp32 (angle p * theta^(-2i/128)), the position of row t
 * is tok_src[t] % S, or t % S when tok_src is NULL, and *t_real (device, nullable) replaces T as the row count. */
int b2e_qk_norm_rope(void* qkv, const float* q_gamma, const float* k_gamma, const float* cos_t, const float* sin_t,
                     int T, int S, int heads, int kv_heads, float eps, const int* t_real /* nullable */,
                     const int* tok_src /* nullable */, void* stream);
/* ESMC's q/k step, in place on qkv [T, 3H] (columns q | k | v, H = 960 or 1152): the q row x (H columns) becomes
 * rotary(q_gamma * (x - mean) * rsqrt(var + eps)), a LayerNorm over the whole row without bias, the k row the same
 * with k_gamma (fp32 [H] each), the rotation per 64-wide head in the halves convention; v is untouched.  cos_t /
 * sin_t are [S, 32] fp32, positions and t_real / tok_src as in b2e_qk_norm_rope. */
int b2e_qk_layernorm_rope(void* qkv, const float* q_gamma, const float* k_gamma, const float* cos_t,
                          const float* sin_t, int T, int S, int H, float eps, const int* t_real /* nullable */,
                          const int* tok_src /* nullable */, void* stream);
/* Exact inner-product top-k over a device-resident embedding matrix (the retrieval query path,
 * distllm/rag/search.py:280-336: faiss IndexFlatIP through semantic_search_faiss, float32/exact).
 * queries [Q,H] f32, corpus [N,H] F32 or BF16 (both row-major on the device), 1 <= k <= 256,
 * H % 128 == 0.  out_scores / out_indices are [Q,k], sorted by descending score (ties: ascending
 * index); when N < k the tail is filled with -inf / -1. */
int b2e_topk_ip(const float* queries, int Q, const void* corpus, int corpus_dtype, int64_t N, int H,
                int k, float* out_scores, int64_t* out_indices, void* stream);
/* The same search for a float32 corpus with the scan on the tensor cores (TF32) and the decision on exact fp32
 * dot products of the few rows the approximation cannot rule out; identical contract and results (a query whose
 * candidates do not fit the 4096-row buffer makes the call fall back to b2e_topk_ip's scan on the device).
 * corpus_max_norm >= the Euclidean norm of every corpus row (1 for L2-normalised embeddings; b2e_max_row_norm
 * computes it once when the index is built): it sizes the error margin.  Problems below 32 768 rows go straight
 * to b2e_topk_ip, and so do corpora of 2^31 rows or more. */
int b2e_topk_ip_tc(const float* queries, int Q, const float* corpus, int64_t N, int H, int k,
                   float corpus_max_norm, float* out_scores, int64_t* out_indices, void* stream);
/* Largest Euclidean row norm of a device-resident float32 [N,H] matrix -> *out_host (synchronises `stream`:
 * an index-build step).  H % 4 == 0. */
int b2e_max_row_norm(const float* x, int64_t N, int H, float* out_host, void* stream);
/* Exact squared-Euclidean top-k (distllm/rag/search.py:402-666: FaissIndexV1 with metric='l2', faiss IndexFlatL2
 * over the dataset's fp32 embeddings).  queries [Q,H] f32, corpus [N,H] F32 (row-major on the device), 1 <= k <= 256,
 * H % 128 == 0 (zero-padded columns add (0 - 0)^2 = 0).  out_dist / out_indices are [Q,k]: D = sum_i (q_i - x_i)^2
 * in fp32, ascending (ties: ascending index); when N < k the tail is filled with +inf / -1. */
int b2e_topk_l2(const float* queries, int Q, const float* corpus, int64_t N, int H, int k, float* out_dist,
                int64_t* out_indices, void* stream);
/* The same search with the scan on the tensor cores (TF32, ranked on q.x - |x|^2 / 2) and the decision on fp32
 * distances of the rows the approximation cannot rule out; identical contract and results (a query whose
 * candidates do not fit the 4096-row buffer makes the call fall back to b2e_topk_l2's scan on the device).
 * corpus_norm2 [N] f32 on the device and corpus_max_norm come from b2e_row_norms on this corpus (corpus_max_norm^2
 * must bound every entry of corpus_norm2 and every squared row norm).  Problems below 32 768 rows go straight to
 * b2e_topk_l2, and so do corpora of 2^31 rows or more. */
int b2e_topk_l2_tc(const float* queries, int Q, const float* corpus, const float* corpus_norm2, int64_t N, int H,
                   int k, float corpus_max_norm, float* out_dist, int64_t* out_indices, void* stream);
/* Squared Euclidean norm of every row of a device-resident float32 [N,H] matrix -> out_norm2 [N] on the device
 * (nullable; fp32, one fixed summation order), and the largest row norm (its square root) -> *out_max_host, the
 * value b2e_max_row_norm returns.  Synchronises `stream`: an index-build step.  H % 4 == 0. */
int b2e_row_norms(const float* x, int64_t N, int H, float* out_norm2, float* out_max_host, void* stream);
/* Binary retrieval (distllm/rag/search.py, precision='ubinary', search_algorithm='exact'):
 * b2e_pack_ubinary = sentence_transformers quantize_embeddings(x, 'ubinary') as called from search.py:34-56
 * (np.packbits(x > 0): eight dimensions per byte, first dimension in the most significant bit), fp32
 * [n_rows,H] -> uint8 [n_rows,H/8] on the device.
 * b2e_search_ubinary = faiss.IndexBinaryFlat.search + the rescoring of semantic_search_faiss(rescore=True)
 * as called from search.py:202-260 and :280-336: the k*rescore_multiplier rows nearest in Hamming distance to
 * the packed query (ties: smaller row ids), rescored as sum_j q[j]*bit[j] with the float query, top k by
 * descending score into out_scores / out_indices [Q,k] (-inf / -1 past the end of a small corpus; NaN / -2
 * when more rows tie at the threshold distance than the 4096-entry candidate buffer holds).
 * H % 32 == 0, k*rescore_multiplier <= 2048, corpus_bits 16-byte aligned. */
int b2e_pack_ubinary(const float* emb, int64_t n_rows, int H, uint8_t* out_bits, void* stream);
int b2e_search_ubinary(const float* queries, int Q, const uint8_t* corpus_bits, int64_t N, int H, int k,
                       int rescore_multiplier, float* out_scores, int64_t* out_indices, void* stream);
int b2e_layernorm(const void* in_h16, const float* gamma, const float* beta, void* out, int rows,
                  int H, float eps, int out_dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2E_H_ */
