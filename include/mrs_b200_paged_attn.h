/* mrs_b200_paged_attn.h — C ABI of the paged-KV attention path (libmrs_b200.so).
 * Same symbols and signatures as mistralrs-paged-attn/src/cuda/ffi.rs:96-509 for the in-scope
 * ops; dtype codes 0 = f16, 1 = bf16, 2 = f32, 3 = fp8_e4m3 (cache only).  Cache layouts:
 *   vLLM  K [NB,KVH,D/x,BS,x], V [NB,KVH,D,BS]      (paged_attention_v1/v2, reshape_and_cache)
 *   HND   K,V [NB,KVH,BS,D]                          (flashinfer_decode, *_flashinfer)
 * Errors: cache/vLLM kernels report on stderr and exit(err) like the reference
 * (pagedattention.cuh:46-56); flashinfer_decode returns the cudaError. */
#ifndef MRS_B200_PAGED_ATTN_H
#define MRS_B200_PAGED_ATTN_H
#include <stdbool.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
typedef struct CUstream_st *mrs_stream_t;

/* REF ffi.rs:96-116 / reshape_and_cache_kernel.cu:89-140 */
void reshape_and_cache(void *key, void *value, void *key_cache, void *value_cache, int64_t *slot_mapping,
                       int32_t num_tokens, int32_t num_heads, int32_t head_size, int32_t block_size, int32_t x,
                       int32_t key_stride, int32_t value_stride, mrs_stream_t stream, uint32_t dtype,
                       uint32_t cache_dtype, float *k_scale, float *v_scale);
/* REF ffi.rs:159-176 / flashinfer_decode.cu:250-312 */
void reshape_and_cache_flashinfer(void *key, void *value, void *key_cache, void *value_cache, int64_t *slot_mapping,
                                  int32_t num_tokens, int32_t num_heads, int32_t head_size, int32_t block_size,
                                  int32_t key_stride, int32_t value_stride, float k_scale, float v_scale,
                                  uint32_t dtype, uint32_t cache_dtype, mrs_stream_t stream);
/* REF ffi.rs:178-209 / flashinfer_decode.cu:314-363 */
int32_t flashinfer_decode(void *q, void *key_cache, void *value_cache, const int32_t *kv_indptr,
                          const int32_t *kv_indices, const int32_t *kv_last_page_len, const int32_t *request_indices,
                          const int32_t *kv_tile_indices, const int32_t *o_indptr, const int32_t *kv_chunk_size_ptr,
                          const bool *block_valid_mask, void *o, void *tmp_v, void *tmp_s, int32_t batch_size,
                          int32_t padded_batch_size, int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size,
                          int32_t page_size, int32_t q_stride_n, int32_t q_stride_h, float sm_scale,
                          int32_t window_left, float logits_soft_cap, float k_scale, float v_scale, uint32_t dtype,
                          uint32_t cache_dtype, mrs_stream_t stream);
/* REF ffi.rs:211-268 */
void gather_kv_cache_flashinfer(void *key_cache, void *value_cache, void *k_out, void *v_out,
                                const int32_t *block_table, const int32_t *cu_seq_lens, int32_t num_tokens,
                                int32_t num_seqs, int32_t block_size, int32_t block_table_stride, int32_t num_kv_heads,
                                int32_t head_size, uint32_t out_dtype, uint32_t cache_dtype, float k_scale,
                                float v_scale, mrs_stream_t stream);
void gather_kv_cache(void *key_cache, void *value_cache, void *k_out, void *v_out, const float *k_scale,
                     const float *v_scale, const int32_t *block_table, const int32_t *cu_seq_lens, int32_t num_tokens,
                     int32_t num_seqs, int32_t block_size, int32_t block_table_stride, int32_t num_kv_heads,
                     int32_t head_size, int32_t x, mrs_stream_t stream, uint32_t out_dtype, uint32_t cache_dtype);

/* REF ffi.rs:269-438 / pagedattention.cuh:687-876 */
#define MRS_PAGED_DECL(t)                                                                                          \
  void paged_attention_v1_##t(void *out, void *query, void *key_cache, void *value_cache, void *alibi_slopes,      \
                              int32_t num_kv_heads, float scale, float softcapping, uint32_t *block_tables,        \
                              uint32_t *context_lens, int32_t block_size, int32_t max_context_len, int32_t num_seqs, \
                              int32_t num_heads, int32_t head_size, int32_t max_num_blocks_per_seq, int32_t q_stride, \
                              int32_t kv_block_stride, int32_t kv_head_stride, mrs_stream_t stream,                \
                              uint32_t cache_dtype, float *k_scale, float *v_scale, const float *sinks);           \
  void paged_attention_v2_##t(void *out, float *exp_sums, float *max_logits, void *tmp_out, void *query,           \
                              void *key_cache, void *value_cache, void *alibi_slopes, int32_t num_kv_heads,        \
                              float scale, float softcapping, uint32_t *block_tables, uint32_t *context_lens,      \
                              int32_t block_size, int32_t max_context_len, int32_t num_seqs, int32_t num_heads,    \
                              int32_t head_size, int32_t max_num_blocks_per_seq, int32_t q_stride,                 \
                              int32_t kv_block_stride, int32_t kv_head_stride, mrs_stream_t stream,                \
                              uint32_t cache_dtype, float *k_scale, float *v_scale, const float *sinks);
MRS_PAGED_DECL(f16) MRS_PAGED_DECL(bf16) MRS_PAGED_DECL(f32)

/* REF ffi.rs:440-482 / copy_blocks_kernel.cu */
#define MRS_COPY_DECL(t)                                                                                     \
  void copy_blocks_##t(int64_t *key_cache_ptrs, int64_t *value_cache_ptrs, const int64_t *block_mapping,     \
                       int32_t num_layers, int32_t num_pairs, int32_t numel_per_block_key,                   \
                       int32_t numel_per_block_value, int64_t stream);
MRS_COPY_DECL(f32) MRS_COPY_DECL(f16) MRS_COPY_DECL(bf16) MRS_COPY_DECL(u8)

/* REF ffi.rs:484-509 / update_kvscales.cu: *k_scales = max(*k_scales, absmax(k) / 240), same for v
 * (FP8 KV-cache scale tracking; one f32 scalar each, updated atomically). */
void update_kv_scales_f32(void *k, void *v, const long num_elements, float *k_scales, float *v_scales, int64_t stream);
void update_kv_scales_f16(void *k, void *v, const long num_elements, float *k_scales, float *v_scales, int64_t stream);
void update_kv_scales_bf16(void *k, void *v, const long num_elements, float *k_scales, float *v_scales, int64_t stream);

/* REF backend/cache.rs:194-300 (`swap_blocks`, Rust-side memcpy loop in the reference): copy cache
 * blocks src[src_block] -> dst[dst_block] for every pair; src/dst may each be device or (pinned) host
 * memory of the same block geometry.  pairs: HOST array [n_pairs][2].  Asynchronous on `stream`;
 * returns a cudaError_t. */
int32_t mrs_swap_blocks(const void *src, void *dst, int64_t block_bytes, const int64_t *pairs, int64_t n_pairs,
                        void *stream);

/* ---- native addition: RoPE + KV write + decode attention + split-KV merge in one launch
 * over the HND cache (replaces rotary_embedding_positions + reshape_and_cache_flashinfer +
 * flashinfer_decode + its merge kernel); see csrc/paged_attn.cu.  `pdl`: bit 0 = the launch uses
 * programmatic stream serialisation, bit 1 = interleaved (GPT-J / GGUF llama) RoPE pairing instead
 * of rotate-half. */
int32_t mrs_paged_decode_fused(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                               const void *rope_cos, const void *rope_sin, const int32_t *positions,
                               const int64_t *slot_mapping, const int32_t *kv_indptr, const int32_t *kv_indices,
                               const int32_t *kv_last_page_len, const int32_t *request_indices,
                               const int32_t *kv_tile_indices, const int32_t *o_indptr,
                               const int32_t *kv_chunk_size_ptr, const uint8_t *block_valid_mask, void *o, void *tmp_v,
                               float *tmp_s, int32_t *counters, int32_t batch_size, int32_t padded_batch_size,
                               int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size, int32_t page_size,
                               float sm_scale, uint32_t dtype, int32_t pdl, void *stream);
/* same with explicit row strides (elements) of q and of k_new / v_new: a fused QKV GEMM writes
 * [B, (H + 2 KVH) D] and hands three pointers into it */
int32_t mrs_paged_decode_fused_strided(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                               const void *rope_cos, const void *rope_sin, const int32_t *positions,
                               const int64_t *slot_mapping, const int32_t *kv_indptr, const int32_t *kv_indices,
                               const int32_t *kv_last_page_len, const int32_t *request_indices,
                               const int32_t *kv_tile_indices, const int32_t *o_indptr,
                               const int32_t *kv_chunk_size_ptr, const uint8_t *block_valid_mask, void *o, void *tmp_v,
                               float *tmp_s, int32_t *counters, int32_t batch_size, int32_t padded_batch_size,
                               int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size, int32_t page_size,
                               float sm_scale, uint32_t dtype, int32_t pdl, int64_t q_stride_n, int64_t kv_new_stride,
                               void *stream);
/* Multi-query form (speculative verify): every sequence brings q_len rows (1..8) at positions kv_len - q_len ..
 * kv_len - 1, where kv_len (from the CSR) already counts them.  q / k_new / v_new / o / positions / slot_mapping hold
 * [batch_size * q_len] rows, sequence-major; q and o are contiguous [*, num_qo_heads * head_size], k_new / v_new
 * [*, num_kv_heads * head_size].  Query row i attends to every cached row below kv_len - q_len and to new rows 0..i
 * (causal); the new rows are rotated, attended from shared memory and written to their slots (slot < 0: not
 * written).  No cached row at or past kv_len - q_len is read.  tmp_v / tmp_s: [padded_batch_size, q_len *
 * num_qo_heads] partials; counters: zeroed int32 [batch_size * num_kv_heads * ceil(group * q_len / 16)], left zero.
 * Head size 64 | 128, dtype 0 f16 / 1 bf16, no window / soft-cap.  At q_len = 1 the result equals
 * mrs_paged_decode_fused bit for bit.  Returns a cudaError_t. */
int32_t mrs_paged_decode_fused_multi(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                               const void *rope_cos, const void *rope_sin, const int32_t *positions,
                               const int64_t *slot_mapping, const int32_t *kv_indptr, const int32_t *kv_indices,
                               const int32_t *kv_last_page_len, const int32_t *request_indices,
                               const int32_t *kv_tile_indices, const int32_t *o_indptr,
                               const int32_t *kv_chunk_size_ptr, const uint8_t *block_valid_mask, void *o, void *tmp_v,
                               float *tmp_s, int32_t *counters, int32_t batch_size, int32_t padded_batch_size,
                               int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size, int32_t page_size,
                               float sm_scale, uint32_t dtype, int32_t pdl, int32_t q_len, void *stream);
/* same with explicit row strides (elements) of q and of k_new / v_new, as mrs_paged_decode_fused_strided: a fused QKV
 * GEMM writes [batch_size * q_len, (H + 2 KVH) D] and hands three pointers into it; o stays contiguous.  With the
 * contiguous strides it is mrs_paged_decode_fused_multi. */
int32_t mrs_paged_decode_fused_multi_strided(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                               const void *rope_cos, const void *rope_sin, const int32_t *positions,
                               const int64_t *slot_mapping, const int32_t *kv_indptr, const int32_t *kv_indices,
                               const int32_t *kv_last_page_len, const int32_t *request_indices,
                               const int32_t *kv_tile_indices, const int32_t *o_indptr,
                               const int32_t *kv_chunk_size_ptr, const uint8_t *block_valid_mask, void *o, void *tmp_v,
                               float *tmp_s, int32_t *counters, int32_t batch_size, int32_t padded_batch_size,
                               int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size, int32_t page_size,
                               float sm_scale, uint32_t dtype, int32_t pdl, int32_t q_len, int64_t q_stride_n,
                               int64_t kv_new_stride, void *stream);
/* ---- prompt attention over fresh q/k/v (SURVEY §8(f) rank 1; REF paged_attention.rs:1413-1475 ->
 * flash_attn_varlen): causal [+ sliding window / soft-cap], GQA, var-len batches via cu_seqlens
 * (device i32 [batch+1], or NULL for one sequence).  q [total,H,D], k/v [total,KVH,D], strides in
 * elements between tokens; head_dim 64 | 128; dtype 0 f16 / 1 bf16.  csrc/prefill_attn.cu. */
int32_t mrs_prefill_attention(const void *q, const void *k, const void *v, void *out, const int32_t *cu_seqlens,
                              int32_t batch, int32_t total_tokens, int32_t max_seqlen, int32_t num_heads,
                              int32_t num_kv_heads, int32_t head_dim, int64_t q_stride, int64_t kv_stride, int64_t o_stride,
                              float softmax_scale, int32_t causal, int32_t window_left, float softcap, uint32_t dtype,
                              void *stream);
/* ---- prompt attention of new query tokens over K/V already in the HND page cache: prefix-cache hits and chunked
 * prompts (REF paged_attention.rs:973-1200 `try_prefix_gather_prefill`, plan FlashAttentionPaged ->
 * flash_attn_varlen_paged_windowed, mistralrs-flash-attn/src/flash.rs:979-1010).
 *   Shapes     q [total_q, H, D] with token stride q_stride (elements), out [total_q, H, D] with o_stride; key_cache /
 *              value_cache HND [num_blocks, KVH, page_size, D] in q's 16-bit dtype (0 f16 / 1 bf16).
 *   Sequences  sequence b owns query rows cu_seqlens_q[b] .. cu_seqlens_q[b+1] and kv_len = cu_seqlens_k[b+1] -
 *              cu_seqlens_k[b] keys (both cumulative, device i32 [batch + 1]); key j sits at slot
 *              block_table[b * block_table_stride + j / page_size] * page_size + j % page_size.
 *   Positions  query i of sequence b is at absolute position kv_len - q_len + i: causal masking is aligned bottom-right;
 *              window_left >= 0 keeps keys j >= pos - window_left; causal = 0 sees all kv_len keys.  softcap <= 0: off.
 *   Ordering   the new tokens' K/V are already in the cache (the caller scatters them first); kv_len >= q_len.
 *   Table      entries at or past ceil(kv_len / page_size) are never read (rows may be padded with anything); cache
 *              rows past kv_len, including stale rows of the last page, contribute exactly zero.
 *   Support    head_dim 64 | 128, page_size 8 | 16 | 32, GQA, var-len batches; no FP8 cache, ALiBi or sinks.
 *   Errors     returns a cudaError_t; stream-ordered, no allocation, no synchronisation (graph-capturable).
 * Head 128 without window / softcap runs on the wgmma kernel (mrs_prefill_attention_paged_tc, cudaErrorNotSupported
 * when the call does not fit), everything else on the mma.sync one; mrs_prefill_attn_tc_debug(0, ...) applies here too. */
int32_t mrs_prefill_attention_paged(const void *q, const void *key_cache, const void *value_cache, void *out,
                                    const int32_t *block_table, int32_t block_table_stride, const int32_t *cu_seqlens_q,
                                    const int32_t *cu_seqlens_k, int32_t batch, int32_t total_q, int32_t max_seqlen_q,
                                    int32_t max_seqlen_k, int32_t num_blocks, int32_t num_heads, int32_t num_kv_heads,
                                    int32_t head_dim, int32_t page_size, int64_t q_stride, int64_t o_stride,
                                    float softmax_scale, int32_t causal, int32_t window_left, float softcap, uint32_t dtype,
                                    void *stream);
int32_t mrs_prefill_attention_paged_tc(const void *q, const void *key_cache, const void *value_cache, void *out,
                                       const int32_t *block_table, int32_t block_table_stride, const int32_t *cu_seqlens_q,
                                       const int32_t *cu_seqlens_k, int32_t batch, int32_t total_q, int32_t max_seqlen_q,
                                       int32_t max_seqlen_k, int32_t num_blocks, int32_t num_heads, int32_t num_kv_heads,
                                       int32_t head_dim, int32_t page_size, int64_t q_stride, int64_t o_stride,
                                       float softmax_scale, int32_t causal, int32_t window_left, float softcap,
                                       uint32_t dtype, void *stream);
/* mrs_prefill_attention picks between csrc/prefill_attn_tc.cu (wgmma: S and P in registers, V as an MN-major
 * shared-memory operand; head size 128, no window / softcap) and csrc/prefill_attn.cu (mma.sync; everything else).
 * mrs_prefill_attention_tc is the first kernel's own entry: cudaErrorNotSupported (801) when the call does not fit.
 * mrs_prefill_attn_tc_debug(enable, lbo, sbo): enable 0 keeps every call on prefill_attn.cu (A/B, tests); lbo / sbo
 * (bytes, 0 = keep) override the V operand's descriptor strides (bring-up knob). */
int32_t mrs_prefill_attention_tc(const void *q, const void *k, const void *v, void *out, const int32_t *cu_seqlens,
                              int32_t batch, int32_t total_tokens, int32_t max_seqlen, int32_t num_heads,
                              int32_t num_kv_heads, int32_t head_dim, int64_t q_stride, int64_t kv_stride, int64_t o_stride,
                              float softmax_scale, int32_t causal, int32_t window_left, float softcap, uint32_t dtype,
                              void *stream);
void mrs_prefill_attn_tc_debug(int32_t enable, uint32_t lbo, uint32_t sbo);
/* diagnostics: bit 0 keeps HND decode attention on the SIMT kernel instead of the tensor-core one;
 * bit 1 disables the cluster/DSMEM merge of split-KV tiles (global partials + counter instead) */
void mrs_set_attn_flags(int32_t flags);
#ifdef __cplusplus
}
#endif
#endif
