/* mrs_b200_host.h — C ABI of libmrs_b200_host.so: the host-side (no CUDA) pieces either side of the
 * hot path.  Plain pointers and sizes only.
 *
 *  - KV index producers: block pool, slot mapping, paged-KV CSR and split-KV tile plans — integers
 *    that must match the reference bit for bit.
 *      REF mistralrs-core/src/paged_attention/block_pool.rs:290-442 (BlockPool),
 *          mistralrs-core/src/pipeline/inputs_processor.rs:896-923 (slots),
 *          mistralrs-core/src/flashinfer/metadata.rs:61-216 (split size, CSR, tiles)
 *  - GGUF archives: header / metadata / tensor catalogue / split shards over mmap; tensor payloads
 *    are handed out as pointers into the mapping for a straight host->device copy.
 *      REF mistralrs-quant/src/gguf/archive.rs:351-611 (GgufArchive)
 */
#ifndef MRS_B200_HOST_H
#define MRS_B200_HOST_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- block pool (block 0 is the null block; FIFO free list) ---- */
void *mrs_block_pool_new(int64_t num_gpu_blocks);
void mrs_block_pool_free(void *pool);
int64_t mrs_block_pool_null_block_id(void *pool);
int64_t mrs_block_pool_num_free_blocks(void *pool);
int64_t mrs_block_pool_ref_cnt(void *pool, int64_t block_id);
int mrs_block_pool_get_new_blocks(void *pool, int64_t num, int64_t *out); /* 1 ok, 0 not enough free blocks */
void mrs_block_pool_free_blocks(void *pool, const int64_t *ids, int64_t n);
void mrs_block_pool_touch(void *pool, const int64_t *ids, int64_t n);

/* ---- prefix cache: full blocks are published under a chained 64-bit hash of their prefix; a freed block keeps its
 *      hashes until it is handed out again.  REF block_pool.rs:182-280,355-372,454-527; block_hash.rs:126-150,232-263;
 *      kv_cache_manager.rs:129-174.  Hash VALUES are this library's own (the reference's are Rust's SipHash and never
 *      leave its scheduler either); equal prefixes <=> equal hashes is the contract. ---- */
void *mrs_block_pool_new_cached(int64_t num_gpu_blocks, int32_t enable_caching, int64_t hash_block_size);
double mrs_block_pool_usage(void *pool);
int64_t mrs_block_pool_num_cached_blocks(void *pool);
int64_t mrs_block_pool_num_block_hashes(void *pool, int64_t block_id);
int mrs_block_pool_get_cached_block(void *pool, uint64_t hash, const uint32_t *groups, int64_t n_groups,
                                    int64_t *out); /* 1 hit in every group, 0 miss */
int mrs_block_pool_cache_full_blocks(void *pool, const int64_t *ids, int64_t n_ids, const uint64_t *hashes,
                                     int64_t n_hashes, int64_t num_cached, int64_t num_full, uint32_t group);
int mrs_block_pool_reset_prefix_cache(void *pool); /* 1 done, 0 refused: blocks still in use */
int64_t mrs_block_hashes(const uint32_t *tokens, int64_t n, int64_t block_size, const uint64_t *extra, int64_t n_extra,
                         const uint64_t *prev, int64_t n_prev, uint64_t *out);
int64_t mrs_block_pool_computed_blocks(void *pool, const uint64_t *hashes, int64_t n_hashes, int64_t num_tokens,
                                       int64_t block_size, const uint32_t *groups, int64_t n_groups, int64_t *out);

/* ---- per-request block tables over a pool: admission with prefix-cache hits, growth, trim, release, publishing,
 *      slot mapping and padded block tables.  REF mistralrs-core/src/paged_attention/kv_cache_manager.rs:62-435.
 *      Request ids are the caller's sequence ids. ---- */
void *mrs_kv_manager_new(int64_t num_gpu_blocks, int64_t block_size, int32_t enable_caching, const uint32_t *groups,
                         int64_t n_groups);
void mrs_kv_manager_free(void *mgr);
void *mrs_kv_manager_pool(void *mgr); /* borrowed mrs_block_pool handle; do not free */
int64_t mrs_kv_manager_num_free_blocks(void *mgr);
int64_t mrs_kv_manager_num_usable_blocks(void *mgr);
double mrs_kv_manager_usage(void *mgr);
int64_t mrs_kv_manager_get_computed_blocks(void *mgr, const uint64_t *hashes, int64_t n_hashes, int64_t num_tokens,
                                           int64_t *out);
int64_t mrs_kv_manager_allocate_slots(void *mgr, uint64_t request_id, int64_t num_tokens, const int64_t *computed,
                                      int64_t n_computed, int64_t *out); /* fresh ids written, or -1: pool exhausted */
void mrs_kv_manager_release(void *mgr, uint64_t request_id);
void mrs_kv_manager_trim(void *mgr, uint64_t request_id, int64_t num_tokens);
int mrs_kv_manager_cache_blocks(void *mgr, uint64_t request_id, const uint64_t *hashes, int64_t n_hashes,
                                int64_t num_computed_tokens);
int mrs_kv_manager_has_request(void *mgr, uint64_t request_id);
int64_t mrs_kv_manager_num_blocks(void *mgr, uint64_t request_id);
int64_t mrs_kv_manager_num_cached_blocks(void *mgr, uint64_t request_id);
int mrs_kv_manager_reset_prefix_cache(void *mgr);
int mrs_kv_manager_slot_mapping(void *mgr, uint64_t request_id, int64_t start_token, int64_t num_tokens, int64_t *out);
int mrs_kv_manager_block_table(void *mgr, uint64_t request_id, int64_t max_blocks, int32_t *out);
/* one decode step of a batch into staging arrays: tables [batch, max_blocks] i32, slots [batch] i64 (slot of the last
 * token); returns -1, or the index of the first request that is unknown or could not grow */
int64_t mrs_kv_manager_decode_step(void *mgr, const uint64_t *request_ids, const int64_t *context_lens, int64_t batch,
                                   int64_t max_blocks, int32_t *tables, int64_t *slots);

/* ---- f32 -> ggml blocks on the host, for in-situ re-quantisation of a GGUF layer (REF gguf/mod.rs:633-708 apply_isq;
 *      arithmetic = candle k_quants `from_float` / ggml `quantize_row_*_ref`).  Types 2,3,6,7,8 (Q4_0 Q4_1 Q5_0 Q5_1 Q8_0);
 *      K-quants have no quantiser here.  n % 32 == 0.  Returns bytes written or -1. ---- */
int64_t mrs_ggml_quantize(int32_t ggml_type, const float *x, int64_t n, uint8_t *out);
int32_t mrs_ggml_quantize_block_bytes(int32_t ggml_type); /* 0: no quantiser for this type */

/* ---- host tail of the on-device sampler: packed rows of topk_large_f32_packed[_batched] / top1_large_f32_packed
 *      (mrs_b200_ops.h) -> token + logprob.  REF mistralrs-core/src/sampler.rs:1172-1273,666-742,1284-1297.
 *      u is the caller's uniform variate in [0,1) (the random stream stays with the caller).
 *      0 ok, -1 bad row length / k, -2 bad softmax normaliser, -3 nothing survives the filters, -4 negative or
 *      non-finite probability, -5 invalid top-1 row ---- */
int mrs_sample_topk_packed_row(const float *packed, int64_t packed_len, int64_t packed_k, int64_t row_k,
                               float inv_temperature, float top_p, float min_p, double u, uint32_t *token,
                               float *logprob);
int64_t mrs_sample_topk_packed_batch(const float *packed, int64_t batch, int64_t packed_k, const int64_t *row_k,
                                     const float *inv_temperature, const float *top_p, const float *min_p,
                                     const double *u, uint32_t *tokens, float *logprobs, int32_t *status);
int mrs_sample_top1_row(const float *packed, uint32_t *token);

/* ---- slots / CSR / tile plans ---- */
int mrs_slot_mapping(const int64_t *table, int64_t table_len, int64_t block_size, int64_t start, int64_t end,
                     int64_t *out);
int mrs_make_paged_kv(const int64_t *tables, int64_t batch, int64_t max_blocks, const int64_t *context_lens,
                      int64_t block_size, int64_t padded_indices_len, int32_t *indptr, int32_t *indices,
                      int32_t *last_page_len);
int64_t mrs_decode_split_pages(int64_t block_size, int64_t batch, int64_t kv_heads, int64_t sm_count, int64_t max_ctx);
int64_t mrs_make_decode_tiles(const int64_t *table_lens, const int64_t *context_lens, int64_t batch, int64_t block_size,
                              int64_t split_pages, int64_t padded_tiles_len, int32_t *request_indices,
                              int32_t *kv_tile_indices, int32_t *o_indptr, int32_t *kv_chunk_size, uint8_t *mask);

/* ---- prompt chunk plan for text prompts (REF pipeline/prompt_chunks.rs, host/prompt_chunks.hpp) ----
 * mrs_prompt_chunk_size: max(1, budget / batch), each scheduled prompt's share of a step's token budget.
 * mrs_build_prompt_chunk_plan: rows [prefix_len, total_len) in chunks of at most chunk_size (>= 1); with block_align > 0
 *   a chunk that would end inside a block ends at that block's start when the chunk stays non-empty.  Writes the chunks
 *   as [start, end) pairs into out[2 * cap] when they fit; returns their count, -1 on a negative argument.
 * mrs_next_prompt_chunk_group: n sequences' plans as one CSR (chunks [total][2], plan_offsets [n + 1]) and the index of
 *   each one's next chunk (plan_indices [n]; past its plan when it has none left).  The first sequence with a chunk
 *   left sets finality (its plan's last chunk or not) and query length; every sequence with a chunk of the same
 *   finality (and, with require_uniform_query_len, the same length) is a member.  Writes the members in order to
 *   members[n] and finality to *is_final; returns the member count, 0 when no chunk is left, -1 on bad arguments. */
int64_t mrs_prompt_chunk_size(int64_t batch, int64_t budget);
int64_t mrs_build_prompt_chunk_plan(int64_t total_len, int64_t prefix_len, int64_t chunk_size, int64_t block_align,
                                    int64_t *out, int64_t cap);
int64_t mrs_next_prompt_chunk_group(const int64_t *plan_indices, const int64_t *plan_offsets, const int64_t *chunks,
                                    int64_t n, int32_t require_uniform_query_len, int64_t *members, int32_t *is_final);

/* ---- GGUF archives ---- */
/* paths: all shards of one model, any order (split.no decides).  NULL + message in err on failure. */
void *mrs_gguf_open(const char *const *paths, int32_t n_paths, char *err, int64_t err_cap);
void mrs_gguf_close(void *archive);
int64_t mrs_gguf_alignment(void *archive);
int64_t mrs_gguf_n_tensors(void *archive);
int64_t mrs_gguf_n_metadata(void *archive);
int64_t mrs_gguf_find_tensor(void *archive, const char *name); /* index or -1 */
/* dims: up to 8 entries, ggml order (dims[0] innermost); offset is absolute inside shard `shard`;
 * nbytes = -1 when the ggml type's block size is unknown.  Returns the name length, -1 on a bad index. */
int32_t mrs_gguf_tensor_info(void *archive, int64_t i, char *name, int64_t name_cap, int32_t *ggml_type, int32_t *n_dims,
                             int64_t *dims, int32_t *shard, int64_t *offset, int64_t *nbytes);
const void *mrs_gguf_tensor_data(void *archive, int64_t i); /* pointer into the mapping, valid until close */
/* metadata: value types as in the GGUF spec (0 u8 .. 8 string, 9 array, 10 u64, 11 i64, 12 f64) */
int32_t mrs_gguf_meta_key(void *archive, int64_t i, char *key, int64_t cap, int32_t *vtype, int32_t *arr_type,
                          int64_t *arr_len);
int32_t mrs_gguf_meta_int(void *archive, const char *key, int64_t *out);   /* 1 found, 0 absent / not an integer */
int32_t mrs_gguf_meta_float(void *archive, const char *key, double *out);
int64_t mrs_gguf_meta_str(void *archive, const char *key, char *buf, int64_t cap); /* length, -1 absent */
int64_t mrs_gguf_meta_arr_str(void *archive, const char *key, int64_t idx, char *buf, int64_t cap);
int64_t mrs_gguf_meta_arr_num(void *archive, const char *key, int64_t start, int64_t cap, double *out, int64_t *out_int);

/* ---- safetensors containers (UQFF shards, residual.safetensors) ----
 * REF docs/src/content/docs/reference/uqff-format.md, mistralrs-quant/src/uqff/reader.rs: a UQFF shard
 * is a safetensors file whose entries follow naming conventions (see mistral.rs_b200/uqff_file.py). */
void *mrs_st_open(const char *path, char *err, int64_t err_cap); /* NULL + message on failure */
void mrs_st_close(void *file);
int64_t mrs_st_n_tensors(void *file);
int64_t mrs_st_find(void *file, const char *name); /* index or -1 */
/* dtype: safetensors dtype string into a >= 16-byte buffer; dims: up to 8 entries, row-major */
int32_t mrs_st_tensor_info(void *file, int64_t i, char *name, int64_t name_cap, char *dtype, int32_t *n_dims,
                           int64_t *dims, int64_t *offset, int64_t *nbytes);
const void *mrs_st_tensor_data(void *file, int64_t i);
int64_t mrs_st_n_metadata(void *file);
int64_t mrs_st_metadata(void *file, int64_t i, char *key, int64_t key_cap, char *val, int64_t val_cap);

#ifdef __cplusplus
}
#endif
#endif
