// host_api.cpp — C API over the C++ host layer (kv_index.hpp) for the Python test/bench harness.
#include "ggml_quantize.hpp"
#include "gguf_reader.hpp"
#include "kv_cache_manager.hpp"
#include "kv_index.hpp"
#include "prompt_chunks.hpp"
#include "safetensors_reader.hpp"
#include "sampler_tail.hpp"

#include <cstring>

using namespace mrs;

extern "C" {

void *mrs_block_pool_new(int64_t num_gpu_blocks) {
  try { return new BlockPool((size_t)num_gpu_blocks); } catch (...) { return nullptr; }
}
void mrs_block_pool_free(void *p) { delete (BlockPool *)p; }
int64_t mrs_block_pool_null_block_id(void *p) { return (int64_t)((BlockPool *)p)->null_block_id(); }
int64_t mrs_block_pool_num_free_blocks(void *p) { return (int64_t)((BlockPool *)p)->num_free_blocks(); }
int64_t mrs_block_pool_ref_cnt(void *p, int64_t id) { return (int64_t)((BlockPool *)p)->block_ref_cnt((size_t)id); }
// returns 1 and fills out[num] on success, 0 when not enough blocks are free
int mrs_block_pool_get_new_blocks(void *p, int64_t num, int64_t *out) {
  std::vector<size_t> v;
  if (!((BlockPool *)p)->get_new_blocks((size_t)num, v)) return 0;
  for (size_t i = 0; i < v.size(); i++) out[i] = (int64_t)v[i];
  return 1;
}
void mrs_block_pool_free_blocks(void *p, const int64_t *ids, int64_t n) {
  std::vector<size_t> v(ids, ids + n);
  ((BlockPool *)p)->free_blocks(v);
}
void mrs_block_pool_touch(void *p, const int64_t *ids, int64_t n) {
  std::vector<size_t> v(ids, ids + n);
  ((BlockPool *)p)->touch(v);
}

// ---- prefix cache ----
void *mrs_block_pool_new_cached(int64_t num_gpu_blocks, int32_t enable_caching, int64_t hash_block_size) {
  try { return new BlockPool((size_t)num_gpu_blocks, enable_caching != 0, (size_t)hash_block_size); } catch (...) { return nullptr; }
}
double mrs_block_pool_usage(void *p) { return ((BlockPool *)p)->usage(); }
int64_t mrs_block_pool_num_cached_blocks(void *p) { return (int64_t)((BlockPool *)p)->num_cached_blocks(); }
int64_t mrs_block_pool_num_block_hashes(void *p, int64_t id) { return (int64_t)((BlockPool *)p)->num_block_hashes((size_t)id); }
// 1 and out[n_groups] when every group holds a block under this hash, else 0
int mrs_block_pool_get_cached_block(void *p, uint64_t hash, const uint32_t *groups, int64_t n_groups, int64_t *out) {
  std::vector<uint32_t> g(groups, groups + n_groups);
  std::vector<size_t> v;
  if (!((BlockPool *)p)->get_cached_block(hash, g, v)) return 0;
  for (size_t i = 0; i < v.size(); i++) out[i] = (int64_t)v[i];
  return 1;
}
// 0 ok, -1 fewer ids / hashes than num_full
int mrs_block_pool_cache_full_blocks(void *p, const int64_t *ids, int64_t n_ids, const uint64_t *hashes, int64_t n_hashes,
                                     int64_t num_cached, int64_t num_full, uint32_t group) {
  try {
    std::vector<size_t> v(ids, ids + n_ids);
    std::vector<uint64_t> h(hashes, hashes + n_hashes);
    ((BlockPool *)p)->cache_full_blocks(v, h, (size_t)num_cached, (size_t)num_full, group);
    return 0;
  } catch (...) { return -1; }
}
int mrs_block_pool_reset_prefix_cache(void *p) { return ((BlockPool *)p)->reset_prefix_cache() ? 1 : 0; }
// chained hashes of the full blocks of tokens[n]; `prev` (n_prev of them) are reused, only the rest are computed.
// Returns the number of full blocks; out holds that many.
int64_t mrs_block_hashes(const uint32_t *tokens, int64_t n, int64_t block_size, const uint64_t *extra, int64_t n_extra,
                         const uint64_t *prev, int64_t n_prev, uint64_t *out) {
  if (block_size <= 0) return -1;
  const int64_t full = n / block_size;
  if (n_prev > full) n_prev = full;
  for (int64_t i = 0; i < n_prev; i++) out[i] = prev[i];
  for (int64_t i = n_prev; i < full; i++)
    out[i] = hash_block_tokens(i > 0, i > 0 ? out[i - 1] : 0, tokens + i * block_size, (size_t)block_size, extra, (size_t)n_extra);
  return full;
}
// longest cached prefix of a request: walks the hashes until a miss, never covering the last token; returns the
// number of blocks written to out.  REF kv_cache_manager.rs:129-174
int64_t mrs_block_pool_computed_blocks(void *p, const uint64_t *hashes, int64_t n_hashes, int64_t num_tokens, int64_t block_size,
                                       const uint32_t *groups, int64_t n_groups, int64_t *out) {
  BlockPool *bp = (BlockPool *)p;
  if (!bp->caching_enabled() || block_size <= 0) return 0;
  const int64_t cap = (num_tokens > 0 ? num_tokens - 1 : 0) / block_size;
  std::vector<uint32_t> g(groups, groups + n_groups);
  std::vector<size_t> v;
  int64_t k = 0;
  for (; k < n_hashes && k < cap; k++) {
    if (!bp->get_cached_block(hashes[k], g, v) || v.empty()) break;
    bool same = true;
    for (size_t id : v) same &= (id == v[0]);
    if (!same) break;
    out[k] = (int64_t)v[0];
  }
  return k;
}

// ---- f32 -> ggml blocks (ggml_quantize.hpp): Q4_0 / Q4_1 / Q5_0 / Q5_1 / Q8_0 ----
int64_t mrs_ggml_quantize(int32_t ggml_type, const float *x, int64_t n, uint8_t *out) { return quantize_row(ggml_type, x, n, out); }
int32_t mrs_ggml_quantize_block_bytes(int32_t ggml_type) { return quantize_block_bytes(ggml_type); }

// ---- host tail of the on-device sampler (sampler_tail.hpp) ----
int mrs_sample_topk_packed_row(const float *packed, int64_t packed_len, int64_t packed_k, int64_t row_k, float inv_temperature, float top_p,
                               float min_p, double u, uint32_t *token, float *logprob) {
  return sample_topk_packed_row(packed, packed_len, packed_k, row_k, inv_temperature, top_p, min_p, u, token, logprob);
}
// rows [batch, 2*packed_k+2]; per-row k / temperature / filters / variate; status[batch] gets each row's code.
// Returns the number of rows that failed.
int64_t mrs_sample_topk_packed_batch(const float *packed, int64_t batch, int64_t packed_k, const int64_t *row_k, const float *inv_temperature,
                                     const float *top_p, const float *min_p, const double *u, uint32_t *tokens, float *logprobs,
                                     int32_t *status) {
  int64_t bad = 0;
  const int64_t w = 2 * packed_k + 2;
  for (int64_t b = 0; b < batch; b++) {
    const int rc = sample_topk_packed_row(packed + b * w, w, packed_k, row_k[b], inv_temperature[b], top_p[b], min_p[b], u[b], tokens + b,
                                          logprobs + b);
    if (status) status[b] = rc;
    bad += (rc != 0);
  }
  return bad;
}
int mrs_sample_top1_row(const float *packed, uint32_t *token) { return sample_top1_row(packed, token); }

// ---- per-request block tables over a pool (kv_cache_manager.hpp) ----
void *mrs_kv_manager_new(int64_t num_gpu_blocks, int64_t block_size, int32_t enable_caching, const uint32_t *groups, int64_t n_groups) {
  try {
    return new KvCacheManager((size_t)num_gpu_blocks, (size_t)block_size, enable_caching != 0, std::vector<uint32_t>(groups, groups + n_groups));
  } catch (...) { return nullptr; }
}
void mrs_kv_manager_free(void *m) { delete (KvCacheManager *)m; }
void *mrs_kv_manager_pool(void *m) { return &((KvCacheManager *)m)->pool(); }   // borrowed: valid while the manager lives
int64_t mrs_kv_manager_num_free_blocks(void *m) { return (int64_t)((KvCacheManager *)m)->pool().num_free_blocks(); }
int64_t mrs_kv_manager_num_usable_blocks(void *m) { return (int64_t)((KvCacheManager *)m)->num_usable_blocks(); }
double mrs_kv_manager_usage(void *m) { return ((KvCacheManager *)m)->pool().usage(); }
// number of cached leading blocks written to out (room for n_hashes)
int64_t mrs_kv_manager_get_computed_blocks(void *m, const uint64_t *hashes, int64_t n_hashes, int64_t num_tokens, int64_t *out) {
  std::vector<size_t> v;
  ((KvCacheManager *)m)->computed_blocks(hashes, (size_t)n_hashes, (size_t)num_tokens, v);
  for (size_t i = 0; i < v.size(); i++) out[i] = (int64_t)v[i];
  return (int64_t)v.size();
}
// >= 0: number of fresh block ids written to out (room for ceil(num_tokens / block_size)); -1: not enough free blocks
int64_t mrs_kv_manager_allocate_slots(void *m, uint64_t req, int64_t num_tokens, const int64_t *computed, int64_t n_computed, int64_t *out) {
  std::vector<size_t> c(computed, computed + n_computed), fresh;
  if (!((KvCacheManager *)m)->allocate_slots(req, (size_t)num_tokens, c, fresh)) return -1;
  for (size_t i = 0; i < fresh.size(); i++) out[i] = (int64_t)fresh[i];
  return (int64_t)fresh.size();
}
void mrs_kv_manager_release(void *m, uint64_t req) { ((KvCacheManager *)m)->free(req); }
void mrs_kv_manager_trim(void *m, uint64_t req, int64_t num_tokens) { ((KvCacheManager *)m)->trim(req, (size_t)num_tokens); }
int mrs_kv_manager_cache_blocks(void *m, uint64_t req, const uint64_t *hashes, int64_t n_hashes, int64_t num_computed_tokens) {
  try { ((KvCacheManager *)m)->cache_blocks(req, hashes, (size_t)n_hashes, (size_t)num_computed_tokens); return 0; } catch (...) { return -1; }
}
int mrs_kv_manager_has_request(void *m, uint64_t req) { return ((KvCacheManager *)m)->has(req) ? 1 : 0; }
int64_t mrs_kv_manager_num_blocks(void *m, uint64_t req) {
  const std::vector<size_t> *v = ((KvCacheManager *)m)->block_ids(req);
  return v ? (int64_t)v->size() : 0;
}
int64_t mrs_kv_manager_num_cached_blocks(void *m, uint64_t req) { return (int64_t)((KvCacheManager *)m)->num_cached_blocks(req); }
int mrs_kv_manager_reset_prefix_cache(void *m) { return ((KvCacheManager *)m)->pool().reset_prefix_cache() ? 1 : 0; }
// 0 ok, -1 unknown request
int mrs_kv_manager_slot_mapping(void *m, uint64_t req, int64_t start_token, int64_t num_tokens, int64_t *out) {
  return ((KvCacheManager *)m)->slot_mapping(req, (size_t)start_token, (size_t)num_tokens, out) ? 0 : -1;
}
int mrs_kv_manager_block_table(void *m, uint64_t req, int64_t max_blocks, int32_t *out) {
  return ((KvCacheManager *)m)->block_table(req, (size_t)max_blocks, out) ? 0 : -1;
}
int64_t mrs_kv_manager_decode_step(void *m, const uint64_t *req_ids, const int64_t *context_lens, int64_t batch, int64_t max_blocks,
                                   int32_t *tables, int64_t *slots) {
  return ((KvCacheManager *)m)->decode_step(req_ids, context_lens, (size_t)batch, (size_t)max_blocks, tables, slots);
}

// slot mapping for tokens [start, end) of one sequence; returns 0 ok, -1 table too small
int mrs_slot_mapping(const int64_t *table, int64_t table_len, int64_t block_size, int64_t start, int64_t end, int64_t *out) {
  try {
    std::vector<size_t> t(table, table + table_len);
    auto s = slot_mapping(t, (size_t)block_size, (size_t)start, (size_t)end);
    std::memcpy(out, s.data(), s.size() * sizeof(int64_t));
    return 0;
  } catch (...) { return -1; }
}

// CSR builder over a dense [batch, max_blocks] table (row b uses its first ceil(ctx/bs) entries)
int mrs_make_paged_kv(const int64_t *tables, int64_t batch, int64_t max_blocks, const int64_t *context_lens,
                      int64_t block_size, int64_t padded_indices_len, int32_t *indptr, int32_t *indices,
                      int32_t *last_page_len) {
  try {
    std::vector<std::vector<size_t>> t(batch);
    std::vector<size_t> cl(context_lens, context_lens + batch);
    for (int64_t b = 0; b < batch; b++) t[b].assign(tables + b * max_blocks, tables + (b + 1) * max_blocks);
    auto r = make_paged_kv(t, cl, (size_t)block_size, (size_t)padded_indices_len);
    std::memcpy(indptr, r.indptr.data(), r.indptr.size() * 4);
    std::memcpy(indices, r.indices.data(), r.indices.size() * 4);
    std::memcpy(last_page_len, r.last_page_len.data(), r.last_page_len.size() * 4);
    return 0;
  } catch (...) { return -1; }
}

int64_t mrs_decode_split_pages(int64_t block_size, int64_t batch, int64_t kv_heads, int64_t sm_count, int64_t max_ctx) {
  return (int64_t)decode_split_pages((size_t)block_size, (size_t)batch, (size_t)kv_heads, (size_t)sm_count, (size_t)max_ctx);
}

// returns number of valid tiles, or -1 on error
int64_t mrs_prompt_chunk_size(int64_t batch, int64_t budget) {
  if (batch < 0 || budget < 0) return -1;
  return (int64_t)prompt_chunk_size((size_t)batch, (size_t)budget);
}

int64_t mrs_build_prompt_chunk_plan(int64_t total_len, int64_t prefix_len, int64_t chunk_size, int64_t block_align,
                                    int64_t *out, int64_t cap) {
  if (total_len < 0 || prefix_len < 0 || chunk_size < 1 || block_align < 0 || cap < 0) return -1;
  const auto plan = build_prompt_chunk_plan((size_t)total_len, (size_t)prefix_len, (size_t)chunk_size, (size_t)block_align);
  if ((int64_t)plan.size() <= cap && out != nullptr)
    for (size_t i = 0; i < plan.size(); i++) { out[2 * i] = (int64_t)plan[i].start; out[2 * i + 1] = (int64_t)plan[i].end; }
  return (int64_t)plan.size();
}

int64_t mrs_next_prompt_chunk_group(const int64_t *plan_indices, const int64_t *plan_offsets, const int64_t *chunks,
                                    int64_t n, int32_t require_uniform_query_len, int64_t *members, int32_t *is_final) {
  if (n < 0 || (n > 0 && (plan_indices == nullptr || plan_offsets == nullptr || members == nullptr)) || is_final == nullptr)
    return -1;
  std::vector<size_t> idx((size_t)n);
  std::vector<std::vector<PromptChunk>> plans((size_t)n);
  for (int64_t i = 0; i < n; i++) {
    if (plan_indices[i] < 0 || plan_offsets[i + 1] < plan_offsets[i] || (plan_offsets[i + 1] > plan_offsets[i] && chunks == nullptr))
      return -1;
    idx[(size_t)i] = (size_t)plan_indices[i];
    for (int64_t c = plan_offsets[i]; c < plan_offsets[i + 1]; c++)
      plans[(size_t)i].push_back({(size_t)chunks[2 * c], (size_t)chunks[2 * c + 1]});
  }
  std::vector<size_t> m;
  bool fin = false;
  if (!next_prompt_chunk_group(idx, plans, require_uniform_query_len != 0, m, fin)) { *is_final = 0; return 0; }
  for (size_t i = 0; i < m.size(); i++) members[i] = (int64_t)m[i];
  *is_final = fin ? 1 : 0;
  return (int64_t)m.size();
}

int64_t mrs_make_decode_tiles(const int64_t *table_lens, const int64_t *context_lens, int64_t batch, int64_t block_size,
                              int64_t split_pages, int64_t padded_tiles_len, int32_t *request_indices,
                              int32_t *kv_tile_indices, int32_t *o_indptr, int32_t *kv_chunk_size, uint8_t *mask) {
  try {
    std::vector<size_t> tl(table_lens, table_lens + batch), cl(context_lens, context_lens + batch);
    auto r = make_decode_tiles(tl, cl, (size_t)block_size, (size_t)split_pages, (size_t)padded_tiles_len);
    std::memcpy(request_indices, r.request_indices.data(), r.request_indices.size() * 4);
    std::memcpy(kv_tile_indices, r.kv_tile_indices.data(), r.kv_tile_indices.size() * 4);
    std::memcpy(o_indptr, r.o_indptr.data(), r.o_indptr.size() * 4);
    std::memcpy(mask, r.block_valid_mask.data(), r.block_valid_mask.size());
    *kv_chunk_size = r.kv_chunk_size;
    return (int64_t)r.o_indptr.back();
  } catch (...) { return -1; }
}


// ---------------------------------------------------------------- GGUF archives (gguf_reader.hpp)
static int copy_out(const std::string &v, char *buf, int64_t cap) {
  if (buf != nullptr && cap > 0) {
    const size_t n = v.size() < (size_t)cap - 1 ? v.size() : (size_t)cap - 1;
    memcpy(buf, v.data(), n);
    buf[n] = 0;
  }
  return (int)v.size();
}

// paths: n_paths shard files (any order; split.no decides).  NULL + message in err on failure.
void *mrs_gguf_open(const char *const *paths, int32_t n_paths, char *err, int64_t err_cap) {
  try {
    std::vector<std::string> v;
    for (int i = 0; i < n_paths; i++) v.emplace_back(paths[i]);
    return new GgufArchive(v);
  } catch (const std::exception &e) {
    copy_out(e.what(), err, err_cap);
    return nullptr;
  }
}
void mrs_gguf_close(void *h) { delete (GgufArchive *)h; }
int64_t mrs_gguf_alignment(void *h) { return (int64_t)((GgufArchive *)h)->alignment(); }
int64_t mrs_gguf_n_tensors(void *h) { return (int64_t)((GgufArchive *)h)->tensors().size(); }
int64_t mrs_gguf_n_metadata(void *h) { return (int64_t)((GgufArchive *)h)->metadata_keys().size(); }
int64_t mrs_gguf_find_tensor(void *h, const char *name) { return ((GgufArchive *)h)->find_tensor(name); }

// dims: up to 8 entries in ggml order (dims[0] innermost).  Returns the name length, -1 on a bad index.
int32_t mrs_gguf_tensor_info(void *h, int64_t i, char *name, int64_t name_cap, int32_t *ggml_type, int32_t *n_dims,
                             int64_t *dims, int32_t *shard, int64_t *offset, int64_t *nbytes) {
  const auto &ts = ((GgufArchive *)h)->tensors();
  if (i < 0 || (size_t)i >= ts.size()) return -1;
  const GgufTensor &t = ts[(size_t)i];
  *ggml_type = (int32_t)t.ggml_type;
  *n_dims = (int32_t)t.dims.size();
  for (size_t d = 0; d < t.dims.size() && d < 8; d++) dims[d] = t.dims[d];
  *shard = t.shard;
  *offset = (int64_t)t.offset;
  *nbytes = t.nbytes;
  return copy_out(t.name, name, name_cap);
}
const void *mrs_gguf_tensor_data(void *h, int64_t i) {
  const auto &ts = ((GgufArchive *)h)->tensors();
  if (i < 0 || (size_t)i >= ts.size()) return nullptr;
  return ((GgufArchive *)h)->tensor_data((size_t)i);
}

// metadata: key by index; value type / array element type / array length
int32_t mrs_gguf_meta_key(void *h, int64_t i, char *key, int64_t cap, int32_t *vtype, int32_t *arr_type, int64_t *arr_len) {
  const auto &keys = ((GgufArchive *)h)->metadata_keys();
  if (i < 0 || (size_t)i >= keys.size()) return -1;
  const GgufValue *v = ((GgufArchive *)h)->metadata(keys[(size_t)i]);
  *vtype = (int32_t)v->type;
  *arr_type = (int32_t)v->arr_type;
  *arr_len = v->type == GV_ARR ? (int64_t)v->arr_len() : 0;
  return copy_out(keys[(size_t)i], key, cap);
}
// 1 = found and of a compatible kind, 0 otherwise
int32_t mrs_gguf_meta_int(void *h, const char *key, int64_t *out) {
  const GgufValue *v = ((GgufArchive *)h)->metadata(key);
  if (v == nullptr || !v->is_int()) return 0;
  *out = v->as_int();
  return 1;
}
int32_t mrs_gguf_meta_float(void *h, const char *key, double *out) {
  const GgufValue *v = ((GgufArchive *)h)->metadata(key);
  if (v == nullptr) return 0;
  if (v->type == GV_F32 || v->type == GV_F64) { *out = v->f; return 1; }
  if (v->is_int()) { *out = (double)v->as_int(); return 1; }
  return 0;
}
// returns the string length (copying at most cap-1 bytes), -1 when absent / not a string
int64_t mrs_gguf_meta_str(void *h, const char *key, char *buf, int64_t cap) {
  const GgufValue *v = ((GgufArchive *)h)->metadata(key);
  if (v == nullptr || v->type != GV_STR) return -1;
  return copy_out(v->s, buf, cap);
}
int64_t mrs_gguf_meta_arr_str(void *h, const char *key, int64_t idx, char *buf, int64_t cap) {
  const GgufValue *v = ((GgufArchive *)h)->metadata(key);
  if (v == nullptr || v->type != GV_ARR || v->arr_type != GV_STR || idx < 0 || (size_t)idx >= v->arr_str.size()) return -1;
  return copy_out(v->arr_str[(size_t)idx], buf, cap);
}
// numeric arrays: copies up to `cap` elements starting at `start` as f64 (and exact ints when out_int != NULL)
int64_t mrs_gguf_meta_arr_num(void *h, const char *key, int64_t start, int64_t cap, double *out, int64_t *out_int) {
  const GgufValue *v = ((GgufArchive *)h)->metadata(key);
  if (v == nullptr || v->type != GV_ARR || v->arr_type == GV_STR || start < 0) return -1;
  int64_t n = 0;
  for (size_t k = (size_t)start; k < v->arr_num.size() && n < cap; k++, n++) {
    if (out != nullptr) out[n] = v->arr_num[k];
    if (out_int != nullptr) out_int[n] = v->arr_int[k];
  }
  return n;
}


// ---------------------------------------------------------------- safetensors containers (UQFF shards)
void *mrs_st_open(const char *path, char *err, int64_t err_cap) {
  try {
    return new SafetensorsFile(path);
  } catch (const std::exception &e) {
    copy_out(e.what(), err, err_cap);
    return nullptr;
  }
}
void mrs_st_close(void *h) { delete (SafetensorsFile *)h; }
int64_t mrs_st_n_tensors(void *h) { return (int64_t)((SafetensorsFile *)h)->tensors().size(); }
int64_t mrs_st_find(void *h, const char *name) { return ((SafetensorsFile *)h)->find(name); }
// dtype: safetensors dtype string ("U8", "U32", "BF16", ...) into a >= 16-byte buffer; dims: up to 8
int32_t mrs_st_tensor_info(void *h, int64_t i, char *name, int64_t name_cap, char *dtype, int32_t *n_dims, int64_t *dims,
                           int64_t *offset, int64_t *nbytes) {
  const auto &ts = ((SafetensorsFile *)h)->tensors();
  if (i < 0 || (size_t)i >= ts.size()) return -1;
  const StTensor &t = ts[(size_t)i];
  copy_out(t.dtype, dtype, 16);
  *n_dims = (int32_t)t.shape.size();
  for (size_t d = 0; d < t.shape.size() && d < 8; d++) dims[d] = t.shape[d];
  *offset = (int64_t)t.begin;
  *nbytes = (int64_t)(t.end - t.begin);
  return copy_out(t.name, name, name_cap);
}
const void *mrs_st_tensor_data(void *h, int64_t i) {
  const auto &ts = ((SafetensorsFile *)h)->tensors();
  if (i < 0 || (size_t)i >= ts.size()) return nullptr;
  return ((SafetensorsFile *)h)->data((size_t)i);
}
int64_t mrs_st_n_metadata(void *h) { return (int64_t)((SafetensorsFile *)h)->metadata().size(); }
// returns the value length (key/value copied with truncation), -1 on a bad index
int64_t mrs_st_metadata(void *h, int64_t i, char *key, int64_t key_cap, char *val, int64_t val_cap) {
  const auto &m = ((SafetensorsFile *)h)->metadata();
  if (i < 0 || (size_t)i >= m.size()) return -1;
  copy_out(m[(size_t)i].first, key, key_cap);
  return copy_out(m[(size_t)i].second, val, val_cap);
}

}  // extern "C"
