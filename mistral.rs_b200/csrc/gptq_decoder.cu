// gptq_decoder.cu — decode layer stack for GPTQ / AWQ int4 checkpoints (Mistral / Llama family)
// at serving batch sizes (BASELINE config 4: Mistral-7B GPTQ g128, batch 32, paged KV block 16).
//
// REF structure mirrored: mistralrs-core/src/models/mistral.rs (Attention / MLP / DecoderLayer
// forward over `QuantMethod` linears), with the linears on the reference's Marlin symbols
// (gptq/marlin_ffi.rs) — here the swap-AB wgmma kernel of w4a16.cu — and the lm_head as the dense
// 16-bit linear the checkpoint keeps.  Per layer (8 launches):
//   [RMSNorm] -> fused QKV GEMM -> RoPE + KV write + paged decode attention (one launch, HND; or the
//   rotary -> reshape_and_cache -> paged_attention_v1 chain for the vLLM layout) -> o_proj GEMM ->
//   add + RMSNorm -> gate||up GEMM -> SiLU*mul -> down GEMM -> add + RMSNorm (next layer's norm)
// Act-order checkpoints (mrs_gptq_layer perm_* set): the norms in front of q||k||v and gate||up write their output in
// the linear's row order, and a column gather of the attention output feeds o_proj; without them no launch changes.
// mrs_gptq_prefill_step runs the same chain over the packed prompt rows of up to 256 sequences, on whole-K GEMMs with
// gate||up through the GLU epilogue, and the prompt attention of the Llama prompt step (prompt_step.cuh).
// mrs_gptq_verify_step runs the decode chain over k + 1 rows per sequence (speculative decoding) with the multi-query
// fused attention, then the greedy acceptance on the device.
#include "common.cuh"
#include "mrs_b200_model.h"
#include "prompt_step.cuh"


extern "C" int32_t mrs_w4a16_gemm(const void *x, const void *w_tiles, const void *scales, const int32_t *qzeros, void *y,
                                  int32_t M, int32_t K, int32_t N, int32_t group, int32_t dtype, int32_t scale_perm,
                                  void *stream);
extern "C" int32_t mrs_dense_linear(const void *x, const void *w, void *y, int32_t M, int32_t K, int32_t N, int32_t dtype,
                                    void *stream);
extern "C" void mrs_rms_norm_f16(const void *x, const void *weight, void *dst, const int nrows, const int ncols, const float eps, int64_t stream);
extern "C" void mrs_rms_norm_bf16(const void *x, const void *weight, void *dst, const int nrows, const int ncols, const float eps, int64_t stream);
extern "C" void add_rms_norm_f16(const void *x, const void *residual, const void *weight, void *residual_dst, void *norm_dst, const int nrows, const int ncols, const float eps, int64_t stream);
extern "C" void add_rms_norm_bf16(const void *x, const void *residual, const void *weight, void *residual_dst, void *norm_dst, const int nrows, const int ncols, const float eps, int64_t stream);
extern "C" void fused_split_glu_f16(const void *input, void *output, uint32_t rows, uint32_t split_size, int activation, cudaStream_t stream);
extern "C" void fused_split_glu_bf16(const void *input, void *output, uint32_t rows, uint32_t split_size, int activation, cudaStream_t stream);
extern "C" int32_t mrs_paged_decode_fused_strided(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                                                  const void *rope_cos, const void *rope_sin, const int32_t *positions,
                                                  const int64_t *slot_mapping, const int32_t *kv_indptr,
                                                  const int32_t *kv_indices, const int32_t *kv_last_page_len,
                                                  const int32_t *request_indices, const int32_t *kv_tile_indices,
                                                  const int32_t *o_indptr, const int32_t *kv_chunk_size_ptr,
                                                  const uint8_t *block_valid_mask, void *o, void *tmp_v, float *tmp_s,
                                                  int32_t *counters, int32_t batch_size, int32_t padded_batch_size,
                                                  int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size,
                                                  int32_t page_size, float sm_scale, uint32_t dtype, int32_t pdl,
                                                  int64_t q_stride_n, int64_t kv_new_stride, void *stream);
extern "C" void rotary_embedding_positions(void *query, void *key, void *cos_cache, void *sin_cache, void *positions,
                                           int32_t is_neox, int32_t head_size, int64_t num_tokens, int32_t rot_dim,
                                           int32_t seq_len, int32_t num_heads, int32_t num_kv_heads, int64_t query_stride,
                                           int64_t key_stride, uint32_t dtype, int64_t stream);
extern "C" void reshape_and_cache(void *key, void *value, void *key_cache, void *value_cache, int64_t *slot_mapping,
                                  int32_t num_tokens, int32_t num_heads, int32_t head_size, int32_t block_size, int32_t x,
                                  int32_t key_stride, int32_t value_stride, cudaStream_t stream, uint32_t dtype,
                                  uint32_t cache_dtype, float *k_scale, float *v_scale);
extern "C" void paged_attention_v1_f16(void *out, void *query, void *key_cache, void *value_cache, void *alibi_slopes,
                                       int32_t num_kv_heads, float scale, float softcapping, uint32_t *block_tables,
                                       uint32_t *context_lens, int32_t block_size, int32_t max_context_len, int32_t num_seqs,
                                       int32_t num_heads, int32_t head_size, int32_t max_num_blocks_per_seq, int32_t q_stride,
                                       int32_t kv_block_stride, int32_t kv_head_stride, cudaStream_t stream,
                                       uint32_t cache_dtype, float *k_scale, float *v_scale, const float *sinks);
extern "C" void paged_attention_v1_bf16(void *out, void *query, void *key_cache, void *value_cache, void *alibi_slopes,
                                        int32_t num_kv_heads, float scale, float softcapping, uint32_t *block_tables,
                                        uint32_t *context_lens, int32_t block_size, int32_t max_context_len, int32_t num_seqs,
                                        int32_t num_heads, int32_t head_size, int32_t max_num_blocks_per_seq, int32_t q_stride,
                                        int32_t kv_block_stride, int32_t kv_head_stride, cudaStream_t stream,
                                        uint32_t cache_dtype, float *k_scale, float *v_scale, const float *sinks);
extern "C" int32_t mrs_argmax(const void *logits, int32_t rows, int32_t cols, int32_t act_dtype, int32_t *out, void *scratch,
                              int32_t pdl, void *stream);

namespace mrs {
// dense embedding rows: out[b, :] = table[ids[b], :]   (16-bit elements, 16-byte vectors)
__global__ void dense_embedding_kernel(const uint4 *__restrict__ table, int cols8, const int32_t *__restrict__ ids,
                                       uint4 *__restrict__ out) {
  const int64_t row = ids[blockIdx.x];
  for (int i = threadIdx.x; i < cols8; i += blockDim.x) out[(int64_t)blockIdx.x * cols8 + i] = table[row * cols8 + i];
}
}  // namespace mrs

extern "C" int32_t mrs_w4a16_gemm_pdl(const void *x, const void *w_tiles, const void *scales, const int32_t *qzeros, void *y,
                                      int32_t M, int32_t K, int32_t N, int32_t group, int32_t dtype, int32_t scale_perm,
                                      int32_t pdl, void *stream);
extern "C" int32_t mrs_dense_linear_pdl(const void *x, const void *w, void *y, int32_t M, int32_t K, int32_t N, int32_t dtype,
                                        int32_t pdl, void *stream);
extern "C" void mrs_add_rms_norm_pdl(const void *x, const void *residual, const void *weight, void *residual_dst, void *norm_dst,
                                     int32_t nrows, int32_t ncols, float eps, int32_t dtype, int32_t pdl, void *stream);
extern "C" void mrs_split_glu_pdl(const void *input, void *output, uint32_t rows, uint32_t split_size, int32_t activation,
                                  int32_t dtype, int32_t pdl, void *stream);
extern "C" int32_t mrs_rms_norm_perm_pdl(const void *x, const void *weight, const int32_t *perm, void *norm_dst, int32_t nrows,
                                         int32_t ncols, float eps, int32_t dtype, int32_t pdl, void *stream);
extern "C" int32_t mrs_add_rms_norm_perm_pdl(const void *x, const void *residual, const void *weight, const int32_t *perm,
                                             void *residual_dst, void *norm_dst, int32_t nrows, int32_t ncols, float eps,
                                             int32_t dtype, int32_t pdl, void *stream);
extern "C" int32_t mrs_gather_cols_pdl(const void *x, const int32_t *perm, void *y, int32_t rows, int32_t cols, int32_t pdl,
                                       void *stream);

extern "C" int32_t mrs_paged_decode_fused_multi_strided(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                                                        const void *rope_cos, const void *rope_sin, const int32_t *positions,
                                                        const int64_t *slot_mapping, const int32_t *kv_indptr,
                                                        const int32_t *kv_indices, const int32_t *kv_last_page_len,
                                                        const int32_t *request_indices, const int32_t *kv_tile_indices,
                                                        const int32_t *o_indptr, const int32_t *kv_chunk_size_ptr,
                                                        const uint8_t *block_valid_mask, void *o, void *tmp_v, float *tmp_s,
                                                        int32_t *counters, int32_t batch_size, int32_t padded_batch_size,
                                                        int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size,
                                                        int32_t page_size, float sm_scale, uint32_t dtype, int32_t pdl,
                                                        int32_t q_len, int64_t q_stride_n, int64_t kv_new_stride,
                                                        void *stream);
extern "C" int32_t mrs_spec_accept(const int32_t *argmax, int32_t *token_ids, const int64_t *slot_mapping,
                                   int32_t *context_lens, int32_t *accepted, int32_t *emitted, int32_t batch, int32_t q_len,
                                   int32_t pdl, void *stream);

// act-order layers: every layer whose perm_o is set needs the attn_perm scratch, and a permuted norm stages a row of
// `hidden` elements in shared memory
static bool gptq_perms_ok(const mrs_gptq_step *s) {
  if (s->layers == nullptr) return true;
  bool any = false;
  for (int l = 0; l < s->n_layers; l++) {
    const mrs_gptq_layer &L = s->layers[l];
    if (L.perm_o != nullptr && s->attn_perm == nullptr) return false;
    any |= L.perm_qkv != nullptr || L.perm_gate_up != nullptr;
  }
  return !any || (size_t)s->hidden * 2 <= 48 * 1024;
}

// the decode layer chain + lm_head + argmax over s->batch sequences of q_len rows each (R = batch * q_len rows in every
// row buffer): q_len == 1 is the decode step, q_len 2..8 a speculative verify step (HND layout only), whose attention is
// the multi-query fused kernel reading q, k and v inside the q||k||v rows
static int32_t gptq_forward(const mrs_gptq_step *s, int q_len, void *stream) {
  const int dt = s->act_dtype, B = s->batch, R = B * q_len, H = s->hidden;
  const int nq = s->n_heads * s->head_dim, nkv = s->n_kv_heads * s->head_dim, nqkv = nq + 2 * nkv;
  cudaStream_t st = (cudaStream_t)stream;
  const bool f16 = dt == MRS_F16;
  auto rms = [&](const void *x, const void *w, void *dst) {
    if (f16) mrs_rms_norm_f16(x, w, dst, R, H, s->rms_eps, (int64_t)stream); else mrs_rms_norm_bf16(x, w, dst, R, H, s->rms_eps, (int64_t)stream);
  };
  // Every launch of the layer loop is a link of ONE programmatic-dependent-launch chain (skip_mask bit 2 turns it
  // off): each kernel triggers its dependents when it starts and waits for the upstream grid before touching its
  // inputs / outputs, so the W4A16 GEMMs stream their weights while the small kernels before them still run.
  // The HND attention launch is PDL-capable; the vLLM-layout chain (reference-ABI kernels, no PDL forms) is not,
  // so that layout keeps plain stream order.
  const int pdl = ((s->skip_mask & 4) || s->cache_layout != 1) ? 0 : 1;
  // a norm whose consumer is an act-order linear writes its output in that linear's row order (perm != NULL)
  auto add_rms = [&](const void *x, const void *res, const void *w, void *res_dst, void *norm_dst, const int32_t *perm) -> int {
    if (perm != nullptr) return mrs_add_rms_norm_perm_pdl(x, res, w, perm, res_dst, norm_dst, R, H, s->rms_eps, dt, pdl, stream);
    mrs_add_rms_norm_pdl(x, res, w, res_dst, norm_dst, R, H, s->rms_eps, dt, pdl, stream);
    return 0;
  };
  // the same GEMM route for plain and verify steps: no whole-K bit, so both pick their K split by row count alone
  auto linear = [&](const mrs_w4_weight &w, const void *x, void *y) -> int {
    return mrs_w4a16_gemm_pdl(x, w.tiles, w.scales, (const int32_t *)w.qzeros, y, R, w.k, w.n, s->group_size, dt, 0, pdl, stream);
  };
  const bool do_attn = !(s->skip_mask & 1), do_lin = !(s->skip_mask & 2);
  void *tmp_v = s->padded_tiles > B ? s->tmp_v : nullptr;
  float *tmp_s = s->padded_tiles > B ? s->tmp_s : nullptr;
  const int rope_flags = (s->rope_neox ? 0 : 2) | pdl;

  mrs::dense_embedding_kernel<<<R, 256, 0, st>>>((const uint4 *)s->tok_embd, H / 8, s->token_ids, (uint4 *)s->x);
  void *x = s->x, *x2 = s->x2;   // residual stream ping-pong
  if (s->layers[0].perm_qkv != nullptr)
    MRS_TRY(mrs_rms_norm_perm_pdl(x, s->layers[0].attn_norm, s->layers[0].perm_qkv, s->h, R, H, s->rms_eps, dt, 0, stream));
  else
    rms(x, s->layers[0].attn_norm, s->h);
  for (int l = 0; l < s->n_layers; l++) {
    const mrs_gptq_layer &L = s->layers[l];
    if (do_lin) MRS_TRY(linear(L.wqkv, s->h, s->qkv));
    void *q = s->qkv, *k = (char *)s->qkv + (size_t)nq * 2, *v = (char *)s->qkv + (size_t)(nq + nkv) * 2;
    if (do_attn && q_len > 1) {
      MRS_TRY(mrs_paged_decode_fused_multi_strided(q, k, v, L.k_cache, L.v_cache, s->rope_cos, s->rope_sin, s->positions,
                                                   s->slot_mapping, s->kv_indptr, s->kv_indices, s->kv_last_page_len,
                                                   s->request_indices, s->kv_tile_indices, s->o_indptr, s->kv_chunk_size,
                                                   s->block_valid_mask, s->attn_out, tmp_v, tmp_s, s->attn_counters, B,
                                                   s->padded_tiles, s->n_heads, s->n_kv_heads, s->head_dim, s->block_size,
                                                   s->sm_scale, (uint32_t)dt, rope_flags, q_len, nqkv, nqkv, stream));
    } else if (do_attn && s->cache_layout == 1) {
      MRS_TRY(mrs_paged_decode_fused_strided(q, k, v, L.k_cache, L.v_cache, s->rope_cos, s->rope_sin, s->positions,
                                             s->slot_mapping, s->kv_indptr, s->kv_indices, s->kv_last_page_len,
                                             s->request_indices, s->kv_tile_indices, s->o_indptr, s->kv_chunk_size,
                                             s->block_valid_mask, s->attn_out, tmp_v, tmp_s, s->attn_counters, B,
                                             s->padded_tiles, s->n_heads, s->n_kv_heads, s->head_dim, s->block_size,
                                             s->sm_scale, (uint32_t)dt, rope_flags, nqkv, nqkv, stream));
    } else if (do_attn) {
      // vLLM cache layout (REF MISTRALRS_FLASHINFER_DECODE=0): rotary -> reshape_and_cache -> paged_attention_v1
      rotary_embedding_positions(q, k, (void *)s->rope_cos, (void *)s->rope_sin, s->positions, s->rope_neox, s->head_dim, B,
                                 s->head_dim / 2, 0, s->n_heads, s->n_kv_heads, nqkv, nqkv, (uint32_t)dt, (int64_t)stream);
      reshape_and_cache(k, v, L.k_cache, L.v_cache, s->slot_mapping, B, s->n_kv_heads, s->head_dim, s->block_size, 8, nqkv,
                        nqkv, st, (uint32_t)dt, (uint32_t)dt, nullptr, nullptr);
      const int kv_block_stride = s->n_kv_heads * s->head_dim * s->block_size, kv_head_stride = s->head_dim * s->block_size;
      if (f16)
        paged_attention_v1_f16(s->attn_out, q, L.k_cache, L.v_cache, nullptr, s->n_kv_heads, s->sm_scale, 1.0f,
                               (uint32_t *)s->block_tables, (uint32_t *)s->context_lens, s->block_size,
                               s->max_blocks_per_seq * s->block_size, B, s->n_heads, s->head_dim, s->max_blocks_per_seq, nqkv,
                               kv_block_stride, kv_head_stride, st, (uint32_t)dt, nullptr, nullptr, nullptr);
      else
        paged_attention_v1_bf16(s->attn_out, q, L.k_cache, L.v_cache, nullptr, s->n_kv_heads, s->sm_scale, 1.0f,
                                (uint32_t *)s->block_tables, (uint32_t *)s->context_lens, s->block_size,
                                s->max_blocks_per_seq * s->block_size, B, s->n_heads, s->head_dim, s->max_blocks_per_seq, nqkv,
                                kv_block_stride, kv_head_stride, st, (uint32_t)dt, nullptr, nullptr, nullptr);
    }
    const void *o_in = s->attn_out;
    if (L.perm_o != nullptr) {                                                // o_proj's rows in act order
      MRS_TRY(mrs_gather_cols_pdl(s->attn_out, L.perm_o, s->attn_perm, R, nq, pdl, stream));
      o_in = s->attn_perm;
    }
    if (do_lin) MRS_TRY(linear(L.wo, o_in, s->o));
    MRS_TRY(add_rms(s->o, x, L.ffn_norm, x2, s->h, L.perm_gate_up));          // x2 = o + x ; h = norm(x2)
    if (do_lin) MRS_TRY(linear(L.w_gate_up, s->h, s->gate_up));
    mrs_split_glu_pdl(s->gate_up, s->act, R, L.w_down.k, 0, dt, pdl, stream);
    if (do_lin) MRS_TRY(linear(L.w_down, s->act, s->o));
    const bool last = l + 1 == s->n_layers;
    const void *next_norm = last ? s->final_norm : s->layers[l + 1].attn_norm;
    MRS_TRY(add_rms(s->o, x2, next_norm, x, s->h, last ? nullptr : s->layers[l + 1].perm_qkv));   // x = down + x2 ; h = next norm(x)
  }
  if (do_lin) MRS_TRY(mrs_dense_linear_pdl(s->h, s->lm_head, s->logits, R, H, s->vocab, dt, pdl, stream));
  MRS_TRY(mrs_argmax(s->logits, R, s->vocab, dt, s->out_token, s->argmax_scratch, 0, stream));
  return (int32_t)cudaGetLastError();
}

extern "C" int32_t mrs_gptq_decode_step(const mrs_gptq_step *s, void *stream) {
  const int dt = s->act_dtype, B = s->batch;
  if (B < 1 || B > 256 || (dt != MRS_F16 && dt != MRS_BF16) || s->hidden % 8 || !gptq_perms_ok(s))
    return (int32_t)cudaErrorInvalidValue;
  return gptq_forward(s, 1, stream);
}

// the verify step of speculative decoding (contract: include/mrs_b200_model.h): the decode chain over B * q_len rows,
// then the greedy acceptance on the device, as mrs_llama_verify_step
extern "C" int32_t mrs_gptq_verify_step(const mrs_gptq_step *s, int32_t q_len, int32_t *context_lens, int32_t *accepted,
                                        int32_t *emitted, void *stream) {
  if (s == nullptr || s->batch < 1 || s->batch > 256 || q_len < 2 || q_len > 8 || s->cache_layout != 1 ||
      (s->head_dim != 64 && s->head_dim != 128) || (s->act_dtype != MRS_F16 && s->act_dtype != MRS_BF16) ||
      s->hidden % 8 != 0 || s->layers == nullptr || s->out_token == s->token_ids || context_lens == nullptr ||
      accepted == nullptr || emitted == nullptr || !gptq_perms_ok(s))
    return (int32_t)cudaErrorInvalidValue;
  MRS_TRY(gptq_forward(s, q_len, stream));
  const int pdl = (s->skip_mask & 4) ? 0 : 1;
  return mrs_spec_accept(s->out_token, s->token_ids, s->slot_mapping, context_lens, accepted, emitted, s->batch, q_len, pdl,
                         stream);
}

// the prompt step over the packed rows of n sequences (contract: include/mrs_b200_model.h): the decode step's layer
// chain over T rows with whole-K GEMMs, gate||up through the GLU epilogue, and the var-len prompt attention
using namespace mrs;

extern "C" int32_t mrs_gptq_prefill_step(const mrs_gptq_step *s, const mrs_llama_prefill *p, void *stream) {
  if (s == nullptr || p == nullptr) return (int32_t)cudaErrorInvalidValue;
  const int n = p->n_seqs, T = p->total_tokens, dt = s->act_dtype, H = s->hidden;
  const bool vllm_cache = s->cache_layout != 1;
  if (n < 1 || n > 256 || T < n || (dt != MRS_F16 && dt != MRS_BF16) || p->lm_rows < 0 || p->lm_rows > 2 ||
      (p->paged != 0 && p->paged != 1) || (p->paged && vllm_cache) || (p->dest_rows != nullptr && p->lm_rows != 1) ||
      p->max_q_len < 1 || p->max_kv_len < p->max_q_len || H % 8 != 0)
    return (int32_t)cudaErrorInvalidValue;
  if (s->layers == nullptr || p->token_ids == nullptr || p->positions == nullptr ||
      p->slot_mapping == nullptr || p->cu_seqlens_q == nullptr || p->cu_seqlens_k == nullptr || p->x == nullptr ||
      p->x2 == nullptr || p->h == nullptr || p->q == nullptr || p->attn_out == nullptr || p->act == nullptr)
    return (int32_t)cudaErrorInvalidValue;
  if (p->paged && (p->block_tables == nullptr || p->block_table_stride < 1 || p->num_blocks < 1)) return (int32_t)cudaErrorInvalidValue;
  if (p->lm_rows == 1 && (p->last_rows == nullptr || p->h_last == nullptr || p->logits == nullptr || p->out_token == nullptr ||
                          p->argmax_scratch == nullptr))
    return (int32_t)cudaErrorInvalidValue;
  if (p->lm_rows == 2 && p->logits == nullptr) return (int32_t)cudaErrorInvalidValue;
  if (p->dest_rows != nullptr && (p->runner_token_ids == nullptr || p->runner_context_lens == nullptr))
    return (int32_t)cudaErrorInvalidValue;
  if (!gptq_perms_ok(s)) return (int32_t)cudaErrorInvalidValue;

  const int nq = s->n_heads * s->head_dim, nkv = s->n_kv_heads * s->head_dim, nqkv = nq + 2 * nkv;
  // the attention launches are plain kernels, which a PDL link may follow: the GEMMs and norms are links in both layouts
  const int pdl = (s->skip_mask & 4) ? 0 : 1;
  // flags | 2: K is never split, so a row's result does not depend on the other rows of the call
  auto linear = [&](const mrs_w4_weight &w, const void *x, void *y, int flags) -> int32_t {
    return mrs_w4a16_gemm_pdl(x, w.tiles, w.scales, (const int32_t *)w.qzeros, y, T, w.k, w.n, s->group_size, dt, 0,
                              pdl | 2 | flags, stream);
  };
  // res_dst = h + res ; h = norm(res_dst), in the row order of the act-order linear after it when perm != NULL
  auto add_rms = [&](const void *res, const void *w, void *res_dst, const int32_t *perm) -> int32_t {
    if (perm != nullptr) return mrs_add_rms_norm_perm_pdl(p->h, res, w, perm, res_dst, p->h, T, H, s->rms_eps, dt, pdl, stream);
    mrs_add_rms_norm_pdl(p->h, res, w, res_dst, p->h, T, H, s->rms_eps, dt, pdl, stream);
    return 0;
  };
  const PromptAttnModel am{s->n_heads, s->n_kv_heads, s->head_dim, s->block_size, s->rope_neox, dt, s->sm_scale, s->rope_cos,
                           s->rope_sin};

  mrs::dense_embedding_kernel<<<T, 256, 0, (cudaStream_t)stream>>>((const uint4 *)s->tok_embd, H / 8, p->token_ids, (uint4 *)p->x);
  if (s->layers[0].perm_qkv != nullptr)
    MRS_TRY(mrs_rms_norm_perm_pdl(p->x, s->layers[0].attn_norm, s->layers[0].perm_qkv, p->h, T, H, s->rms_eps, dt, 0, stream));
  else if (dt == MRS_F16) mrs_rms_norm_f16(p->x, s->layers[0].attn_norm, p->h, T, H, s->rms_eps, (int64_t)stream);
  else mrs_rms_norm_bf16(p->x, s->layers[0].attn_norm, p->h, T, H, s->rms_eps, (int64_t)stream);
  for (int l = 0; l < s->n_layers; l++) {
    const mrs_gptq_layer &L = s->layers[l];
    MRS_TRY(linear(L.wqkv, p->h, p->q, 0));                                   // p->q holds the [T, nqkv] qkv rows
    void *q = p->q, *k = (char *)p->q + (size_t)nq * 2, *v = (char *)p->q + (size_t)(nq + nkv) * 2;
    MRS_TRY(prompt_attention(p, am, q, k, v, nqkv, nqkv, L.k_cache, L.v_cache, vllm_cache, stream));
    // the o and down GEMMs write into h, which the add + RMSNorm after them reads as its input and overwrites
    const void *o_in = p->attn_out;
    if (L.perm_o != nullptr) {                                                // o_proj's rows in act order: [T, nq] scratch
      MRS_TRY(mrs_gather_cols_pdl(p->attn_out, L.perm_o, s->attn_perm, T, nq, pdl, stream));
      o_in = s->attn_perm;
    }
    MRS_TRY(linear(L.wo, o_in, p->h, 0));
    MRS_TRY(add_rms(p->x, L.ffn_norm, p->x2, L.perm_gate_up));               // x2 = o + x ; h = norm(x2)
    MRS_TRY(linear(L.w_gate_up, p->h, p->act, 4));                           // act = silu(gate) * up
    MRS_TRY(linear(L.w_down, p->act, p->h, 0));
    const bool last = l + 1 == s->n_layers;
    MRS_TRY(add_rms(p->x2, last ? s->final_norm : s->layers[l + 1].attn_norm, p->x,
                    last ? nullptr : s->layers[l + 1].perm_qkv));            // x = down + x2 ; h = next norm(x)
  }
  if (p->lm_rows == 2) {
    MRS_TRY(mrs_dense_linear_pdl(p->h, s->lm_head, p->logits, T, H, s->vocab, dt, pdl | 2, stream));
  } else if (p->lm_rows == 1) {
    prompt_gather_last_rows(p, p->h, H, stream);
    MRS_TRY(mrs_dense_linear_pdl(p->h_last, s->lm_head, p->logits, n, H, s->vocab, dt, pdl | 2, stream));
    MRS_TRY(mrs_argmax(p->logits, n, s->vocab, dt, p->out_token, p->argmax_scratch, pdl, stream));
    if (p->dest_rows != nullptr) prompt_commit(p, stream);
  }
  return (int32_t)cudaGetLastError();
}
