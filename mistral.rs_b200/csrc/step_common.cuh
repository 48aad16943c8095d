// step_common.cuh — the parts of the Llama (decoder.cu) and GPTQ (gptq_decoder.cu) steps that do not depend on how the
// linears are stored: the fused decode attention of the decode and verify steps (a template, defined here), and the
// plan check, attention, last-row gather and runner commit of the prompt steps (mrs_b200_model.h: mrs_llama_prefill),
// defined in decoder.cu.
#pragma once
#include "mrs_b200_model.h"
#include "mrs_b200_paged_attn.h"

namespace mrs {

// The fused HND decode attention of layer caches k_cache / v_cache over s->batch sequences of q_len rows each (Step:
// mrs_llama_step or mrs_gptq_step, which name the decode metadata alike): RoPE + KV write + paged attention + split-KV
// merge in one launch, mrs_paged_decode_fused_multi_strided for a verify step (q_len > 1), else
// mrs_paged_decode_fused_strided.  q rows are q_stride elements apart, k / v rows kv_stride; output into s->attn_out.
// pdl: bit 0 of the launch's flags (bit 1, the interleaved RoPE pairing, comes from s->rope_neox).  The split-KV
// partials tmp_v / tmp_s are passed only when the plan has more tiles than sequences.
template <class Step>
int32_t fused_decode_attention(const Step *s, void *k_cache, void *v_cache, void *q, void *k, void *v, int64_t q_stride,
                               int64_t kv_stride, int q_len, int pdl, void *stream) {
  const int B = s->batch, flags = pdl | (s->rope_neox ? 0 : 2);
  void *tmp_v = s->padded_tiles > B ? s->tmp_v : nullptr;
  float *tmp_s = s->padded_tiles > B ? s->tmp_s : nullptr;
  if (q_len > 1)
    return mrs_paged_decode_fused_multi_strided(q, k, v, k_cache, v_cache, s->rope_cos, s->rope_sin, s->positions,
                                                s->slot_mapping, s->kv_indptr, s->kv_indices, s->kv_last_page_len,
                                                s->request_indices, s->kv_tile_indices, s->o_indptr, s->kv_chunk_size,
                                                s->block_valid_mask, s->attn_out, tmp_v, tmp_s, s->attn_counters, B,
                                                s->padded_tiles, s->n_heads, s->n_kv_heads, s->head_dim, s->block_size,
                                                s->sm_scale, (uint32_t)s->act_dtype, flags, q_len, q_stride, kv_stride,
                                                stream);
  return mrs_paged_decode_fused_strided(q, k, v, k_cache, v_cache, s->rope_cos, s->rope_sin, s->positions, s->slot_mapping,
                                        s->kv_indptr, s->kv_indices, s->kv_last_page_len, s->request_indices,
                                        s->kv_tile_indices, s->o_indptr, s->kv_chunk_size, s->block_valid_mask, s->attn_out,
                                        tmp_v, tmp_s, s->attn_counters, B, s->padded_tiles, s->n_heads, s->n_kv_heads,
                                        s->head_dim, s->block_size, s->sm_scale, (uint32_t)s->act_dtype, flags, q_stride,
                                        kv_stride, stream);
}

// what the Llama and GPTQ prompt steps both need of a plan: n 1..256, T >= n, an f16 / bf16 activation dtype, lm_rows
// 0..2, paged 0..1, dest_rows only with lm_rows 1, max_q_len >= 1, max_kv_len >= max_q_len, hidden % 8 == 0, and the
// pointers every step reads: the plan arrays, x / x2 / h / q / attn_out / act; block_tables (block_table_stride and
// num_blocks >= 1) when paged; last_rows / h_last / logits / out_token / argmax_scratch when lm_rows == 1; logits when
// lm_rows == 2; runner_token_ids / runner_context_lens when dest_rows is set
bool prompt_plan_ok(const mrs_llama_prefill *p, int act_dtype, int hidden);

// what the prompt attention needs of a model
struct PromptAttnModel {
  int n_heads, n_kv_heads, head_dim, block_size, rope_neox, act_dtype;
  float sm_scale;
  const void *rope_cos, *rope_sin;
};

// One layer's attention over the plan's T rows: RoPE at p->positions, then
//   paged 0: causal attention over the fresh q/k/v (cu_seqlens_q), then the K/V scatter into the cache;
//   paged 1: the scatter first, then the paged prompt attention over p->block_tables (HND cache only).
// q, k, v: rows of q_stride / kv_stride elements (k and v share theirs); attention output into p->attn_out [T, nq].
// vllm_cache: the cache is in the vLLM layout (K [NB, KVH, D/8, BS, 8], V [NB, KVH, D, BS]), written by
// reshape_and_cache; the caller rejects paged with it.
int32_t prompt_attention(const mrs_llama_prefill *p, const PromptAttnModel &m, void *q, void *k, void *v, int64_t q_stride,
                         int64_t kv_stride, void *k_cache, void *v_cache, bool vllm_cache, void *stream);
// p->h_last[i] = h[p->last_rows[i]] for the n sequences, rows of `hidden` 16-bit elements (hidden % 8 == 0)
void prompt_gather_last_rows(const mrs_llama_prefill *p, const void *h, int hidden, void *stream);
// the hand-off to a decode runner (p->dest_rows set): its row dest_rows[i] continues sequence i from out_token[i], at
// the context length the step left in the cache
void prompt_commit(const mrs_llama_prefill *p, void *stream);

}  // namespace mrs
