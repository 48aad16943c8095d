// prompt_step.cuh — the parts of a prompt step (mrs_b200_model.h: mrs_llama_prefill) that do not depend on how the
// linears are stored, shared by the Llama (decoder.cu) and GPTQ (gptq_decoder.cu) prompt steps; defined in decoder.cu.
#pragma once
#include "mrs_b200_model.h"

namespace mrs {

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
