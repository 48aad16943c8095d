/* mrs_b200_model.h — C ABI of the native Llama-family decode layer stack.
 *
 * This is the host-side caller of the hot path (the role of `Llama::forward` /
 * `Block::forward` in the reference: mistralrs-core/src/models/llama.rs:243-260,475-…),
 * restricted to what the benchmark needs: it owns no memory, takes raw device pointers, and
 * enqueues the per-token kernel chain on the given stream (CUDA-graph capturable: no
 * allocation, no host sync).  Per decoder layer it issues
 *     [RMSNorm + Q8_1 + fused QKV GEMV] -> RoPE -> KV-cache write -> paged decode attention
 *     -> [Q8_1 + o_proj GEMV + residual] -> [RMSNorm + Q8_1 + gate/up GEMV + SiLU*mul + Q8_1]
 *     -> [down GEMV + residual]
 * with the bracketed groups being single `mrs_mmvq_fused` launches.
 */
#ifndef MRS_B200_MODEL_H
#define MRS_B200_MODEL_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { const void *data; int32_t ggml_type; int32_t rows; int32_t cols; } mrs_qweight;

typedef struct {
  mrs_qweight wq, wk, wv, wo, w_gate, w_up, w_down; /* local (possibly TP-sharded) shapes */
  const void *attn_norm, *ffn_norm;                  /* [hidden] in the activation dtype */
  void *k_cache, *v_cache;                           /* HND [num_blocks, kv_heads, block_size, head_dim] */
} mrs_llama_layer;

/* Tensor-parallel context of the peer-memory all-reduce (one process per GPU; the buffers are
 * symmetric allocations whose peer mappings the host obtained by rendezvous, e.g.
 * torch.distributed._symmetric_memory): every rank owns [flags | slot 0 | slot 1] at the same offsets. */
typedef struct {
  int32_t world, rank;
  void *peer_base[8];            /* base of rank r's buffer as mapped in THIS process (own included) */
  int64_t flags_offset;          /* >= world uint32 flag words, zero-initialised */
  int64_t slot_offset[2];        /* two partial buffers of >= batch * hidden activation elements each */
  void *seq_counter;             /* local device uint32[2], zero-initialised: [0] all-reduces so far, [1] set to 1 when a
                                  * low-latency all-reduce gave up waiting for a peer (~0.25 s): results are invalid */
  /* low-latency protocol (used when ll_offset != 0): every rank PUSHES its partial to every peer as 8-byte words
   * {two activation elements, sequence number} — one NVLink store hop, no flag round trip, no fence; the receiver
   * polls the words themselves.  Region: [2 slots][world source ranks][ll_src_stride bytes], zero-initialised,
   * ll_src_stride >= 4 bytes per element of the largest all-reduce. */
  int64_t ll_offset, ll_slot_stride, ll_src_stride;
} mrs_tp_ctx;
/* out = T(T(sum over ranks of slot partials, rank order, f32) + residual); count % 8 == 0; one CTA, in-graph,
 * PDL-chained.  Stands in for SumAllReduce::sum_all_reduce + the residual add (REF distributed/mod.rs:436-453).
 * Two protocols, same arithmetic and bit-identical results on every rank: flags + pull (ll_offset == 0) and the
 * low-latency push above. */
int32_t mrs_tp_allreduce_residual(const mrs_tp_ctx *ctx, int32_t slot, const void *residual, void *out, int32_t count,
                                  int32_t dtype, int32_t pdl, void *stream);

typedef struct {
  int32_t hidden, n_layers, n_heads, n_kv_heads, head_dim, vocab; /* heads are LOCAL counts under TP */
  int32_t block_size, act_dtype;   /* act_dtype: 0 f16, 1 bf16 */
  float rms_eps, sm_scale;
  int32_t rope_neox, pdl;
  const mrs_llama_layer *layers;   /* host array [n_layers] */
  mrs_qweight tok_embd, lm_head;
  const void *final_norm, *rope_cos, *rope_sin; /* rope tables [max_pos, head_dim/2] act dtype */
  /* per-step device metadata (see mrs_decode_advance) */
  int32_t batch, padded_tiles, max_blocks_per_seq;
  int32_t skip_mask;         /* measurement only: bit0 skip rope/cache/attention, bit1 skip the GEMVs / GEMMs */
  int32_t fused_attention;   /* 1: mrs_paged_decode_fused; 0: rotary + reshape_and_cache + flashinfer_decode */
  int32_t reserved0;
  int32_t *token_ids;        /* [batch] in: token to process; out_token may alias it */
  int32_t *positions;        /* [batch] */
  int64_t *slot_mapping;     /* [batch] */
  int32_t *kv_indptr, *kv_indices, *kv_last_page_len;
  int32_t *request_indices, *kv_tile_indices, *o_indptr, *kv_chunk_size;
  uint8_t *block_valid_mask;
  /* scratch (activation dtype unless noted) */
  void *x, *x2, *q, *k, *v, *attn_out, *act, *logits; /* x, x2: [batch, hidden] residual stream ping-pong; on the
                              * GEMV route (batch <= 8) act holds the block_q8_1 form of the GLU output (36 B per 32) */
  void *tmp_v; float *tmp_s;
  int32_t *out_token;        /* [batch] argmax of the logits */
  int32_t *attn_counters;    /* zeroed int32 [batch * n_kv_heads * 2] (fused attention merge) */
  void *argmax_scratch;      /* zeroed, >= 16 * batch + 16 bytes */
  /* tensor parallel: called after the row-parallel projections when non-NULL */
  void (*all_reduce)(void *buf, int64_t count, int32_t dtype, void *stream, void *user);
  void *all_reduce_user;
  const mrs_tp_ctx *tp;      /* non-NULL with world > 1: peer-memory sum (takes precedence over all_reduce) */
  void *h;                   /* [batch, hidden] normed-activation scratch ([batch*q_len, hidden] for a verify step);
                              * read only when batch > 8 */
} mrs_llama_step;

/* Enqueue one decode step (all layers + lm_head + argmax) on `stream`. Returns cudaError.  batch 1..256.
 * batch 1..8: the GEMV chain above (Q8_1 activations, MMVQ numerics).
 * batch 9..256: the reference's MMQ branch — every linear is the wgmma dequant GEMM (mrs_mmq_gguf_grouped: weights
 * dequantised with the f32 formula and rounded once to the activation format, activations unquantised, f32
 * accumulation, the prefill GEMM's numerics).  Per layer: grouped QKV (one launch, or q|k + v when attn_v has its own
 * type) -> the same attention -> o GEMM -> add + RMSNorm -> gate|up GEMM with the SiLU*mul epilogue -> down GEMM
 * -> add + RMSNorm with the next layer's norm; then the lm_head GEMM and argmax.  Needs `h`; skip_mask bit 1 skips
 * the GEMMs.
 * cudaErrorInvalidValue, before any launch, for: batch outside 1..256; (batch >= 9) tp or all_reduce set (no tensor
 * parallelism above 8 rows), a NULL h or an activation dtype other than f16 / bf16; a NULL `layers` with n_layers >= 1;
 * a layer whose w_gate and w_up differ in ggml type or rows. */
int32_t mrs_llama_decode_step(const mrs_llama_step *s, void *stream);

/* On-device restatement of the scheduler-side index producers for a running decode batch
 * (REF inputs_processor.rs:896-923, flashinfer/metadata.rs:88-216): context_lens[b] += 1,
 * positions, slot_mapping, the paged-KV CSR and the split-KV tile plan for the new lengths,
 * all from the dense block table — so a whole generation replays as one CUDA graph.
 * batch <= 256.  A sequence at min(max_blocks_per_seq*block_size, max_pos) (max_pos <= 0: no RoPE
 * bound) stops growing: slot -1 (no KV write) and bit 0 of *error_flag (nullable) is set. */
int32_t mrs_decode_advance(const int32_t *block_tables, int32_t max_blocks_per_seq, int32_t *context_lens,
                           int32_t batch, int32_t block_size, int32_t split_pages, int32_t padded_tiles,
                           int32_t *positions, int64_t *slot_mapping, int32_t *kv_indptr, int32_t *kv_indices,
                           int32_t *kv_last_page_len, int32_t *request_indices, int32_t *kv_tile_indices,
                           int32_t *o_indptr, int32_t *kv_chunk_size, uint8_t *block_valid_mask,
                           int32_t max_pos, int32_t *error_flag, void *stream);

/* Speculative decoding (REF mistralrs-core/src/speculative/, greedy verification): one verify step scores q_len =
 * k + 1 rows per sequence — the anchor (the last sampled token, not yet in the cache) and k drafts — in one pass over
 * the weights, then accepts drafts on the device.
 *
 * mrs_decode_advance_multi: mrs_decode_advance for q_len rows per sequence.  Sequence b at context c gets
 * positions[b*q_len + i] = c + i with their slots, context_lens[b] = c + q_len, and the CSR / tile plan for that
 * length.  A sequence with c + q_len > min(max_blocks_per_seq*block_size, max_pos) is frozen whole: all its slots are
 * -1, context_lens[b] stays c, bit 0 of *error_flag is set.  q_len 1..8, that bound >= q_len.
 *
 * mrs_spec_accept: per sequence b, rows token_ids[b*q_len ..] = [anchor, draft 1..k] and argmax[b*q_len + i] = the
 * target's token after row i.  a = number of leading i < k with draft i+1 == argmax[i]; emitted[b*q_len + i] =
 * argmax[b*q_len + i] for i <= a, else -1; accepted[b] = a; context_lens[b] goes from c + q_len to c + 1 + a; the next
 * anchor token_ids[b*q_len] = argmax[b*q_len + a].  A frozen sequence (slot_mapping[b*q_len] < 0) gets accepted -1,
 * emitted all -1 and keeps its context and anchor.
 *
 * mrs_llama_verify_step: s->batch = B sequences, every row buffer of `s` (token_ids, positions, slot_mapping, x, x2,
 * q, k, v, attn_out, act, logits, out_token, and h on the GEMM route) holds B*q_len rows, tmp_v / tmp_s hold
 * [padded_tiles, q_len*n_heads], attn_counters B*n_kv_heads*ceil(group*q_len/16), argmax_scratch >= 16*B*q_len + 16
 * bytes; the metadata comes from mrs_decode_advance_multi.  Embedding gather of the B*q_len ids -> the decode layer
 * chain with the multi-query fused attention -> lm_head on every row -> mrs_argmax into out_token (must not alias
 * token_ids) -> mrs_spec_accept with `context_lens` (the lengths the advance read; the step struct carries none), all
 * one PDL chain when s->pdl is set.  The linears take the route of mrs_llama_decode_step for the same B, so plain and
 * verify steps of one batch share their numerics:
 *   B 1..8:   the GEMV chain, B*q_len <= 8 rows;
 *   B 9..256: the wgmma dequant-GEMM chain (prefill GEMM numerics) over B*q_len rows, up to 2048; needs `h` and an
 *             f16 / bf16 activation dtype.
 * Graph-capturable.  skip_mask as for decode.  cudaErrorInvalidValue, before any launch, for B outside 1..256, B <= 8
 * with B*q_len > 8, q_len outside 2..8, fused_attention == 0, head_dim other than 64 / 128, tp / all_reduce set,
 * out_token == token_ids, a NULL context_lens / accepted / emitted, (B >= 9) a NULL h or another activation dtype, or
 * the model faults of mrs_llama_decode_step (NULL layers, mismatched w_gate / w_up). */
int32_t mrs_decode_advance_multi(const int32_t *block_tables, int32_t max_blocks_per_seq, int32_t *context_lens,
                                 int32_t batch, int32_t block_size, int32_t split_pages, int32_t padded_tiles,
                                 int32_t *positions, int64_t *slot_mapping, int32_t *kv_indptr, int32_t *kv_indices,
                                 int32_t *kv_last_page_len, int32_t *request_indices, int32_t *kv_tile_indices,
                                 int32_t *o_indptr, int32_t *kv_chunk_size, uint8_t *block_valid_mask,
                                 int32_t max_pos, int32_t *error_flag, int32_t q_len, void *stream);
int32_t mrs_spec_accept(const int32_t *argmax, int32_t *token_ids, const int64_t *slot_mapping, int32_t *context_lens,
                        int32_t *accepted, int32_t *emitted, int32_t batch, int32_t q_len, int32_t pdl, void *stream);
int32_t mrs_llama_verify_step(const mrs_llama_step *s, int32_t q_len, int32_t *context_lens, int32_t *accepted,
                              int32_t *emitted, void *stream);

/* Batched prompt prefill (REF: the scheduler's prompt step, paged_attention/scheduler.rs, run as one model forward over
 * the packed rows of every scheduled sequence; `extract_logits`, pipeline/mod.rs, keeps each sequence's last row for the
 * lm_head): the prompts (or prompt chunks) of n sequences, T rows in all, through the layer stack in one pass.
 *
 * One call's plan and buffers.  Row r of every [T, ...] array is a new token of some sequence; sequence i owns rows
 * cu_seqlens_q[i] .. cu_seqlens_q[i+1] - 1, in order.  All pointers are device pointers unless noted. */
typedef struct {
  int32_t n_seqs;              /* n, 1..256 */
  int32_t total_tokens;        /* T = cu_seqlens_q[n], >= n */
  int32_t max_q_len;           /* max over i of the new rows of sequence i */
  int32_t max_kv_len;          /* max over i of cu_seqlens_k[i+1] - cu_seqlens_k[i] (cached + new rows) */
  int32_t paged;               /* 0: no sequence has cached rows (cu_seqlens_k == cu_seqlens_q): causal attention over the
                                *    fresh q/k/v, then the KV scatter; 1: the scatter first, then the paged prompt
                                *    attention over block_tables (prefix-cache hits, later chunks of a chunked prompt) */
  int32_t lm_rows;             /* 0: no lm_head (a non-final chunk group); 1: each sequence's last row (logits [n, vocab],
                                *    argmax into out_token); 2: every row (logits [T, vocab], no argmax) */
  int32_t block_table_stride;  /* entries per row of block_tables (paged) */
  int32_t num_blocks;          /* blocks in each layer's cache (paged) */
  const int32_t *token_ids;    /* [T] */
  const int32_t *positions;    /* [T] RoPE positions (cached + i for the i-th new row of a sequence) */
  const int64_t *slot_mapping; /* [T] cache slot of each new row (block * block_size + offset) */
  const int32_t *cu_seqlens_q; /* [n + 1] cumulative new rows */
  const int32_t *cu_seqlens_k; /* [n + 1] cumulative cached + new rows */
  const int32_t *block_tables; /* [n, block_table_stride] block ids per sequence (read when paged) */
  const int32_t *last_rows;    /* [n] row of each sequence's last new token (read when lm_rows == 1) */
  /* scratch, activation dtype: x, x2 [T, hidden] residual ping-pong, h [T, hidden] normed activations, q [T, n_heads *
   * head_dim], k, v [T, n_kv_heads * head_dim], attn_out [T, n_heads * head_dim], act [T, inter] */
  void *x, *x2, *h, *q, *k, *v, *attn_out, *act;
  void *gate_up;               /* [2, T, inter]: the separate gate and up GEMM outputs; read only when T > 2048 */
  void *h_last;                /* [n, hidden] the last rows' normed activations (lm_rows == 1) */
  void *logits;                /* [n, vocab] (lm_rows 1) or [T, vocab] (lm_rows 2) */
  int32_t *out_token;          /* [n] argmax of each sequence's logits (lm_rows 1) */
  void *argmax_scratch;        /* zeroed, >= 16 * n + 16 bytes (lm_rows 1); left zeroed */
  void *q8_scratch;            /* >= n * ceil(hidden / 512) * 16 * 36 bytes: the Q8_1 activations of the n <= 8 lm_head */
  /* optional commit into a decode runner's rows (lm_rows == 1 only; NULL dest_rows: no commit) */
  const int32_t *dest_rows;    /* [n] runner row of sequence i */
  int32_t *runner_token_ids;   /* [runner batch] runner_token_ids[dest_rows[i]] = out_token[i] */
  int32_t *runner_context_lens;/* [runner batch] runner_context_lens[dest_rows[i]] = cu_seqlens_k[i+1] - cu_seqlens_k[i] */
} mrs_llama_prefill;

/* Enqueue one prompt step on `stream`: `s` gives weights, norms, per-layer caches, dims, activation dtype, RoPE tables,
 * rope_neox and pdl (its per-step decode metadata and scratch are not read).  Launches:
 *   embedding gather over the T rows -> RMSNorm;
 *   per layer: QKV on the wgmma dequant GEMM (grouped as in the 9..256-sequence decode step: one launch when q, k and v
 *   share a ggml type, q|k + v when attn_v has its own, else three; above 2048 rows always three, where the grouped
 *   form measured slower) -> RoPE at `positions` -> attention (paged 0:
 *   mrs_prefill_attention over cu_seqlens_q, then reshape_and_cache_flashinfer; paged 1: the scatter, then
 *   mrs_prefill_attention_paged) -> o GEMM -> add + RMSNorm -> gate|up GEMM with the SiLU*mul epilogue (above 2048
 *   rows: gate and up GEMMs into gate_up, then fused_glu; bit-identical) -> down GEMM
 *   -> add + RMSNorm with the next layer's norm (the final norm after the last layer);
 *   lm_rows 1: the last rows gathered into h_last, the lm_head on those n rows by the reference's n-row route (n <= 8:
 *   Q8_1 quantiser + MMVQ, as `fast_mmvq` plain; n > 8: the dequant GEMM), mrs_argmax into out_token, then the commit
 *   when dest_rows is set; lm_rows 2: the lm_head GEMM over all T rows.
 * Each row's GEMMs (never split over K) and norms, and each sequence's attention, are computed on their own: a
 * sequence's K/V rows do not depend on the other sequences of the call, nor do its logits for a given n-row route.  The GEMMs and norms are links of a PDL chain when s->pdl
 * is set.  Not graph-capturable in general (T and the max lengths change from call to call).
 * cudaErrorInvalidValue, before any launch, for: n outside 1..256; T < n; a NULL required pointer (the plan arrays,
 * x / x2 / h / q / k / v / attn_out / act; gate_up when T > 2048; block_tables, with block_table_stride and num_blocks >= 1, when paged; last_rows, h_last, logits, out_token,
 * argmax_scratch, and q8_scratch for n <= 8, when lm_rows == 1; logits when lm_rows == 2; runner_token_ids and
 * runner_context_lens when dest_rows is set); an activation dtype other than f16 / bf16; tensor parallelism (s->tp or
 * s->all_reduce set); lm_rows outside 0..2; dest_rows set while lm_rows != 1; paged outside 0..1; a NULL s->layers; a
 * layer whose w_gate and w_up differ in ggml type or rows; (lm_rows == 1, n <= 8) an lm_head type without an MMVQ
 * launcher. */
int32_t mrs_llama_prefill_step(const mrs_llama_step *s, const mrs_llama_prefill *p, void *stream);

/* rows of a quantised table -> activation dtype (embedding gather). ids on device. */
int32_t mrs_embedding_gather(int32_t ggml_type, const void *table, int32_t cols, const int32_t *ids, int32_t n,
                             void *out, int32_t act_dtype, void *stream);
/* out[b] = argmax_v logits[b, v] (first maximum), logits in act dtype */
int32_t mrs_argmax(const void *logits, int32_t rows, int32_t cols, int32_t act_dtype, int32_t *out, void *scratch,
                   int32_t pdl, void *stream);

/* ---- GPTQ / AWQ int4 decode stack (BASELINE config 4: Mistral-7B GPTQ g128, batch 32) --------------
 * Linears are int4 tiles produced by gptq_marlin_repack / awq_marlin_repack (mrs_b200_quant.h) with
 * UNPERMUTED scales [K/group, N] in the activation dtype; q||k||v and gate||up are concatenated along
 * N at load time.  cache_layout 1: HND cache + fused RoPE/KV-write/attention; 0: vLLM layout
 * (K [NB,KVH,D/8,BS,8], V [NB,KVH,D,BS]) through rotary + reshape_and_cache + paged_attention_v1. */
typedef struct { const void *tiles; const void *scales; const void *qzeros; int32_t k, n; } mrs_w4_weight;
typedef struct {
  mrs_w4_weight wqkv, wo, w_gate_up, w_down;
  const void *attn_norm, *ffn_norm;
  void *k_cache, *v_cache;
  /* act-order (GPTQ desc_act) row permutations of the linears, device int32 [K] each, NULL = natural order.  A linear
   * repacked with `perm` (gptq_marlin_repack) holds checkpoint row perm[i] as its row i, so its input must arrive as
   * x[:, perm].  perm_qkv: q, k and v share one (the norm in front of wqkv writes in that order: the first RMSNorm for
   * layer 0, the previous layer's closing add + RMSNorm otherwise); perm_o: the attention output is gathered into
   * attn_perm in that order before the o GEMM; perm_gate_up: gate and up share one (ffn_norm writes in that order).
   * down_proj has no field: a loader permutes the N columns of gate and up by down's permutation instead, so the GLU
   * output arrives in down's order.  The final norm is never permuted. */
  const int32_t *perm_qkv, *perm_o, *perm_gate_up;
} mrs_gptq_layer;
typedef struct {
  int32_t hidden, n_layers, n_heads, n_kv_heads, head_dim, vocab, block_size, act_dtype, group_size;
  float rms_eps, sm_scale;
  int32_t rope_neox, cache_layout, batch, padded_tiles, max_blocks_per_seq, skip_mask;
  const mrs_gptq_layer *layers;            /* host array [n_layers] */
  const void *tok_embd, *lm_head;          /* dense [vocab, hidden] in the activation dtype */
  const void *final_norm, *rope_cos, *rope_sin;
  int32_t *token_ids, *positions; int64_t *slot_mapping;
  int32_t *kv_indptr, *kv_indices, *kv_last_page_len, *request_indices, *kv_tile_indices, *o_indptr, *kv_chunk_size;
  uint8_t *block_valid_mask;
  int32_t *block_tables, *context_lens;    /* dense table + lengths (vLLM-layout attention) */
  void *x, *x2, *h, *qkv, *attn_out, *o, *gate_up, *act, *logits, *tmp_v; float *tmp_s;
  int32_t *out_token, *attn_counters; void *argmax_scratch;
  void *attn_perm;                         /* [rows, n_heads*head_dim] act-order o_proj input, activation dtype; needed
                                            * when any layer sets perm_o (NULL otherwise): rows = batch (decode step),
                                            * batch*q_len (verify step), total_tokens (prompt step) */
} mrs_gptq_step;
/* Act-order layers (a perm_* field set) add launches to the chains below and change no other launch: the RMSNorm or
 * add + RMSNorm in front of wqkv (w_gate_up) is mrs_rms_norm_perm_pdl / mrs_add_rms_norm_perm_pdl with perm_qkv
 * (perm_gate_up), and mrs_gather_cols_pdl(attn_out -> attn_perm, perm_o) runs between the attention and the o GEMM as
 * a link of the same chain.  Every step returns cudaErrorInvalidValue, before any launch, when a layer sets perm_o and
 * attn_perm is NULL, or when a layer sets perm_qkv / perm_gate_up and hidden * 2 bytes exceed 48 KB.
 * skip_mask: bit0 skip rope/cache/attention, bit1 skip the linears (measurement only), bit2 plain stream order instead of
 * the programmatic-dependent-launch chain (HND layout: every launch of the layer loop triggers its dependents at start
 * and waits for the upstream grid before touching its inputs/outputs, so each W4A16 GEMM streams weights while the
 * small kernel before it still runs).
 * mrs_gptq_decode_step: the chain above over s->batch rows, the dense lm_head and mrs_argmax into out_token.
 * cudaErrorInvalidValue, before any launch, for: a NULL s; batch outside 1..256; an activation dtype other than
 * f16 / bf16; hidden % 8 != 0; a NULL s->layers or n_layers < 1; cache_layout outside 0..1; the act-order faults above.
 * The verify step below rejects all of these too, and so does the prompt step, with the plan's n in place of batch. */
int32_t mrs_gptq_decode_step(const mrs_gptq_step *s, void *stream);
/* Batched prompt prefill of a GPTQ / AWQ model: mrs_llama_prefill_step's contract over the int4 layer stack.  `s` gives
 * weights, norms, per-layer caches (in s->cache_layout), dims, activation dtype, group size, RoPE tables and rope_neox;
 * its per-step decode metadata and scratch are not read, and skip_mask bit 2 turns the PDL chain off.  `p` is the plan
 * of mrs_llama_prefill_step, with one difference: p->q is the [T, n_heads*head_dim + 2*n_kv_heads*head_dim] q||k||v
 * buffer of the concatenated wqkv GEMM, and p->k / p->v / p->gate_up / p->q8_scratch are not read.  Launches:
 *   dense embedding gather over the T rows -> RMSNorm;
 *   per layer: qkv W4A16 GEMM -> RoPE at `positions`, strided over qkv -> attention (HND cache, paged 0:
 *   mrs_prefill_attention, then reshape_and_cache_flashinfer; paged 1: the scatter, then mrs_prefill_attention_paged;
 *   vLLM layout: mrs_prefill_attention, then reshape_and_cache) -> o GEMM -> add + RMSNorm -> gate||up GEMM with the GLU
 *   epilogue -> down GEMM -> add + RMSNorm with the next layer's norm (the final norm after the last layer);
 *   lm_rows 1: the last rows gathered into h_last, the dense lm_head on those n rows, mrs_argmax into out_token, then
 *   the commit when dest_rows is set; lm_rows 2: the dense lm_head over all T rows.
 * Every GEMM runs over whole K (`pdl` bit 1 below), so a sequence's K/V rows and logits do not depend on the other
 * sequences of the call.  The GEMMs and norms are links of a PDL chain.  Not graph-capturable in general.
 * cudaErrorInvalidValue, before any launch, for: n outside 1..256; T < n; a NULL required pointer (s->layers, the plan
 * arrays, x / x2 / h / q / attn_out / act; block_tables, with block_table_stride and num_blocks >= 1, when paged;
 * last_rows, h_last, logits, out_token and argmax_scratch when lm_rows == 1; logits when lm_rows == 2;
 * runner_token_ids and runner_context_lens when dest_rows is set); lm_rows outside 0..2; dest_rows set while
 * lm_rows != 1; paged outside 0..1, or paged 1 with the vLLM layout (the paged prompt kernel reads HND pages); an
 * activation dtype other than f16 / bf16; hidden % 8 != 0; n_layers < 1; cache_layout outside 0..1. */
int32_t mrs_gptq_prefill_step(const mrs_gptq_step *s, const mrs_llama_prefill *p, void *stream);
/* Speculative decoding of a GPTQ / AWQ model: mrs_llama_verify_step's contract over the int4 layer stack.  s->batch = B
 * sequences of q_len = k + 1 rows each (the anchor and k drafts); the metadata comes from mrs_decode_advance_multi.
 * Every row buffer of `s` holds B*q_len rows: token_ids, positions, slot_mapping, x, x2, h, qkv, attn_out, o, gate_up,
 * act, logits and out_token (which must not alias token_ids).  tmp_v / tmp_s hold [padded_tiles, q_len*n_heads(,
 * head_dim)], attn_counters B*n_kv_heads*ceil(group*q_len/16) zeroed entries (left zero), argmax_scratch >= 16*B*q_len
 * + 16 zeroed bytes.  Launches: the chain of mrs_gptq_decode_step over the B*q_len rows, with the same W4A16 GEMM
 * flags (so plain and verify steps take one GEMM route), with mrs_paged_decode_fused_multi_strided reading q, k and v
 * inside the q||k||v rows as the attention -> the dense lm_head on every row -> mrs_argmax into out_token ->
 * mrs_spec_accept with `context_lens` (the lengths the advance read).  HND cache layout only: no multi-query kernel
 * reads the vLLM layout.  Graph-capturable; skip_mask as for decode (bit 2 also takes mrs_spec_accept off the PDL
 * chain).  cudaErrorInvalidValue, before any launch, for: B outside 1..256; q_len outside 2..8; cache_layout != 1; a
 * head_dim other than 64 / 128; an activation dtype other than f16 / bf16; hidden % 8 != 0; a NULL s->layers or
 * n_layers < 1; out_token == token_ids; a NULL context_lens, accepted or emitted. */
int32_t mrs_gptq_verify_step(const mrs_gptq_step *s, int32_t q_len, int32_t *context_lens, int32_t *accepted,
                             int32_t *emitted, void *stream);
/* The chain's links (not reference ABI): mrs_w4a16_gemm / mrs_dense_linear / add_rms_norm / fused_split_glu with a
 * `pdl` flag.  pdl bit 0 (value 1) makes the launch a link: it requires that the launch before it on `stream` is also a
 * link (or a plain kernel).  For mrs_w4a16_gemm_pdl and mrs_dense_linear_pdl, bit 1 (value 2) never splits K over a
 * cluster, so row r of Y does not depend on M (without it, token tiles of up to 64 rows may split K, which sums the
 * partials in another order).  For mrs_w4a16_gemm_pdl only, bit 2 (value 4) is the GLU epilogue: w_tiles is gate||up
 * concatenated along N (N = 2I, I % 8 == 0), and y [M, I] = T(silu(T(X gate^T))) * T(X up^T) is written (with bit 1
 * set, bit-identical to the plain whole-K GEMM followed by fused_split_glu); the [M, 2I] product is never stored.  Other bits are invalid. */
int32_t mrs_w4a16_gemm_pdl(const void *x, const void *w_tiles, const void *scales, const int32_t *qzeros, void *y,
                           int32_t M, int32_t K, int32_t N, int32_t group, int32_t dtype, int32_t scale_perm,
                           int32_t pdl, void *stream);
int32_t mrs_dense_linear_pdl(const void *x, const void *w, void *y, int32_t M, int32_t K, int32_t N, int32_t dtype,
                             int32_t pdl, void *stream);
void mrs_add_rms_norm_pdl(const void *x, const void *residual, const void *weight, void *residual_dst, void *norm_dst,
                          int32_t nrows, int32_t ncols, float eps, int32_t dtype, int32_t pdl, void *stream);
void mrs_split_glu_pdl(const void *input, void *output, uint32_t rows, uint32_t split_size, int32_t activation,
                       int32_t dtype, int32_t pdl, void *stream);
/* Norms in front of an act-order linear: the RMSNorm (mrs_rms_norm_f16 / _bf16) and the add + RMSNorm
 * (mrs_add_rms_norm_pdl) with the normed output permuted, norm_dst[r, j] = norm[r, perm[j]] bit for bit, while
 * residual_dst (the rounded sum x + residual) stays in natural order.  perm: device int32 [ncols], a permutation.  x may
 * alias norm_dst (the row is staged in shared memory, so ncols * 2 bytes must not exceed 48 KB).  dtype f16 / bf16; pdl
 * as above, 0 for the plain stream-ordered launch.  cudaErrorInvalidValue for a NULL perm (and, add form, a NULL
 * residual or residual_dst), another dtype, or a row over 48 KB. */
int32_t mrs_rms_norm_perm_pdl(const void *x, const void *weight, const int32_t *perm, void *norm_dst, int32_t nrows,
                              int32_t ncols, float eps, int32_t dtype, int32_t pdl, void *stream);
int32_t mrs_add_rms_norm_perm_pdl(const void *x, const void *residual, const void *weight, const int32_t *perm,
                                  void *residual_dst, void *norm_dst, int32_t nrows, int32_t ncols, float eps, int32_t dtype,
                                  int32_t pdl, void *stream);
/* Column gather of 16-bit rows: y[r, j] = x[r, perm[j]], x and y [rows, cols] contiguous and distinct; pdl as above. */
int32_t mrs_gather_cols_pdl(const void *x, const int32_t *perm, void *y, int32_t rows, int32_t cols, int32_t pdl,
                            void *stream);

#ifdef __cplusplus
}
#endif
#endif
