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
// The decode, verify and prompt steps run this chain (w4_layer_chain) with their own attention.
// mrs_gptq_prefill_step runs it over the packed prompt rows of up to 256 sequences, on whole-K GEMMs with gate||up
// through the GLU epilogue, and the prompt attention of the Llama prompt step (step_common.cuh).
// mrs_gptq_verify_step runs the decode chain over k + 1 rows per sequence (speculative decoding) with the multi-query
// fused attention, then the greedy acceptance on the device.
#include "common.cuh"
#include "mrs_b200_model.h"
#include "mrs_b200_ops.h"
#include "mrs_b200_paged_attn.h"
#include "step_common.cuh"

using namespace mrs;

namespace mrs {
// dense embedding rows: out[b, :] = table[ids[b], :]   (16-bit elements, 16-byte vectors)
__global__ void dense_embedding_kernel(const uint4 *__restrict__ table, int cols8, const int32_t *__restrict__ ids,
                                       uint4 *__restrict__ out) {
  const int64_t row = ids[blockIdx.x];
  for (int i = threadIdx.x; i < cols8; i += blockDim.x) out[(int64_t)blockIdx.x * cols8 + i] = table[row * cols8 + i];
}
}  // namespace mrs

// what every GPTQ step needs of `s`, checked before its first launch (contract: include/mrs_b200_model.h): `batch`
// sequences (the prompt step's n) in 1..256, an f16 / bf16 activation dtype, hidden % 8 == 0, a layer array of at least
// one layer, cache_layout 0 or 1; act-order layers: every layer whose perm_o is set needs the attn_perm scratch, and a
// permuted norm stages a row of `hidden` elements in shared memory
static bool gptq_step_ok(const mrs_gptq_step *s, int batch) {
  if (batch < 1 || batch > 256 || (s->act_dtype != MRS_F16 && s->act_dtype != MRS_BF16) || s->hidden % 8 != 0 ||
      s->layers == nullptr || s->n_layers < 1 || (s->cache_layout != 0 && s->cache_layout != 1))
    return false;
  bool any = false;
  for (int l = 0; l < s->n_layers; l++) {
    const mrs_gptq_layer &L = s->layers[l];
    if (L.perm_o != nullptr && s->attn_perm == nullptr) return false;
    any |= L.perm_qkv != nullptr || L.perm_gate_up != nullptr;
  }
  return !any || (size_t)s->hidden * 2 <= 48 * 1024;
}

// what the callers of the int4 layer chain choose: `rows` rows in every row buffer; whole_k: every W4A16 GEMM runs
// over whole K (flags pdl | 2), so a row's result does not depend on the other rows, and gate||up goes through the GLU
// epilogue (flag 4), which is bit-identical to the GEMM + SiLU*mul launches only over whole K; pdl: the chain's
// programmatic-dependent-launch bit
struct W4Chain {
  const mrs_gptq_step *s;
  int rows;
  bool whole_k;
  int pdl;
  void *stream;
};

// the chain's buffers, of c.rows rows each: qkv [rows, nq + 2 nkv]; o receives the o and down GEMMs (it may be h: the
// add + RMSNorm after them reads it as its input and overwrites it with the norm); gate_up [rows, 2 inter] is read only
// without whole_k
struct W4ChainBufs {
  const int32_t *token_ids;
  void *x, *x2, *h, *qkv, *attn_out, *o, *gate_up, *act;
};

// The int4 layer stack of the decode, verify and prompt steps, up to the final norm in h:
//   dense embedding gather -> RMSNorm (permuted by layers[0].perm_qkv); per layer:
//   qkv GEMM -> attention(L, q, k, v, stride): q, k and v inside the qkv rows, `stride` elements apart, output into
//   attn_out -> (perm_o) column gather into attn_perm -> o GEMM -> add + RMSNorm (x2 = o + x, h = norm, permuted by
//   perm_gate_up) -> gate||up GEMM (+ SiLU*mul) -> down GEMM -> add + RMSNorm (x = down + x2, h = the next layer's
//   norm permuted by its perm_qkv, the final norm after the last layer)
// Every launch after the embedding gather and the first norm is a link of the PDL chain when c.pdl is set.
// do_lin == false skips the linears (decode's skip_mask bit 1).
template <class Attention>
static int32_t w4_layer_chain(const W4Chain &c, const W4ChainBufs &b, bool do_lin, Attention attention) {
  const mrs_gptq_step *s = c.s;
  const int dt = s->act_dtype, H = s->hidden, R = c.rows, pdl = c.pdl;
  const int nq = s->n_heads * s->head_dim, nkv = s->n_kv_heads * s->head_dim, nqkv = nq + 2 * nkv;
  const int flags = c.whole_k ? pdl | 2 : pdl;
  auto linear = [&](const mrs_w4_weight &w, const void *x, void *y, int glu) -> int32_t {
    return mrs_w4a16_gemm_pdl(x, w.tiles, w.scales, (const int32_t *)w.qzeros, y, R, w.k, w.n, s->group_size, dt, 0,
                              flags | glu, c.stream);
  };
  // res_dst = x + res ; h = norm(res_dst), in the row order of the act-order linear after it when perm != NULL
  auto add_rms = [&](const void *x, const void *res, const void *w, void *res_dst, const int32_t *perm) -> int32_t {
    if (perm != nullptr) return mrs_add_rms_norm_perm_pdl(x, res, w, perm, res_dst, b.h, R, H, s->rms_eps, dt, pdl, c.stream);
    mrs_add_rms_norm_pdl(x, res, w, res_dst, b.h, R, H, s->rms_eps, dt, pdl, c.stream);
    return 0;
  };

  mrs::dense_embedding_kernel<<<R, 256, 0, (cudaStream_t)c.stream>>>((const uint4 *)s->tok_embd, H / 8, b.token_ids,
                                                                    (uint4 *)b.x);
  const mrs_gptq_layer &L0 = s->layers[0];
  if (L0.perm_qkv != nullptr)
    MRS_TRY(mrs_rms_norm_perm_pdl(b.x, L0.attn_norm, L0.perm_qkv, b.h, R, H, s->rms_eps, dt, 0, c.stream));
  else if (dt == MRS_F16) mrs_rms_norm_f16(b.x, L0.attn_norm, b.h, R, H, s->rms_eps, (int64_t)c.stream);
  else mrs_rms_norm_bf16(b.x, L0.attn_norm, b.h, R, H, s->rms_eps, (int64_t)c.stream);
  for (int l = 0; l < s->n_layers; l++) {
    const mrs_gptq_layer &L = s->layers[l];
    if (do_lin) MRS_TRY(linear(L.wqkv, b.h, b.qkv, 0));
    MRS_TRY(attention(L, b.qkv, (char *)b.qkv + (size_t)nq * 2, (char *)b.qkv + (size_t)(nq + nkv) * 2, nqkv));
    const void *o_in = b.attn_out;
    if (L.perm_o != nullptr) {                                                // o_proj's rows in act order
      MRS_TRY(mrs_gather_cols_pdl(b.attn_out, L.perm_o, s->attn_perm, R, nq, pdl, c.stream));
      o_in = s->attn_perm;
    }
    if (do_lin) MRS_TRY(linear(L.wo, o_in, b.o, 0));
    MRS_TRY(add_rms(b.o, b.x, L.ffn_norm, b.x2, L.perm_gate_up));            // x2 = o + x ; h = norm(x2)
    if (c.whole_k) {
      if (do_lin) MRS_TRY(linear(L.w_gate_up, b.h, b.act, 4));              // act = silu(gate) * up
    } else {
      if (do_lin) MRS_TRY(linear(L.w_gate_up, b.h, b.gate_up, 0));
      mrs_split_glu_pdl(b.gate_up, b.act, R, L.w_down.k, 0, dt, pdl, c.stream);
    }
    if (do_lin) MRS_TRY(linear(L.w_down, b.act, b.o, 0));
    const bool last = l + 1 == s->n_layers;
    MRS_TRY(add_rms(b.o, b.x2, last ? s->final_norm : s->layers[l + 1].attn_norm, b.x,
                    last ? nullptr : s->layers[l + 1].perm_qkv));           // x = down + x2 ; h = next norm(x)
  }
  return 0;
}

// the decode chain + lm_head + argmax over s->batch sequences of q_len rows each (R = batch * q_len rows in every
// row buffer): q_len == 1 is the decode step, q_len 2..8 a speculative verify step (HND layout only), whose attention is
// the multi-query fused kernel reading q, k and v inside the q||k||v rows
static int32_t gptq_forward(const mrs_gptq_step *s, int q_len, void *stream) {
  const int dt = s->act_dtype, B = s->batch, R = B * q_len;
  cudaStream_t st = (cudaStream_t)stream;
  // Every launch of the layer loop is a link of ONE programmatic-dependent-launch chain (skip_mask bit 2 turns it
  // off): each kernel triggers its dependents when it starts and waits for the upstream grid before touching its
  // inputs / outputs, so the W4A16 GEMMs stream their weights while the small kernels before them still run.
  // The HND attention launch is PDL-capable; the vLLM-layout chain (reference-ABI kernels, no PDL forms) is not,
  // so that layout keeps plain stream order.
  const int pdl = ((s->skip_mask & 4) || s->cache_layout != 1) ? 0 : 1;
  const bool do_attn = !(s->skip_mask & 1), do_lin = !(s->skip_mask & 2);
  auto attention = [&](const mrs_gptq_layer &L, void *q, void *k, void *v, int stride) -> int32_t {
    if (!do_attn) return 0;
    if (s->cache_layout == 1) return fused_decode_attention(s, L.k_cache, L.v_cache, q, k, v, stride, stride, q_len, pdl, stream);
    // vLLM cache layout (REF MISTRALRS_FLASHINFER_DECODE=0): rotary -> reshape_and_cache -> paged_attention_v1
    rotary_embedding_positions(q, k, (void *)s->rope_cos, (void *)s->rope_sin, s->positions, s->rope_neox, s->head_dim, B,
                               s->head_dim / 2, 0, s->n_heads, s->n_kv_heads, stride, stride, (uint32_t)dt, (int64_t)stream);
    reshape_and_cache(k, v, L.k_cache, L.v_cache, s->slot_mapping, B, s->n_kv_heads, s->head_dim, s->block_size, 8, stride,
                      stride, st, (uint32_t)dt, (uint32_t)dt, nullptr, nullptr);
    const int kv_block_stride = s->n_kv_heads * s->head_dim * s->block_size, kv_head_stride = s->head_dim * s->block_size;
    (dt == MRS_F16 ? paged_attention_v1_f16 : paged_attention_v1_bf16)(
        s->attn_out, q, L.k_cache, L.v_cache, nullptr, s->n_kv_heads, s->sm_scale, 1.0f, (uint32_t *)s->block_tables,
        (uint32_t *)s->context_lens, s->block_size, s->max_blocks_per_seq * s->block_size, B, s->n_heads, s->head_dim,
        s->max_blocks_per_seq, stride, kv_block_stride, kv_head_stride, st, (uint32_t)dt, nullptr, nullptr, nullptr);
    return 0;
  };
  MRS_TRY(w4_layer_chain(W4Chain{s, R, false, pdl, stream},
                         W4ChainBufs{s->token_ids, s->x, s->x2, s->h, s->qkv, s->attn_out, s->o, s->gate_up, s->act},
                         do_lin, attention));
  if (do_lin) MRS_TRY(mrs_dense_linear_pdl(s->h, s->lm_head, s->logits, R, s->hidden, s->vocab, dt, pdl, stream));
  MRS_TRY(mrs_argmax(s->logits, R, s->vocab, dt, s->out_token, s->argmax_scratch, 0, stream));
  return (int32_t)cudaGetLastError();
}

extern "C" int32_t mrs_gptq_decode_step(const mrs_gptq_step *s, void *stream) {
  if (s == nullptr || !gptq_step_ok(s, s->batch)) return (int32_t)cudaErrorInvalidValue;
  return gptq_forward(s, 1, stream);
}

// the verify step of speculative decoding (contract: include/mrs_b200_model.h): the decode chain over B * q_len rows,
// then the greedy acceptance on the device, as mrs_llama_verify_step
extern "C" int32_t mrs_gptq_verify_step(const mrs_gptq_step *s, int32_t q_len, int32_t *context_lens, int32_t *accepted,
                                        int32_t *emitted, void *stream) {
  if (s == nullptr || !gptq_step_ok(s, s->batch) || q_len < 2 || q_len > 8 || s->cache_layout != 1 ||
      (s->head_dim != 64 && s->head_dim != 128) || s->out_token == s->token_ids || context_lens == nullptr ||
      accepted == nullptr || emitted == nullptr)
    return (int32_t)cudaErrorInvalidValue;
  MRS_TRY(gptq_forward(s, q_len, stream));
  const int pdl = (s->skip_mask & 4) ? 0 : 1;
  return mrs_spec_accept(s->out_token, s->token_ids, s->slot_mapping, context_lens, accepted, emitted, s->batch, q_len, pdl,
                         stream);
}

// the prompt step over the packed rows of n sequences (contract: include/mrs_b200_model.h): the decode step's layer
// chain over T rows with whole-K GEMMs, gate||up through the GLU epilogue, and the var-len prompt attention
extern "C" int32_t mrs_gptq_prefill_step(const mrs_gptq_step *s, const mrs_llama_prefill *p, void *stream) {
  if (s == nullptr || p == nullptr || !gptq_step_ok(s, p->n_seqs) || !prompt_plan_ok(p, s->act_dtype, s->hidden) ||
      (p->paged && s->cache_layout != 1))
    return (int32_t)cudaErrorInvalidValue;
  const int n = p->n_seqs, T = p->total_tokens, dt = s->act_dtype, H = s->hidden;
  // the attention launches are plain kernels, which a PDL link may follow: the GEMMs and norms are links in both layouts
  const int pdl = (s->skip_mask & 4) ? 0 : 1;
  const PromptAttnModel am{s->n_heads, s->n_kv_heads, s->head_dim, s->block_size, s->rope_neox, dt, s->sm_scale, s->rope_cos,
                           s->rope_sin};
  auto attention = [&](const mrs_gptq_layer &L, void *q, void *k, void *v, int stride) -> int32_t {
    return prompt_attention(p, am, q, k, v, stride, stride, L.k_cache, L.v_cache, s->cache_layout != 1, stream);
  };
  // p->q holds the [T, nqkv] qkv rows; the o and down GEMMs write into h
  MRS_TRY(w4_layer_chain(W4Chain{s, T, true, pdl, stream},
                         W4ChainBufs{p->token_ids, p->x, p->x2, p->h, p->q, p->attn_out, p->h, nullptr, p->act}, true,
                         attention));
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
