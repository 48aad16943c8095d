// decoder.cu — the caller of the hot path: a Llama-family decode layer stack over the kernels in
// this library (see include/mrs_b200_model.h), plus the few glue kernels a token step needs
// (quantised embedding gather, argmax, on-device KV index advance, greedy acceptance of a speculative
// verify step).
//
// REF structure being mirrored: mistralrs-core/src/models/llama.rs:68-135 (attention),
// :243-260 (block), :475-… (model forward); embedding gather over ggml blocks:
// mistralrs-quant/src/gguf/mod.rs:815-845; KV indices: see mrs_decode_advance in the header.
#include "common.cuh"
#include "dequant.cuh"
#include "mrs_b200_model.h"
#include "mrs_b200_ops.h"
#include "mrs_b200_quant.h"
#include "step_common.cuh"

namespace mrs {

__global__ void embedding_gather_kernel(int type, const uint8_t *__restrict__ table, int cols,
                                        const int32_t *__restrict__ ids, void *__restrict__ out, int act_dtype) {
  const int row = ids[blockIdx.x];
  const int be = blk_elems(type), bb = blk_bytes(type);
  const uint8_t *rp = table + (size_t)row * (cols / be) * bb;
  for (int i = threadIdx.x; i < cols; i += blockDim.x)
    store_act(out, (int64_t)blockIdx.x * cols + i, dequant_elem(type, rp + (size_t)(i / be) * bb, i % be), act_dtype);
}

// first-maximum argmax: grid (chunks, rows); each CTA reduces a chunk and folds it into a packed
// 64-bit key (order-preserving float bits << 32 | ~index) with atomicMax; the last CTA of a row
// publishes the index and re-zeroes the scratch (scratch: u64 key[rows] then u32 count[rows]).
__device__ __forceinline__ unsigned long long pack_key(float v, int idx) {
  unsigned int b = __float_as_uint(v);
  b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  return ((unsigned long long)b << 32) | (unsigned int)(0xFFFFFFFFu - (unsigned int)idx);
}
__global__ void argmax_kernel(const void *__restrict__ logits, int cols, int act_dtype, int32_t *__restrict__ out,
                              unsigned long long *__restrict__ keys, unsigned int *__restrict__ counts, int pdl) {
  __shared__ unsigned long long sk[32];
  if (pdl) pdl_wait();
  const int row = blockIdx.y;
  const int64_t base = (int64_t)row * cols;
  unsigned long long best = 0ull;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cols; i += gridDim.x * blockDim.x) {
    const unsigned long long k = pack_key(load_act(logits, base + i, act_dtype), i);
    best = k > best ? k : best;
  }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) {
    const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, m);
    best = o > best ? o : best;
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sk[w] = best;
  __syncthreads();
  if (w == 0) {
    best = (l < (blockDim.x >> 5)) ? sk[l] : 0ull;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, m);
      best = o > best ? o : best;
    }
    if (l == 0) {
      atomicMax(&keys[row], best);
      __threadfence();
      const unsigned int done = atomicAdd(&counts[row], 1u);
      if (done == gridDim.x - 1) {
        __threadfence();
        const unsigned long long k = atomicExch(&keys[row], 0ull);
        out[row] = (int32_t)(0xFFFFFFFFu - (unsigned int)(k & 0xFFFFFFFFull));
        counts[row] = 0u;
      }
    }
  }
}

// dst = T(dst + res) — the residual add after a row-parallel all-reduce
__global__ void add_residual_kernel(void *__restrict__ dst, const void *__restrict__ res, int64_t n, int dt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) store_act(dst, i, load_act(dst, i, dt) + load_act(res, i, dt), dt);
}

// ---- tensor-parallel sum of the row-parallel partials (REF SumAllReduce::sum_all_reduce,
// mistralrs-quant/src/distributed/mod.rs:436-453: ncclAllReduce(sum) in the activation dtype, then the
// residual add of the decoder layer) as ONE small kernel over NVLink peer memory, in the CUDA graph and
// on the PDL chain — a latency-bound 8-16 KB message does not need a collective library:
//   every rank's row-parallel GEMV wrote its partial [count] (activation dtype) into ITS slot buffer;
//   thread 0 publishes "rank r reached all-reduce #seq" into every peer's flag word r (system-scope
//   release), waits until its own flag words show every peer at #seq (acquire), then all threads pull
//   the peers' partials with 16-byte loads (ld.volatile: the same addresses are reused every second
//   all-reduce), sum them in f32 IN RANK ORDER (every rank computes bit-identical sums), round to the
//   dtype like the collective's output, add the residual, round again.
// Two slot buffers alternate: a rank can only overwrite slot s two all-reduces later, after a barrier
// every peer reaches only once it has finished reading s.
struct ArCtxDev {
  int world, rank;
  const uint8_t *peer_base[8];     // peers' symmetric buffers (own included), mapped into this process
  uint32_t *flags_local;           // [world] flag words in the own buffer
  unsigned long long flags_off, slot_off[2];
  uint32_t *seq;                   // [0] device counter of all-reduces done (graph replays continue it); [1] time-out flag
  unsigned long long ll_off, ll_slot_stride, ll_src_stride;   // low-latency region (ll_off == 0: flags + pull)
};
__global__ void __launch_bounds__(1024) tp_allreduce_residual_kernel(const ArCtxDev c, int slot, const void *__restrict__ residual,
                                                                     void *__restrict__ out, int count, int dt, int pdl) {
  __shared__ uint32_t s_seq;
  if (pdl && threadIdx.x == 0) pdl_launch_dependents();
  if (pdl) pdl_wait();                       // the own partial is complete and flushed
  if (threadIdx.x == 0) {
    const uint32_t seq = *c.seq + 1u;
    *c.seq = seq;
    __threadfence_system();
    for (int r = 0; r < c.world; r++) {
      uint32_t *flag = (uint32_t *)(c.peer_base[r] + c.flags_off) + c.rank;
      asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(seq) : "memory");
    }
    for (int r = 0; r < c.world; r++) {
      uint32_t v;
      do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(c.flags_local + r) : "memory");
      } while ((int32_t)(v - seq) < 0);
    }
    s_seq = seq;
  }
  __syncthreads();
  for (int i = threadIdx.x * 8; i < count; i += blockDim.x * 8) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int r = 0; r < c.world; r++) {
      const uint4 raw = __ldcv((const uint4 *)(c.peer_base[r] + c.slot_off[slot]) + (i >> 3));
      float v[8];
      unpack_act8(raw, dt, v);
#pragma unroll
      for (int k = 0; k < 8; k++) acc[k] += v[k];
    }
    float res[8];
    load_act8(residual, i, dt, res);
#pragma unroll
    for (int k = 0; k < 8; k++) store_act(out, (int64_t)i + k, round_act(acc[k], dt) + res[k], dt);
  }
}

// Low-latency form (NCCL's "LL" idea on our own buffers): the partial travels as 8-byte words {two activation elements,
// sequence number}.  An 8-byte store is delivered whole, so the receiver needs no flag and no fence — it polls the word
// until the sequence number is the current one.  One NVLink store hop instead of flag round trip + pull round trip.
// Thread t owns element pairs t, t + blockDim, ...: reads its own partial (local), pushes it to every peer, then collects
// the peers' words from its own region, sums in rank order in f32, rounds, adds the residual.  Two slots alternate, the
// sequence number grows monotonically: a word of the all-reduce two steps back can never be mistaken for the current one,
// and a rank can only overwrite slot s after every peer has sent it the all-reduce in between, i.e. finished reading s.
__global__ void __launch_bounds__(1024) tp_allreduce_ll_kernel(const ArCtxDev c, int slot, const void *__restrict__ partial,
                                                               const void *__restrict__ residual, void *__restrict__ out, int count,
                                                               int dt, int pdl) {
  if (pdl && threadIdx.x == 0) pdl_launch_dependents();
  if (pdl) pdl_wait();                       // the own partial is complete and flushed
  const uint32_t seq = *(volatile const uint32_t *)c.seq + 1u;
  const bool dead = *(volatile const uint32_t *)(c.seq + 1) != 0u;   // an earlier all-reduce gave up on a peer: never wait again
  __syncthreads();
  if (threadIdx.x == 0) *(volatile uint32_t *)c.seq = seq;
  const unsigned long long area = c.ll_off + (unsigned long long)slot * c.ll_slot_stride;
  const int npairs = count >> 1;
  for (int i = threadIdx.x; i < npairs; i += blockDim.x) {
    const uint32_t mine = ((const uint32_t *)partial)[i];
    for (int r = 0; r < c.world; r++) {
      if (r == c.rank) continue;
      uint2 *dst = (uint2 *)(c.peer_base[r] + area + (unsigned long long)c.rank * c.ll_src_stride) + i;
      asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(dst), "r"(mine), "r"(seq) : "memory");
    }
  }
  for (int i = threadIdx.x; i < npairs; i += blockDim.x) {
    const uint32_t mine = ((const uint32_t *)partial)[i];
    float a0 = 0.f, a1 = 0.f;
    for (int r = 0; r < c.world; r++) {
      uint32_t w = mine;
      if (r != c.rank) {
        const uint2 *src = (const uint2 *)(c.peer_base[c.rank] + area + (unsigned long long)r * c.ll_src_stride) + i;
        // bounded wait: a peer that never shows up (ranks out of step) must not hang the GPU — after ~0.25 s the
        // kernel gives up on the word, raises the flag next to the sequence counter and carries on with stale data
        uint32_t fl, spins = 0;
        const long long t0 = clock64();
        for (;;) {
          asm volatile("ld.volatile.global.v2.u32 {%0, %1}, [%2];" : "=r"(w), "=r"(fl) : "l"(src) : "memory");
          if (fl == seq || dead) break;
          if ((++spins & 1023u) == 0u &&
              (clock64() - t0 > 500000000ll || *(volatile const uint32_t *)(c.seq + 1) != 0u)) { c.seq[1] = 1u; break; }
        }
      }
      float v0, v1;
      if (dt == MRS_BF16) { const float2 f = __bfloat1622float2(*(const __nv_bfloat162 *)&w); v0 = f.x; v1 = f.y; }
      else { const float2 f = __half22float2(*(const __half2 *)&w); v0 = f.x; v1 = f.y; }
      a0 += v0; a1 += v1;
    }
    const float r0 = load_act(residual, 2 * (int64_t)i, dt), r1 = load_act(residual, 2 * (int64_t)i + 1, dt);
    store_act(out, 2 * (int64_t)i, round_act(a0, dt) + r0, dt);
    store_act(out, 2 * (int64_t)i + 1, round_act(a1, dt) + r1, dt);
  }
}

// one CTA: integers only, must match the host producers.  Thread b owns sequence b (lengths, slot,
// chunk count), thread 0 turns the per-sequence counts into the two prefix sums, then all threads
// fill the tile list and the page indices.  A sequence that has used up its block table or the RoPE
// table (pos >= min(max_blocks*bs, max_pos)) is frozen: its context does not grow, its KV write is
// skipped (slot -1, the reference's _PAD_SLOT_ID) and *error_flag gets bit 0 — generation past the
// allocated context must never turn into an out-of-bounds cache write.
// q > 1 (speculative verify): sequence b processes q rows at positions c .. c + q - 1 (rows b * q + i of positions /
// slot_mapping) and its context becomes c + q.  A sequence with c + q > cap is frozen whole: every slot is -1 and its
// context_lens entry keeps c (the acceptance kernel recognises it by slot -1 and leaves it there); its attention
// still runs over the last q table positions, whose rows are never written.  Requires cap >= q.
constexpr int ADV_MAX_BATCH = 256;
__global__ void decode_advance_kernel(const int32_t *__restrict__ block_tables, int max_blocks,
                                      int32_t *__restrict__ context_lens, int batch, int bs, int split_pages,
                                      int padded_tiles, int max_pos, int32_t *positions, int64_t *slot_mapping,
                                      int32_t *kv_indptr, int32_t *kv_indices, int32_t *kv_last_page_len,
                                      int32_t *request_indices, int32_t *kv_tile_indices, int32_t *o_indptr,
                                      int32_t *kv_chunk_size, uint8_t *block_valid_mask, int32_t *error_flag, int q) {
  __shared__ int s_nb[ADV_MAX_BATCH], s_chunks[ADV_MAX_BATCH], s_indptr[ADV_MAX_BATCH + 1], s_oind[ADV_MAX_BATCH + 1];
  const int cap = min(max_blocks * bs, max_pos > 0 ? max_pos : max_blocks * bs);
  for (int b = threadIdx.x; b < batch; b += blockDim.x) {
    const int c = context_lens[b];         // position of the (first) token being processed now
    const bool full = c + q > cap;
    if (full && error_flag != nullptr) atomicOr(error_flag, 1);
    const int ctx = full ? cap : c + q;    // context length including the processed tokens
    context_lens[b] = (full && q > 1) ? c : ctx;
    for (int i = 0; i < q; i++) {
      const int pos = ctx - q + i;
      positions[b * q + i] = pos;
      slot_mapping[b * q + i] = full ? (int64_t)-1 : (int64_t)block_tables[(int64_t)b * max_blocks + pos / bs] * bs + pos % bs;
    }
    const int nb = (ctx + bs - 1) / bs;
    s_nb[b] = nb;
    kv_last_page_len[b] = ctx - (nb - 1) * bs;
    s_chunks[b] = (split_pages > 0) ? ((nb < 1 ? 1 : nb) + split_pages - 1) / split_pages : 1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int nnz = 0, tiles = 0;
    s_indptr[0] = 0; s_oind[0] = 0;
    for (int b = 0; b < batch; b++) {
      nnz += s_nb[b];
      tiles = min(tiles + s_chunks[b], padded_tiles);
      s_indptr[b + 1] = nnz; s_oind[b + 1] = tiles;
    }
    kv_chunk_size[0] = (split_pages > 0 ? split_pages : 1) * bs;
  }
  __syncthreads();
  const int tiles = s_oind[batch];
  for (int b = threadIdx.x; b <= batch; b += blockDim.x) { kv_indptr[b] = s_indptr[b]; o_indptr[b] = s_oind[b]; }
  for (int b = 0; b < batch; b++) {
    const int t0 = s_oind[b], nt = s_oind[b + 1] - t0;
    for (int t = threadIdx.x; t < nt; t += blockDim.x) { request_indices[t0 + t] = b; kv_tile_indices[t0 + t] = t; }
    // page indices: parallel over (b, i)
    const int p0 = s_indptr[b], nb = s_indptr[b + 1] - p0;
    for (int i = threadIdx.x; i < nb; i += blockDim.x) kv_indices[p0 + i] = block_tables[(int64_t)b * max_blocks + i];
  }
  for (int t = threadIdx.x; t < padded_tiles; t += blockDim.x) {
    block_valid_mask[t] = t < tiles ? 1 : 0;
    if (t >= tiles) { request_indices[t] = 0; kv_tile_indices[t] = 0; }
  }
}

// greedy acceptance of a verify step (REF mistralrs-core/src/speculative/verifier.rs:198-291, top-1 rule): sequence b
// fed rows [anchor, draft 1 .. k] (token_ids[b * q ..]) and argmax[b * q + i] is the target's choice after row i.
// Drafts are accepted while draft i + 1 == argmax[i]; a accepted drafts emit argmax[0 .. a] (a + 1 tokens), the
// context keeps the anchor and the accepted drafts (c + 1 + a, the reference's keep_len) and argmax[a] is the next
// anchor.  A sequence the advance froze (slot -1) emits nothing: accepted -1, emitted all -1, context unchanged.
__global__ void spec_accept_kernel(const int32_t *__restrict__ argmax, int32_t *__restrict__ token_ids,
                                   const int64_t *__restrict__ slot_mapping, int32_t *__restrict__ context_lens,
                                   int32_t *__restrict__ accepted, int32_t *__restrict__ emitted, int batch, int q, int pdl) {
  if (pdl) pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const int32_t *am = argmax + (int64_t)b * q;
  int32_t *row = token_ids + (int64_t)b * q, *em = emitted + (int64_t)b * q;
  if (slot_mapping[(int64_t)b * q] < 0) {
    accepted[b] = -1;
    for (int i = 0; i < q; i++) em[i] = -1;
    return;
  }
  int a = 0;
  while (a < q - 1 && row[a + 1] == am[a]) a++;
  for (int i = 0; i < q; i++) em[i] = (i <= a) ? am[i] : -1;
  accepted[b] = a;
  context_lens[b] += 1 + a - q;            // the advance left c + q
  row[0] = am[a];
}

// prompt step: h_last[i] = h[last_rows[i]] (the reference's extract_logits: only each sequence's last row goes through
// the lm_head).  Grid n, 16-byte copies (hidden * 2 bytes is a multiple of 16).
__global__ void last_row_gather_kernel(const uint4 *__restrict__ h, const int32_t *__restrict__ last_rows,
                                       uint4 *__restrict__ h_last, int row_vecs) {
  const int64_t src = (int64_t)last_rows[blockIdx.x] * row_vecs, dst = (int64_t)blockIdx.x * row_vecs;
  for (int i = threadIdx.x; i < row_vecs; i += blockDim.x) h_last[dst + i] = h[src + i];
}

// prompt step hand-off to a decode runner: row dest_rows[i] continues sequence i from its first sampled token, at the
// context length the prompt step left in the cache
__global__ void prefill_commit_kernel(const int32_t *__restrict__ out_token, const int32_t *__restrict__ cu_k,
                                      const int32_t *__restrict__ dest_rows, int32_t *__restrict__ token_ids,
                                      int32_t *__restrict__ context_lens, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = dest_rows[i];
  token_ids[r] = out_token[i];
  context_lens[r] = cu_k[i + 1] - cu_k[i];
}

// ---- the prompt-step parts shared with the GPTQ prompt step (step_common.cuh)
bool prompt_plan_ok(const mrs_llama_prefill *p, int act_dtype, int hidden) {
  const int n = p->n_seqs;
  if (n < 1 || n > 256 || p->total_tokens < n || (act_dtype != MRS_F16 && act_dtype != MRS_BF16) || p->lm_rows < 0 ||
      p->lm_rows > 2 || (p->paged != 0 && p->paged != 1) || (p->dest_rows != nullptr && p->lm_rows != 1) ||
      p->max_q_len < 1 || p->max_kv_len < p->max_q_len || hidden % 8 != 0)
    return false;
  if (p->token_ids == nullptr || p->positions == nullptr || p->slot_mapping == nullptr || p->cu_seqlens_q == nullptr ||
      p->cu_seqlens_k == nullptr || p->x == nullptr || p->x2 == nullptr || p->h == nullptr || p->q == nullptr ||
      p->attn_out == nullptr || p->act == nullptr)
    return false;
  if (p->paged && (p->block_tables == nullptr || p->block_table_stride < 1 || p->num_blocks < 1)) return false;
  if (p->lm_rows == 1 && (p->last_rows == nullptr || p->h_last == nullptr || p->logits == nullptr || p->out_token == nullptr ||
                          p->argmax_scratch == nullptr))
    return false;
  if (p->lm_rows == 2 && p->logits == nullptr) return false;
  return p->dest_rows == nullptr || (p->runner_token_ids != nullptr && p->runner_context_lens != nullptr);
}

int32_t prompt_attention(const mrs_llama_prefill *p, const PromptAttnModel &m, void *q, void *k, void *v, int64_t q_stride,
                         int64_t kv_stride, void *k_cache, void *v_cache, bool vllm_cache, void *stream) {
  const int n = p->n_seqs, T = p->total_tokens, dt = m.act_dtype, nq = m.n_heads * m.head_dim;
  cudaStream_t st = (cudaStream_t)stream;
  rotary_embedding_positions(q, k, (void *)m.rope_cos, (void *)m.rope_sin, (void *)p->positions, m.rope_neox, m.head_dim, T,
                             m.head_dim / 2, 0, m.n_heads, m.n_kv_heads, q_stride, kv_stride, (uint32_t)dt, (int64_t)stream);
  auto scatter = [&] {
    if (vllm_cache)
      reshape_and_cache(k, v, k_cache, v_cache, (int64_t *)p->slot_mapping, T, m.n_kv_heads, m.head_dim, m.block_size, 8,
                        (int32_t)kv_stride, (int32_t)kv_stride, st, (uint32_t)dt, (uint32_t)dt, nullptr, nullptr);
    else
      reshape_and_cache_flashinfer(k, v, k_cache, v_cache, (int64_t *)p->slot_mapping, T, m.n_kv_heads, m.head_dim,
                                   m.block_size, (int32_t)kv_stride, (int32_t)kv_stride, 1.f, 1.f, (uint32_t)dt, (uint32_t)dt, st);
  };
  if (!p->paged) {   // every key is new: attend over the fresh rows, then write them to the cache
    MRS_TRY(mrs_prefill_attention(q, k, v, p->attn_out, p->cu_seqlens_q, n, T, p->max_q_len, m.n_heads, m.n_kv_heads,
                                  m.head_dim, q_stride, kv_stride, nq, m.sm_scale, 1, -1, 0.f, (uint32_t)dt, stream));
    scatter();
    return 0;
  }
  if (vllm_cache) return (int32_t)cudaErrorInvalidValue;
  // the new rows join the cached ones in the cache, then attend over the pages
  scatter();
  return mrs_prefill_attention_paged(q, k_cache, v_cache, p->attn_out, p->block_tables, p->block_table_stride, p->cu_seqlens_q,
                                     p->cu_seqlens_k, n, T, p->max_q_len, p->max_kv_len, p->num_blocks, m.n_heads,
                                     m.n_kv_heads, m.head_dim, m.block_size, q_stride, nq, m.sm_scale, 1, -1, 0.f, (uint32_t)dt,
                                     stream);
}

void prompt_gather_last_rows(const mrs_llama_prefill *p, const void *h, int hidden, void *stream) {
  last_row_gather_kernel<<<p->n_seqs, 128, 0, (cudaStream_t)stream>>>((const uint4 *)h, p->last_rows, (uint4 *)p->h_last,
                                                                      hidden / 8);
}

void prompt_commit(const mrs_llama_prefill *p, void *stream) {
  prefill_commit_kernel<<<(p->n_seqs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      p->out_token, p->cu_seqlens_k, p->dest_rows, p->runner_token_ids, p->runner_context_lens, p->n_seqs);
}

}  // namespace mrs

using namespace mrs;

extern "C" int32_t mrs_embedding_gather(int32_t ggml_type, const void *table, int32_t cols, const int32_t *ids,
                                        int32_t n, void *out, int32_t act_dtype, void *stream) {
  if (n <= 0) return 0;
  if (blk_bytes(ggml_type) == 0 || cols % blk_elems(ggml_type)) return (int32_t)cudaErrorInvalidValue;
  embedding_gather_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(ggml_type, (const uint8_t *)table, cols, ids, out, act_dtype);
  return (int32_t)cudaGetLastError();
}

extern "C" int32_t mrs_argmax(const void *logits, int32_t rows, int32_t cols, int32_t act_dtype, int32_t *out,
                              void *scratch, int32_t pdl, void *stream) {
  if (rows <= 0) return 0;
  if (scratch == nullptr) return (int32_t)cudaErrorInvalidValue;
  unsigned long long *keys = (unsigned long long *)scratch;
  unsigned int *counts = (unsigned int *)(keys + rows);
  int chunks = (cols + 4095) / 4096;
  if (chunks > 64) chunks = 64;
  return (int32_t)launch_pdl(argmax_kernel, dim3(chunks, rows), dim3(256), 0, (cudaStream_t)stream, pdl, logits, (int)cols,
                             (int)act_dtype, out, keys, counts, (int)pdl);
}

extern "C" int32_t mrs_decode_advance(const int32_t *block_tables, int32_t max_blocks_per_seq, int32_t *context_lens,
                                      int32_t batch, int32_t block_size, int32_t split_pages, int32_t padded_tiles,
                                      int32_t *positions, int64_t *slot_mapping, int32_t *kv_indptr,
                                      int32_t *kv_indices, int32_t *kv_last_page_len, int32_t *request_indices,
                                      int32_t *kv_tile_indices, int32_t *o_indptr, int32_t *kv_chunk_size,
                                      uint8_t *block_valid_mask, int32_t max_pos, int32_t *error_flag, void *stream) {
  return mrs_decode_advance_multi(block_tables, max_blocks_per_seq, context_lens, batch, block_size, split_pages, padded_tiles,
                                  positions, slot_mapping, kv_indptr, kv_indices, kv_last_page_len, request_indices,
                                  kv_tile_indices, o_indptr, kv_chunk_size, block_valid_mask, max_pos, error_flag, 1, stream);
}

extern "C" int32_t mrs_decode_advance_multi(const int32_t *block_tables, int32_t max_blocks_per_seq, int32_t *context_lens,
                                            int32_t batch, int32_t block_size, int32_t split_pages, int32_t padded_tiles,
                                            int32_t *positions, int64_t *slot_mapping, int32_t *kv_indptr,
                                            int32_t *kv_indices, int32_t *kv_last_page_len, int32_t *request_indices,
                                            int32_t *kv_tile_indices, int32_t *o_indptr, int32_t *kv_chunk_size,
                                            uint8_t *block_valid_mask, int32_t max_pos, int32_t *error_flag, int32_t q_len,
                                            void *stream) {
  if (batch < 1 || batch > ADV_MAX_BATCH || max_blocks_per_seq < 1 || block_size < 1 || q_len < 1 || q_len > 8)
    return (int32_t)cudaErrorInvalidValue;
  const int cap = max_pos > 0 && max_pos < max_blocks_per_seq * block_size ? max_pos : max_blocks_per_seq * block_size;
  if (cap < q_len) return (int32_t)cudaErrorInvalidValue;
  decode_advance_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(block_tables, max_blocks_per_seq, context_lens, batch,
                                                             block_size, split_pages, padded_tiles, max_pos, positions,
                                                             slot_mapping, kv_indptr, kv_indices, kv_last_page_len,
                                                             request_indices, kv_tile_indices, o_indptr, kv_chunk_size,
                                                             block_valid_mask, error_flag, q_len);
  return (int32_t)cudaGetLastError();
}

extern "C" int32_t mrs_spec_accept(const int32_t *argmax, int32_t *token_ids, const int64_t *slot_mapping,
                                   int32_t *context_lens, int32_t *accepted, int32_t *emitted, int32_t batch, int32_t q_len,
                                   int32_t pdl, void *stream) {
  if (batch < 1 || q_len < 1) return (int32_t)cudaErrorInvalidValue;
  return (int32_t)launch_pdl(spec_accept_kernel, dim3((batch + 127) / 128), dim3(128), 0, (cudaStream_t)stream, pdl, argmax,
                             token_ids, slot_mapping, context_lens, accepted, emitted, (int)batch, (int)q_len, (int)pdl);
}

extern "C" int32_t mrs_tp_allreduce_residual(const mrs_tp_ctx *ctx, int32_t slot, const void *residual, void *out,
                                             int32_t count, int32_t dtype, int32_t pdl, void *stream) {
  if (ctx == nullptr || ctx->world < 1 || ctx->world > 8 || (slot & ~1) || count % 8 || (dtype != MRS_F16 && dtype != MRS_BF16))
    return (int32_t)cudaErrorInvalidValue;
  ArCtxDev c = {};
  c.world = ctx->world; c.rank = ctx->rank;
  for (int r = 0; r < ctx->world; r++) c.peer_base[r] = (const uint8_t *)ctx->peer_base[r];
  c.flags_off = (unsigned long long)ctx->flags_offset;
  c.slot_off[0] = (unsigned long long)ctx->slot_offset[0]; c.slot_off[1] = (unsigned long long)ctx->slot_offset[1];
  c.flags_local = (uint32_t *)((uint8_t *)ctx->peer_base[ctx->rank] + ctx->flags_offset);
  c.seq = (uint32_t *)ctx->seq_counter;
  c.ll_off = (unsigned long long)ctx->ll_offset; c.ll_slot_stride = (unsigned long long)ctx->ll_slot_stride;
  c.ll_src_stride = (unsigned long long)ctx->ll_src_stride;
  if (ctx->ll_offset != 0) {
    if ((int64_t)count * 4 > ctx->ll_src_stride) return (int32_t)cudaErrorInvalidValue;
    int th = (count / 2 + 31) / 32 * 32;
    if (th > 1024) th = 1024;
    // the partial of this rank: its slot in the symmetric buffer (what the row-parallel GEMV wrote)
    const void *partial = (const uint8_t *)ctx->peer_base[ctx->rank] + ctx->slot_offset[slot];
    return (int32_t)launch_pdl(tp_allreduce_ll_kernel, dim3(1), dim3(th), 0, (cudaStream_t)stream, pdl, c, (int)slot, partial,
                               residual, out, (int)count, (int)dtype, (int)pdl);
  }
  int threads = (count / 8 + 31) / 32 * 32;
  if (threads > 1024) threads = 1024;
  if (threads < 32) threads = 32;
  return (int32_t)launch_pdl(tp_allreduce_residual_kernel, dim3(1), dim3(threads), 0, (cudaStream_t)stream, pdl, c, (int)slot,
                             residual, out, (int)count, (int)dtype, (int)pdl);
}

// cudaErrorInvalidValue for a model the layer chains cannot run, checked before a step's first launch: a NULL layer
// array, or a layer whose gate and up differ in ggml type or rows (every route runs them as one gate|up launch)
static int32_t check_model(const mrs_llama_step *s) {
  if (s->n_layers >= 1 && s->layers == nullptr) return (int32_t)cudaErrorInvalidValue;
  for (int l = 0; l < s->n_layers; l++) {
    const mrs_llama_layer &L = s->layers[l];
    if (L.w_gate.ggml_type != L.w_up.ggml_type || L.w_gate.rows != L.w_up.rows) return (int32_t)cudaErrorInvalidValue;
  }
  return 0;
}

// the decode attention of layer L over s->batch sequences of q_len rows each: the fused kernel (multi-query for a verify
// step, q_len > 1), or with fused_attention == 0 the RoPE -> KV scatter -> paged decode chain
static int32_t decode_attention(const mrs_llama_step *s, const mrs_llama_layer &L, int q_len, void *stream) {
  const int B = s->batch, dt = s->act_dtype, nq = s->n_heads * s->head_dim, nkv = s->n_kv_heads * s->head_dim;
  if (q_len > 1 || s->fused_attention)
    return fused_decode_attention(s, L.k_cache, L.v_cache, s->q, s->k, s->v, nq, nkv, q_len, s->pdl, stream);
  void *tmp_v = s->padded_tiles > B ? s->tmp_v : nullptr;
  float *tmp_s = s->padded_tiles > B ? s->tmp_s : nullptr;
  rotary_embedding_positions(s->q, s->k, (void *)s->rope_cos, (void *)s->rope_sin, s->positions, s->rope_neox, s->head_dim,
                             B, s->head_dim / 2, 0, s->n_heads, s->n_kv_heads, nq, nkv, (uint32_t)dt, (int64_t)stream);
  reshape_and_cache_flashinfer(s->k, s->v, L.k_cache, L.v_cache, s->slot_mapping, B, s->n_kv_heads, s->head_dim,
                               s->block_size, nkv, nkv, 1.f, 1.f, (uint32_t)dt, (uint32_t)dt, (cudaStream_t)stream);
  return flashinfer_decode(s->q, L.k_cache, L.v_cache, s->kv_indptr, s->kv_indices, s->kv_last_page_len, s->request_indices,
                           s->kv_tile_indices, s->o_indptr, s->kv_chunk_size, (const bool *)s->block_valid_mask, s->attn_out,
                           tmp_v, tmp_s, B, s->padded_tiles, s->n_heads, s->n_kv_heads, s->head_dim, s->block_size, nq,
                           s->head_dim, s->sm_scale, -1, 0.f, 1.f, 1.f, (uint32_t)dt, (uint32_t)dt, (cudaStream_t)stream);
}

// the GEMV chain (batch 1..8): the layer stack + lm_head + argmax over batch * q_len token rows; q_len > 1 is a
// speculative verify step, q_len == 1 the decode step
static int32_t llama_forward(const mrs_llama_step *s, int q_len, void *stream) {
  if (const int32_t e = check_model(s)) return e;
  const int dt = s->act_dtype, B = s->batch * q_len, H = s->hidden, pdl = s->pdl;
  const int nq = s->n_heads * s->head_dim, nkv = s->n_kv_heads * s->head_dim;
  const bool do_attn = !(s->skip_mask & 1), do_gemv = !(s->skip_mask & 2);
  const mrs_tp_ctx *tp = (s->tp != nullptr && s->tp->world > 1) ? s->tp : nullptr;
  // a row-parallel projection: dst = residual + W x.  Single GPU: the GEMV's residual epilogue.  Tensor parallel: the
  // partial sums of every rank summed, then the residual added: the peer-memory sum (one kernel on the PDL chain, the
  // partial in this rank's slot buffer), or the all_reduce callback and add_residual_kernel (REF
  // distributed/layers.rs:965-975)
  auto row_parallel = [&](const mrs_qweight &W, int mode, const void *x, int K, const void *residual, void *dst,
                          int slot) -> int32_t {
    if (tp != nullptr) {
      void *part = (uint8_t *)tp->peer_base[tp->rank] + tp->slot_offset[slot];
      MRS_TRY(mrs_mmvq_fused(W.ggml_type, mode, dt, W.data, nullptr, nullptr, x, nullptr, 0.f, nullptr, part, nullptr,
                             nullptr, K, H, 0, 0, B, 0, pdl, stream));
      return mrs_tp_allreduce_residual(tp, slot, residual, dst, B * H, dt, pdl, stream);
    }
    MRS_TRY(mrs_mmvq_fused(W.ggml_type, mode, dt, W.data, nullptr, nullptr, x, nullptr, 0.f,
                           s->all_reduce == nullptr ? residual : nullptr, dst, nullptr, nullptr, K, H, 0, 0, B, 0, pdl, stream));
    if (s->all_reduce != nullptr) {
      s->all_reduce(dst, (int64_t)B * H, dt, stream, s->all_reduce_user);
      add_residual_kernel<<<(unsigned)(((int64_t)B * H + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dst, residual,
                                                                                                    (int64_t)B * H, dt);
    }
    return 0;
  };

  MRS_TRY(mrs_embedding_gather(s->tok_embd.ggml_type, s->tok_embd.data, H, s->token_ids, B, s->x, dt, stream));
  void *hidden = s->x, *hidden2 = s->x2;
  for (int l = 0; l < s->n_layers; l++) {
    const mrs_llama_layer &L = s->layers[l];
    // --- attention block: x = x + o_proj(attn(rope(qkv(norm(x)))))
    // the fused launches decode every matrix of a group with ONE ggml type: per-tensor type
    // overrides (GGUF --tensor-type, per-layer UQFF topologies) take separate launches
    if (!do_gemv) {
    } else if (L.wq.ggml_type != L.wk.ggml_type) {
      MRS_TRY(mrs_mmvq_fused(L.wq.ggml_type, 0, dt, L.wq.data, nullptr, nullptr, hidden, L.attn_norm, s->rms_eps,
                             nullptr, s->q, nullptr, nullptr, H, nq, 0, 0, B, 0, pdl, stream));
      MRS_TRY(mrs_mmvq_fused(L.wk.ggml_type, 0, dt, L.wk.data, nullptr, nullptr, hidden, L.attn_norm, s->rms_eps,
                             nullptr, s->k, nullptr, nullptr, H, nkv, 0, 0, B, 0, pdl, stream));
      MRS_TRY(mrs_mmvq_fused(L.wv.ggml_type, 0, dt, L.wv.data, nullptr, nullptr, hidden, L.attn_norm, s->rms_eps,
                             nullptr, s->v, nullptr, nullptr, H, nkv, 0, 0, B, 0, pdl, stream));
    } else if (L.wk.ggml_type == L.wv.ggml_type) {
      MRS_TRY(mrs_mmvq_fused(L.wq.ggml_type, 2, dt, L.wq.data, L.wk.data, L.wv.data, hidden, L.attn_norm, s->rms_eps,
                             nullptr, s->q, s->k, s->v, H, nq, nkv, nkv, B, 0, pdl, stream));
    } else {
      MRS_TRY(mrs_mmvq_fused_qkv_mixed(L.wq.ggml_type, L.wv.ggml_type, dt, L.wq.data, L.wk.data, L.wv.data, hidden,
                                       L.attn_norm, s->rms_eps, s->q, s->k, s->v, H, nq, nkv, nkv, B, pdl, stream));
    }
    if (do_attn) MRS_TRY(decode_attention(s, L, q_len, stream));
    if (!do_gemv) continue;
    MRS_TRY(row_parallel(L.wo, 0, s->attn_out, nq, hidden, hidden2, 0));
    // --- MLP block: x = x + down(silu(gate(norm(x))) * up(norm(x)))
    // the GLU epilogue writes act in its Q8_1 form (block_q8_1 [B][rows / 32], inside act's B x rows activation-dtype
    // bytes), the form down_proj consumes: quantised once, not again by every CTA of down_proj
    const int q8 = (L.w_gate.rows % 32 == 0) ? 1 : 0;
    MRS_TRY(mrs_mmvq_fused(L.w_gate.ggml_type, 1 | (q8 ? 8 : 0), dt, L.w_gate.data, L.w_up.data, nullptr, hidden2, L.ffn_norm,
                           s->rms_eps, nullptr, s->act, nullptr, nullptr, H, L.w_gate.rows, L.w_gate.rows, 0, B, 0,
                           pdl, stream));
    MRS_TRY(row_parallel(L.w_down, q8 ? 4 : 0, s->act, L.w_down.cols, hidden2, hidden, 1));
  }
  if (do_gemv)
  MRS_TRY(mrs_mmvq_fused(s->lm_head.ggml_type, 0, dt, s->lm_head.data, nullptr, nullptr, hidden, s->final_norm,
                         s->rms_eps, nullptr, s->logits, nullptr, nullptr, H, s->vocab, 0, 0, B, 0, pdl, stream));
  MRS_TRY(mrs_argmax(s->logits, B, s->vocab, dt, s->out_token, s->argmax_scratch, pdl, stream));
  return (int32_t)cudaGetLastError();
}

// Above this many rows the GEMM layer chain runs q, k and v as separate GEMMs, and gate and up as two GEMMs +
// fused_glu, instead of the grouped launches.  Measured on an H100 SXM (700 W), Llama-3-8B layer shapes (DESIGN §5.3):
// the grouped QKV takes 0.54-0.89 x the separate launches from 256 to 2048 rows on Q8_0 but 1.17 x at 4096 and 1.12 x
// at 8192 (Q4_K_M's q|k + v: 0.89 x at 256 rows, 1.09-1.15 x from 1024 up); the GLU epilogue takes 0.93-0.94 x at 1024
// rows and 1.00-1.03 x from 2048 up.  Results are bit-identical either way.  A decode or verify step has at most 2048
// rows, so only the prompt step reaches the separate launches.
constexpr int GEMM_CHAIN_GROUPED_MAX_ROWS = 2048;

// the linears of the GEMM layer chain: `rows` rows on the wgmma dequant GEMM (mrs_mmq_gguf_grouped).
// whole_k: a row's result must not depend on the other rows of the launch, so K is never split (pdl | 2: a K split is
// chosen from the row count and sums the partials in another order), and a single matrix above 64 rows takes the
// plain ggml source of mrs_mmq_gguf, which runs faster than the one-matrix grouped source at prefill sizes and never
// splits K there (tc_gemm.cuh splits only token tiles of up to 64 rows).
struct GemmChain {
  const mrs_llama_step *s;
  int rows;
  bool whole_k;
  void *stream;

  int32_t grouped(int type, int n, const void **w, const int32_t *n_rows, void **y, const void *x, int K, int glu) const {
    return mrs_mmq_gguf_grouped(type, n, w, n_rows, y, x, rows, K, s->act_dtype, glu, whole_k ? s->pdl | 2 : s->pdl, stream);
  }
  // y = x W^T for the N-row matrix W
  int32_t single(const mrs_qweight &W, int N, void *y, const void *x, int K) const {
    if (whole_k && rows > 64) return mrs_mmq_gguf(W.ggml_type, W.data, x, y, rows, N, K, s->act_dtype, stream);
    const void *w[1] = {W.data};
    const int32_t n_rows[1] = {N};
    void *yy[1] = {y};
    return grouped(W.ggml_type, 1, w, n_rows, yy, x, K, 0);
  }
};

// the GEMM layer chain's buffers, of c.rows rows each: gate_up [2, rows, inter] is read only above
// GEMM_CHAIN_GROUPED_MAX_ROWS rows
struct GemmChainBufs {
  const int32_t *token_ids;
  void *x, *x2, *h, *q, *k, *v, *attn_out, *act, *gate_up;
};

// The layer stack of the 9..256-sequence decode and verify steps and of the prompt step, up to the final norm in h.  The
// norms are their own launches (the GEMM reads X through the TMA, unmodified), into the normed-activation buffer h:
//   embedding gather -> RMSNorm; per layer:
//   QKV (grouped: one launch, or q|k + v when attn_v has its own type; else three) -> attention(L) -> o GEMM (into h)
//   -> add + RMSNorm (x2 = o + x, h = norm) -> gate|up GEMM with the GLU epilogue (act) -> down GEMM (into h)
//   -> add + RMSNorm (x = down + x2, h = the next layer's norm, the final norm after the last layer)
// The o and down GEMMs write into h, which the add + RMSNorm after them reads as its input and overwrites with the
// norm: the norm kernel reads a row's input before its block-wide reduction and writes the row after it.  Every launch
// after the embedding gather and the first norm is a link of the PDL chain when s->pdl is set.  do_gemm == false
// skips the linears (decode's skip_mask bit 1).
template <class Attention>
static int32_t gemm_layer_chain(const GemmChain &c, const GemmChainBufs &b, bool do_gemm, Attention attention) {
  const mrs_llama_step *s = c.s;
  const int dt = s->act_dtype, H = s->hidden, T = c.rows;
  const int nq = s->n_heads * s->head_dim, nkv = s->n_kv_heads * s->head_dim;
  const bool grouped = T <= GEMM_CHAIN_GROUPED_MAX_ROWS;
  auto add_rms = [&](const void *x, const void *res, const void *w, void *res_dst) {
    mrs_add_rms_norm_pdl(x, res, w, res_dst, b.h, T, H, s->rms_eps, dt, s->pdl, c.stream);
  };

  MRS_TRY(mrs_embedding_gather(s->tok_embd.ggml_type, s->tok_embd.data, H, b.token_ids, T, b.x, dt, c.stream));
  if (dt == MRS_F16) mrs_rms_norm_f16(b.x, s->layers[0].attn_norm, b.h, T, H, s->rms_eps, (int64_t)c.stream);
  else mrs_rms_norm_bf16(b.x, s->layers[0].attn_norm, b.h, T, H, s->rms_eps, (int64_t)c.stream);
  for (int l = 0; l < s->n_layers; l++) {
    const mrs_llama_layer &L = s->layers[l];
    if (do_gemm) {
      const void *w[3] = {L.wq.data, L.wk.data, L.wv.data};
      const int32_t rows[3] = {nq, nkv, nkv};
      void *y[3] = {b.q, b.k, b.v};
      if (grouped && L.wq.ggml_type == L.wk.ggml_type && L.wk.ggml_type == L.wv.ggml_type) {
        MRS_TRY(c.grouped(L.wq.ggml_type, 3, w, rows, y, b.h, H, 0));
      } else if (grouped && L.wq.ggml_type == L.wk.ggml_type) {   // Q4_K_M keeps attn_v in Q6_K on some layers
        MRS_TRY(c.grouped(L.wq.ggml_type, 2, w, rows, y, b.h, H, 0));
        MRS_TRY(c.single(L.wv, nkv, b.v, b.h, H));
      } else {
        MRS_TRY(c.single(L.wq, nq, b.q, b.h, H));
        MRS_TRY(c.single(L.wk, nkv, b.k, b.h, H));
        MRS_TRY(c.single(L.wv, nkv, b.v, b.h, H));
      }
    }
    MRS_TRY(attention(L));
    if (!do_gemm) continue;
    MRS_TRY(c.single(L.wo, H, b.h, b.attn_out, nq));
    add_rms(b.h, b.x, L.ffn_norm, b.x2);                                     // x2 = o + x ; h = norm(x2)
    if (grouped) {
      const void *w[2] = {L.w_gate.data, L.w_up.data};
      const int32_t rows[2] = {L.w_gate.rows, L.w_up.rows};
      void *y[2] = {b.act, nullptr};
      MRS_TRY(c.grouped(L.w_gate.ggml_type, 2, w, rows, y, b.h, H, 1));
    } else {   // gate and up into the two halves of gate_up, then SiLU(gate) * up
      const int I = L.w_gate.rows;
      void *up = (uint8_t *)b.gate_up + (size_t)T * I * 2;
      MRS_TRY(c.single(L.w_gate, I, b.gate_up, b.h, H));
      MRS_TRY(c.single(L.w_up, I, up, b.h, H));
      if (dt == MRS_F16) fused_glu_f16(b.gate_up, up, b.act, T, I, I, I, 0, (cudaStream_t)c.stream);
      else fused_glu_bf16(b.gate_up, up, b.act, T, I, I, I, 0, (cudaStream_t)c.stream);
    }
    MRS_TRY(c.single(L.w_down, H, b.h, b.act, L.w_down.cols));
    add_rms(b.h, b.x2, l + 1 < s->n_layers ? s->layers[l + 1].attn_norm : s->final_norm, b.x);   // x = down + x2 ; h = next norm(x)
  }
  return 0;
}

// the decode step for 9..256 sequences: the reference's GgmlMatMul sends batches above 8 rows to MMQ, so the linears are
// the wgmma dequant GEMM with the prefill GEMM's numerics: the GEMM layer chain over batch * q_len rows with the decode
// attention, then the lm_head GEMM on h and argmax.  q_len > 1 is a speculative verify step of the 9..256-sequence route.
static int32_t llama_forward_gemm(const mrs_llama_step *s, int q_len, void *stream) {
  if (s->h == nullptr || (s->act_dtype != MRS_F16 && s->act_dtype != MRS_BF16)) return (int32_t)cudaErrorInvalidValue;
  if (const int32_t e = check_model(s)) return e;
  const bool do_attn = !(s->skip_mask & 1), do_gemm = !(s->skip_mask & 2);
  const GemmChain c{s, s->batch * q_len, false, stream};
  MRS_TRY(gemm_layer_chain(c, {s->token_ids, s->x, s->x2, s->h, s->q, s->k, s->v, s->attn_out, s->act, nullptr}, do_gemm,
                           [&](const mrs_llama_layer &L) { return do_attn ? decode_attention(s, L, q_len, stream) : 0; }));
  if (do_gemm) MRS_TRY(c.single(s->lm_head, s->vocab, s->logits, s->h, s->hidden));
  MRS_TRY(mrs_argmax(s->logits, c.rows, s->vocab, s->act_dtype, s->out_token, s->argmax_scratch, s->pdl, stream));
  return (int32_t)cudaGetLastError();
}

extern "C" int32_t mrs_llama_decode_step(const mrs_llama_step *s, void *stream) {
  if (s->batch < 1 || s->batch > 256) return (int32_t)cudaErrorInvalidValue;
  if (s->batch <= 8) return llama_forward(s, 1, stream);
  if (s->tp != nullptr || s->all_reduce != nullptr) return (int32_t)cudaErrorInvalidValue;
  return llama_forward_gemm(s, 1, stream);
}

// the verify step takes the linear route of the runner's plain step, chosen by the sequence count: batch 1..8 the GEMV
// chain (batch * q_len <= 8 rows), batch 9..256 the GEMM chain (up to 2048 rows)
extern "C" int32_t mrs_llama_verify_step(const mrs_llama_step *s, int32_t q_len, int32_t *context_lens, int32_t *accepted,
                                         int32_t *emitted, void *stream) {
  const bool gemm = s->batch > 8;
  if (q_len < 2 || q_len > 8 || s->batch < 1 || s->batch > 256 || (!gemm && s->batch * q_len > 8) || s->tp != nullptr ||
      s->all_reduce != nullptr || !s->fused_attention || (s->head_dim != 64 && s->head_dim != 128) ||
      s->out_token == s->token_ids || context_lens == nullptr || accepted == nullptr || emitted == nullptr)
    return (int32_t)cudaErrorInvalidValue;
  MRS_TRY(gemm ? llama_forward_gemm(s, q_len, stream) : llama_forward(s, q_len, stream));
  return mrs_spec_accept(s->out_token, s->token_ids, s->slot_mapping, context_lens, accepted, emitted, s->batch, q_len,
                         s->pdl, stream);
}

// the prompt step over the packed rows of n sequences (contract: include/mrs_b200_model.h): the GEMM layer chain over T
// rows with whole K, with the var-len prompt attention instead of the decode attention
extern "C" int32_t mrs_llama_prefill_step(const mrs_llama_step *s, const mrs_llama_prefill *p, void *stream) {
  if (s == nullptr || p == nullptr || !prompt_plan_ok(p, s->act_dtype, s->hidden)) return (int32_t)cudaErrorInvalidValue;
  const int n = p->n_seqs, T = p->total_tokens, dt = s->act_dtype, H = s->hidden, pdl = s->pdl;
  if (s->tp != nullptr || s->all_reduce != nullptr || s->layers == nullptr || p->k == nullptr || p->v == nullptr ||
      (T > GEMM_CHAIN_GROUPED_MAX_ROWS && p->gate_up == nullptr) || (p->lm_rows == 1 && n <= 8 && p->q8_scratch == nullptr))
    return (int32_t)cudaErrorInvalidValue;
  if (const int32_t e = check_model(s)) return e;
  // the lm_head of n <= 8 last rows: the reference-shaped MMVQ launcher of its type
  void (*lm_mmvq)(const void *, const void *, void *, int, int, int, int, int, void *) = nullptr;
  if (p->lm_rows == 1 && n <= 8) {
#define MRS_PLAIN_CASE(TYPE, tag) \
  case TYPE: lm_mmvq = dt == MRS_F16 ? launch_mmvq_gguf_##tag##_f16_plain : launch_mmvq_gguf_##tag##_bf16_plain; break;
    switch (s->lm_head.ggml_type) {
      MRS_PLAIN_CASE(MRS_Q4_0, q4_0) MRS_PLAIN_CASE(MRS_Q4_1, q4_1) MRS_PLAIN_CASE(MRS_Q5_0, q5_0)
      MRS_PLAIN_CASE(MRS_Q5_1, q5_1) MRS_PLAIN_CASE(MRS_Q8_0, q8_0) MRS_PLAIN_CASE(MRS_Q2_K, q2_k)
      MRS_PLAIN_CASE(MRS_Q3_K, q3_k) MRS_PLAIN_CASE(MRS_Q4_K, q4_k) MRS_PLAIN_CASE(MRS_Q5_K, q5_k)
      MRS_PLAIN_CASE(MRS_Q6_K, q6_k)
      default: return (int32_t)cudaErrorInvalidValue;
    }
#undef MRS_PLAIN_CASE
  }

  const int nq = s->n_heads * s->head_dim, nkv = s->n_kv_heads * s->head_dim;
  const GemmChain c{s, T, true, stream};
  const PromptAttnModel am{s->n_heads, s->n_kv_heads, s->head_dim, s->block_size, s->rope_neox, dt, s->sm_scale, s->rope_cos,
                           s->rope_sin};
  auto attention = [&](const mrs_llama_layer &L) -> int32_t {
    return prompt_attention(p, am, p->q, p->k, p->v, nq, nkv, L.k_cache, L.v_cache, false, stream);
  };
  MRS_TRY(gemm_layer_chain(c, {p->token_ids, p->x, p->x2, p->h, p->q, p->k, p->v, p->attn_out, p->act, p->gate_up}, true,
                           attention));
  if (p->lm_rows == 2) {
    MRS_TRY(c.single(s->lm_head, s->vocab, p->logits, p->h, H));
  } else if (p->lm_rows == 1) {
    prompt_gather_last_rows(p, p->h, H, stream);
    if (n <= 8) {    // the reference's GgufMatMul at 1..8 rows: Q8_1 activations + MMVQ (fast_mmvq plain)
      const int kpad = (H + 511) / 512 * 512;
      if (dt == MRS_F16) launch_mmvq_gguf_quantize_q8_1_f16(p->h_last, p->q8_scratch, H, kpad, n, stream);
      else launch_mmvq_gguf_quantize_q8_1_bf16(p->h_last, p->q8_scratch, H, kpad, n, stream);
      lm_mmvq(s->lm_head.data, p->q8_scratch, p->logits, H, s->vocab, kpad / 32, s->vocab, n, stream);
    } else {         // 9 and more rows: the dequant GEMM (the reference's MMQ branch)
      MRS_TRY((GemmChain{s, n, true, stream}.single(s->lm_head, s->vocab, p->logits, p->h_last, H)));
    }
    MRS_TRY(mrs_argmax(p->logits, n, s->vocab, dt, p->out_token, p->argmax_scratch, pdl, stream));
    if (p->dest_rows != nullptr) prompt_commit(p, stream);
  }
  return (int32_t)cudaGetLastError();
}
