// prefill_attn.cu — causal (var-len) prompt attention over fresh q/k/v tensors for sm_90a.
//
// The reference runs FlashAttention-2 (an sm80 CuTe kernel) on a fresh prompt:
//   REF mistralrs-core/src/paged_attention/layers/paged_attention.rs:1413-1475 (prompt path: attention over
//   the just-projected q/k/v, then reshape_and_cache), mistralrs-flash-attn/kernels/flash_fwd_*_sm80.cu,
//   API flash_attn_varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_q, max_k, softmax_scale, causal).
// SURVEY §8(f) rank 1.  This is an original kernel with the same arithmetic class: S = QK^T and O = PV on
// 16-bit tensor-core MMAs with f32 accumulation, online softmax in f32 (base-2 exponent, scale folded),
// P rounded to the activation dtype before the second GEMM.
//
// One CTA = 128 query rows of one (sequence, head): 8 warps x 16 rows.  Q fragments stay in
// registers; K/V tiles of 64 tokens stream through a double-buffered, XOR-swizzled shared-memory
// ring with cp.async (16-byte copies, two tiles in flight); B fragments come from ldmatrix
// (transposed for V).  GQA: head h reads KV head h / (H / KVH).  Causal tiles beyond the diagonal
// are skipped, the diagonal tile is masked in registers; heavy (late) query tiles are scheduled first.
// Legacy mma.sync path (SASS HMMA).  Head size 128 without window / softcap now runs on prefill_attn_tc.cu (wgmma);
// this kernel keeps head size 64, sliding window, softcap, and is the A/B for the other one.
//
// PAGED = true reads K/V from the HND page cache [num_blocks, KVH, page, D] (mrs_prefill_attention_paged): each
// cp.async row looks its page up in the sequence's block table; rows at or past kv_len are zero-filled and their
// page is never looked up.  Query i of a sequence sits at key position kv_len - q_len + i (bottom-right causal).
#include "mma_common.cuh"

#include <stdio.h>

namespace mrs {

constexpr int FA_BM = 128, FA_BN = 64, FA_WARPS = 8, FA_THREADS = FA_WARPS * 32;

struct FaParams {
  const void *q, *k, *v;
  void *o;
  const int32_t *cu_seqlens;   // [B + 1] or nullptr (single sequence of length T)
  int T, H, KVH;
  int64_t q_stride, kv_stride, o_stride;   // elements between consecutive tokens
  float scale_log2;            // softmax_scale * log2(e)
  float softcap;               // <= 0: off (applied to scale * qk, like the reference's flash-attn softcap)
  float softmax_scale;
  int causal, window_left;     // window_left < 0: off
  const int32_t *cu_seqlens_k; // paged: [B + 1] cumulative key counts (cu_seqlens then holds the query rows)
  const int32_t *block_table;  // paged: [B][bt_stride] page ids
  int bt_stride, page_shift;   // paged: page = 1 << page_shift tokens
};

template <typename T, int D, bool PAGED>
__global__ void __launch_bounds__(FA_THREADS, 1) prefill_attn_kernel(const FaParams p) {
  constexpr int KSTEPS = D / 16;        // k-steps of QK^T
  constexpr int DT = D / 8;             // 8-wide n-tiles of the output
  constexpr int CPR = D / 8;            // 16-byte chunks per row
  constexpr int TILE_BYTES = FA_BN * D * 2;
  extern __shared__ __align__(128) uint8_t fa_smem[];
  uint8_t *sk[2] = {fa_smem, fa_smem + 2 * TILE_BYTES};
  uint8_t *sv[2] = {fa_smem + TILE_BYTES, fa_smem + 3 * TILE_BYTES};

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y;
  const int kvh = h / (p.H / p.KVH);
  int seq0 = 0, len = p.T;
  if (p.cu_seqlens != nullptr) { seq0 = p.cu_seqlens[b]; len = p.cu_seqlens[b + 1] - seq0; }
  int kv_len = len;                                  // keys of the sequence; query i sits at key kv_len - len + i
  if constexpr (PAGED) kv_len = p.cu_seqlens_k[b + 1] - p.cu_seqlens_k[b];
  const int off = kv_len - len;
  const int ntile_q = (len + FA_BM - 1) / FA_BM;
  const int qt = ntile_q - 1 - (int)blockIdx.x;     // heavy tiles first
  if (qt < 0) return;
  const int q0 = qt * FA_BM;
  const T *qg = (const T *)p.q + (int64_t)seq0 * p.q_stride + (int64_t)h * D;
  const int64_t kv_base = PAGED ? ((int64_t)kvh * D << p.page_shift) : (int64_t)seq0 * p.kv_stride + (int64_t)kvh * D;
  const T *kg = (const T *)p.k + kv_base;
  const T *vg = (const T *)p.v + kv_base;
  // elements from kg / vg to key j < kv_len of a paged sequence
  auto page_off = [&](int j) -> int64_t {
    const int64_t blk = p.block_table[(int64_t)b * p.bt_stride + (j >> p.page_shift)];
    return ((blk * p.KVH << p.page_shift) + (j & ((1 << p.page_shift) - 1))) * D;
  };
  T *og = (T *)p.o + (int64_t)seq0 * p.o_stride + (int64_t)h * D;

  // KV range of this query tile
  const int q_hi = min(len, q0 + FA_BM) - 1;                               // last query row
  const int kv_end = p.causal ? (off + q_hi + 1) : kv_len;
  const int kv_begin = (p.window_left >= 0) ? max(0, off + q0 - p.window_left) / FA_BN * FA_BN : 0;
  const int nt = (kv_end - kv_begin + FA_BN - 1) / FA_BN;

  auto load_tile = [&](int t, int buf) {
    const int t0 = kv_begin + t * FA_BN;
    for (int c = tid; c < FA_BN * CPR; c += FA_THREADS) {
      const int row = c / CPR, ch = c % CPR;
      const bool ok = t0 + row < kv_len;
      const int64_t goff = PAGED ? (ok ? page_off(t0 + row) : 0) + ch * 8 : (int64_t)(ok ? t0 + row : 0) * p.kv_stride + ch * 8;
      cp_async16(sk[buf] + tile_off<D>(row, ch), kg + goff, ok);
      cp_async16(sv[buf] + tile_off<D>(row, ch), vg + goff, ok);
    }
    cp_async_commit();
  };

  // ---- Q fragments: warp rows q0 + 16 warp .. +15, staged through shared memory (buffer 1 of K/V is free yet)
  uint32_t qa[KSTEPS][4];
  {
    uint8_t *sq = sk[1];   // 128 rows x D: uses sk[1] and sv[1] (2 * TILE_BYTES = 128 * D * 2)
    for (int c = tid; c < FA_BM * CPR; c += FA_THREADS) {
      const int row = c / CPR, ch = c % CPR;
      const bool ok = q0 + row < len;
      cp_async16(sq + tile_off<D>(row, ch), qg + (int64_t)(ok ? q0 + row : 0) * p.q_stride + ch * 8, ok);
    }
    cp_async_commit();
    if (nt > 0) load_tile(0, 0);
    else cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const int r = warp * 16 + (lane & 15);
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ks++) {
      const int ch = 2 * ks + (lane >> 4);
      ldsm_x4(smem_u32(sq + tile_off<D>(r, ch)), qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3]);
    }
    __syncthreads();   // everyone has its Q before buffer 1 is overwritten
  }

  float oacc[DT][4];
#pragma unroll
  for (int i = 0; i < DT; i++) { oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const int row_a = q0 + warp * 16 + (lane >> 2);   // query rows of this thread's accumulators: row_a, row_a + 8

  for (int t = 0; t < nt; t++) {
    const int buf = t & 1;
    if (t + 1 < nt) load_tile(t + 1, buf ^ 1);
    else cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const int t0 = kv_begin + t * FA_BN;

    // ---- S = Q K^T : 16 rows x 64 tokens per warp
    float sacc[FA_BN / 8][4];
#pragma unroll
    for (int j = 0; j < FA_BN / 8; j++) { sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ks++) {
#pragma unroll
      for (int jp = 0; jp < FA_BN / 16; jp++) {
        // four 8x8 matrices: (tokens 16jp..+7, d 16ks..+7), (same tokens, d +8), (tokens +8, d), (tokens +8, d +8)
        const int row = 16 * jp + (lane & 7) + ((lane >> 4) << 3);
        const int ch = 2 * ks + ((lane >> 3) & 1);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(smem_u32(sk[buf] + tile_off<D>(row, ch)), b0, b1, b2, b3);
        mma16816<T>(sacc[2 * jp], qa[ks], b0, b1);
        mma16816<T>(sacc[2 * jp + 1], qa[ks], b2, b3);
      }
    }

    // ---- scale, soft-cap, mask, online softmax (base 2)
    const bool need_mask = (t0 + FA_BN > kv_end) || (p.causal && t0 + FA_BN - 1 > off + q0 + warp * 16) || (p.window_left >= 0);
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int j = 0; j < FA_BN / 8; j++) {
#pragma unroll
      for (int e = 0; e < 4; e++) {
        float s = sacc[j][e];
        if (p.softcap > 0.f) s = p.softcap * tanhf(s * p.softmax_scale / p.softcap) * 1.4426950408889634f;
        else s *= p.scale_log2;
        if (need_mask) {
          const int col = t0 + 8 * j + 2 * (lane & 3) + (e & 1);
          const int pos = off + row_a + ((e >> 1) << 3);
          const bool ok = col < kv_len && (!p.causal || col <= pos) && (p.window_left < 0 || col >= pos - p.window_left);
          if (!ok) s = -INFINITY;
        }
        sacc[j][e] = s;
        mx[e >> 1] = fmaxf(mx[e >> 1], s);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; r++) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; r++) {
      corr[r] = (mx[r] == -INFINITY) ? 1.f : exp2f(m_run[r] - mx[r]);
      m_run[r] = mx[r];
    }
    uint32_t pa[FA_BN / 16][4];
#pragma unroll
    for (int j = 0; j < FA_BN / 8; j++) {
      const float p0 = (mx[0] == -INFINITY) ? 0.f : exp2f(sacc[j][0] - mx[0]);
      const float p1 = (mx[0] == -INFINITY) ? 0.f : exp2f(sacc[j][1] - mx[0]);
      const float p2 = (mx[1] == -INFINITY) ? 0.f : exp2f(sacc[j][2] - mx[1]);
      const float p3 = (mx[1] == -INFINITY) ? 0.f : exp2f(sacc[j][3] - mx[1]);
      rs[0] += p0 + p1; rs[1] += p2 + p3;
      pa[j >> 1][(j & 1) * 2] = pack2<T>(p0, p1);
      pa[j >> 1][(j & 1) * 2 + 1] = pack2<T>(p2, p3);
    }
#pragma unroll
    for (int r = 0; r < 2; r++) l_run[r] = l_run[r] * corr[r] + rs[r];
#pragma unroll
    for (int i = 0; i < DT; i++) { oacc[i][0] *= corr[0]; oacc[i][1] *= corr[0]; oacc[i][2] *= corr[1]; oacc[i][3] *= corr[1]; }

    // ---- O += P V : V^T fragments through ldmatrix.trans
#pragma unroll
    for (int kk = 0; kk < FA_BN / 16; kk++) {
#pragma unroll
      for (int dp = 0; dp < DT / 2; dp++) {
        // matrices: (tokens 16kk..+7, d 16dp..+7), (tokens +8, same d), (tokens, d +8), (tokens +8, d +8)
        const int row = 16 * kk + (lane & 7) + (((lane >> 3) & 1) << 3);
        const int ch = 2 * dp + (lane >> 4);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(smem_u32(sv[buf] + tile_off<D>(row, ch)), b0, b1, b2, b3);
        mma16816<T>(oacc[2 * dp], pa[kk], b0, b1);
        mma16816<T>(oacc[2 * dp + 1], pa[kk], b2, b3);
      }
    }
    __syncthreads();   // buffer `buf` may be refilled by the next iteration's prefetch
  }
  cp_async_wait<0>();

  // ---- normalise and store
#pragma unroll
  for (int r = 0; r < 2; r++) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv0 = l_run[0] > 0.f ? 1.f / l_run[0] : 0.f, inv1 = l_run[1] > 0.f ? 1.f / l_run[1] : 0.f;
#pragma unroll
  for (int i = 0; i < DT; i++) {
    const int col = 8 * i + 2 * (lane & 3);
    if (row_a < len) *(uint32_t *)(og + (int64_t)row_a * p.o_stride + col) = pack2<T>(oacc[i][0] * inv0, oacc[i][1] * inv0);
    if (row_a + 8 < len) *(uint32_t *)(og + (int64_t)(row_a + 8) * p.o_stride + col) = pack2<T>(oacc[i][2] * inv1, oacc[i][3] * inv1);
  }
}

template <typename T, int D, bool PAGED = false>
static cudaError_t launch_fa(const FaParams &p, int batch, int max_len, cudaStream_t st) {
  auto kern = prefill_attn_kernel<T, D, PAGED>;
  const size_t smem = 4 * (size_t)FA_BN * D * 2;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid((max_len + FA_BM - 1) / FA_BM, p.H, batch);
  kern<<<grid, FA_THREADS, smem, st>>>(p);
  return cudaGetLastError();
}

}  // namespace mrs

using namespace mrs;

// out[t, h, :] = softmax_j(scale * q[t,h,:].k[j, h/g, :]) v[j, h/g, :] over j <= t (causal) of the same
// sequence.  q [total, H, D] (token stride q_stride elements), k/v [total, KVH, D] (kv_stride), out
// [total, H, D] (o_stride); cu_seqlens [batch + 1] i32 on the device or NULL (one sequence of
// `total` tokens; max_seqlen = longest sequence).  head_dim 64 or 128; dtype 0 f16 / 1 bf16;
// window_left < 0: full causal; softcap <= 0: off.  Returns a cudaError_t.
extern "C" int32_t mrs_prefill_attention_tc(const void *q, const void *k, const void *v, void *out, const int32_t *cu_seqlens,
                                            int32_t batch, int32_t total_tokens, int32_t max_seqlen, int32_t num_heads,
                                            int32_t num_kv_heads, int32_t head_dim, int64_t q_stride, int64_t kv_stride,
                                            int64_t o_stride, float softmax_scale, int32_t causal, int32_t window_left,
                                            float softcap, uint32_t dtype, void *stream);   // prefill_attn_tc.cu

extern "C" int32_t mrs_prefill_attention(const void *q, const void *k, const void *v, void *out, const int32_t *cu_seqlens,
                                         int32_t batch, int32_t total_tokens, int32_t max_seqlen, int32_t num_heads,
                                         int32_t num_kv_heads, int32_t head_dim, int64_t q_stride, int64_t kv_stride,
                                         int64_t o_stride, float softmax_scale, int32_t causal, int32_t window_left,
                                         float softcap, uint32_t dtype, void *stream) {
  if (total_tokens <= 0) return 0;
  {   // the wgmma kernel when the call fits it (head size 128, no window, no softcap)
    const int32_t e = mrs_prefill_attention_tc(q, k, v, out, cu_seqlens, batch, total_tokens, max_seqlen, num_heads, num_kv_heads,
                                               head_dim, q_stride, kv_stride, o_stride, softmax_scale, causal, window_left, softcap,
                                               dtype, stream);
    if (e != (int32_t)cudaErrorNotSupported) return e;
  }
  if ((dtype != 0 && dtype != 1) || num_kv_heads <= 0 || num_heads % num_kv_heads || (q_stride | kv_stride | o_stride) % 8)
    return (int32_t)cudaErrorInvalidValue;
  if (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15) return (int32_t)cudaErrorMisalignedAddress;
  FaParams p = {};
  p.q = q; p.k = k; p.v = v; p.o = out; p.cu_seqlens = cu_seqlens;
  p.T = total_tokens; p.H = num_heads; p.KVH = num_kv_heads;
  p.q_stride = q_stride; p.kv_stride = kv_stride; p.o_stride = o_stride;
  p.softmax_scale = softmax_scale; p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.softcap = softcap; p.causal = causal; p.window_left = window_left;
  const int nb = cu_seqlens ? batch : 1, ml = cu_seqlens ? max_seqlen : total_tokens;
  cudaStream_t st = (cudaStream_t)stream;
  if (head_dim == 128) return (int32_t)(dtype == 0 ? launch_fa<__half, 128>(p, nb, ml, st) : launch_fa<__nv_bfloat16, 128>(p, nb, ml, st));
  if (head_dim == 64) return (int32_t)(dtype == 0 ? launch_fa<__half, 64>(p, nb, ml, st) : launch_fa<__nv_bfloat16, 64>(p, nb, ml, st));
  return (int32_t)cudaErrorInvalidValue;
}

extern "C" int32_t mrs_prefill_attention_paged_tc(const void *q, const void *key_cache, const void *value_cache, void *out,
                                                  const int32_t *block_table, int32_t block_table_stride,
                                                  const int32_t *cu_seqlens_q, const int32_t *cu_seqlens_k, int32_t batch,
                                                  int32_t total_q, int32_t max_seqlen_q, int32_t max_seqlen_k, int32_t num_blocks,
                                                  int32_t num_heads, int32_t num_kv_heads, int32_t head_dim, int32_t page_size,
                                                  int64_t q_stride, int64_t o_stride, float softmax_scale, int32_t causal,
                                                  int32_t window_left, float softcap, uint32_t dtype, void *stream);   // prefill_attn_tc.cu

// prompt attention of new query tokens over K/V already in the HND page cache; contract in include/mrs_b200_paged_attn.h
extern "C" int32_t mrs_prefill_attention_paged(const void *q, const void *key_cache, const void *value_cache, void *out,
                                               const int32_t *block_table, int32_t block_table_stride,
                                               const int32_t *cu_seqlens_q, const int32_t *cu_seqlens_k, int32_t batch,
                                               int32_t total_q, int32_t max_seqlen_q, int32_t max_seqlen_k, int32_t num_blocks,
                                               int32_t num_heads, int32_t num_kv_heads, int32_t head_dim, int32_t page_size,
                                               int64_t q_stride, int64_t o_stride, float softmax_scale, int32_t causal,
                                               int32_t window_left, float softcap, uint32_t dtype, void *stream) {
  if (total_q <= 0 || batch <= 0) return 0;
  if ((dtype != 0 && dtype != 1) || (head_dim != 64 && head_dim != 128) || num_kv_heads <= 0 || num_heads % num_kv_heads ||
      (page_size != 8 && page_size != 16 && page_size != 32) || (q_stride | o_stride) % 8 || num_blocks <= 0 ||
      block_table == nullptr || cu_seqlens_q == nullptr || cu_seqlens_k == nullptr || block_table_stride <= 0)
    return (int32_t)cudaErrorInvalidValue;
  if (((uintptr_t)q | (uintptr_t)key_cache | (uintptr_t)value_cache | (uintptr_t)out) & 15) return (int32_t)cudaErrorMisalignedAddress;
  {   // the wgmma kernel when the call fits it (head size 128, no window, no softcap)
    const int32_t e = mrs_prefill_attention_paged_tc(q, key_cache, value_cache, out, block_table, block_table_stride, cu_seqlens_q,
                                                     cu_seqlens_k, batch, total_q, max_seqlen_q, max_seqlen_k, num_blocks, num_heads,
                                                     num_kv_heads, head_dim, page_size, q_stride, o_stride, softmax_scale, causal,
                                                     window_left, softcap, dtype, stream);
    if (e != (int32_t)cudaErrorNotSupported) return e;
  }
  FaParams p = {};
  p.q = q; p.k = key_cache; p.v = value_cache; p.o = out; p.cu_seqlens = cu_seqlens_q; p.cu_seqlens_k = cu_seqlens_k;
  p.block_table = block_table; p.bt_stride = block_table_stride; p.page_shift = page_size == 8 ? 3 : page_size == 16 ? 4 : 5;
  p.T = total_q; p.H = num_heads; p.KVH = num_kv_heads;
  p.q_stride = q_stride; p.kv_stride = head_dim; p.o_stride = o_stride;
  p.softmax_scale = softmax_scale; p.scale_log2 = softmax_scale * 1.4426950408889634f;
  p.softcap = softcap; p.causal = causal; p.window_left = window_left;
  cudaStream_t st = (cudaStream_t)stream;
  if (head_dim == 128)
    return (int32_t)(dtype == 0 ? launch_fa<__half, 128, true>(p, batch, max_seqlen_q, st) : launch_fa<__nv_bfloat16, 128, true>(p, batch, max_seqlen_q, st));
  return (int32_t)(dtype == 0 ? launch_fa<__half, 64, true>(p, batch, max_seqlen_q, st) : launch_fa<__nv_bfloat16, 64, true>(p, batch, max_seqlen_q, st));
}
