// paged_attn.cu — decode attention over a paged KV cache for sm_90a, behind the reference's
// C symbols:
//   paged_attention_v1_{f16,bf16}, paged_attention_v2_{f16,bf16}   (vLLM cache layout)
//        REF mistralrs-paged-attn/src/cuda/ffi.rs:269-438, pagedattention.cuh:110-485,549-665
//   flashinfer_decode                                              (HND cache, CSR page table, split-KV tiles)
//        REF mistralrs-paged-attn/src/cuda/ffi.rs:178-209, flashinfer_decode.cu:103-148,314-363
//
// Design: one CTA per (work tile, KV head).  A tile is a (sequence, KV chunk) pair.  The CTA
// serves the whole GQA group of the KV head, so every K/V byte is read from HBM once (the
// reference's vLLM kernel re-reads it per query head).  LPT = D/8 lanes own one token: each lane
// holds a 16-byte (8-element) slice of the head dimension for q (all G heads), k and v; a token's
// K and V rows are each one coalesced 16-byte-per-lane load.  Token groups walk the chunk with
// 4-deep unrolled loads, run an online softmax privately (f32), and are merged once at the end
// through shared memory.  Split-KV partials (normalised o + log-sum-exp) are merged by a second
// tiny kernel.  Softcap, sliding window (window_left), ALiBi and attention sinks follow the
// reference's formulas.
#include "common.cuh"

#include <cuda_fp8.h>
#include <stdio.h>
#include <stdlib.h>

namespace mrs {

constexpr int PA_THREADS = 256;
constexpr int PA_UNROLL = 4;

struct PagedParams {
  const void *q;       // [S, H, D] (+strides)
  const void *kc, *vc; // caches
  void *out;           // [S, H, D] contiguous
  // split scratch (nullptr -> write final output directly)
  void *tmp_o;         // [tiles, H, D] in T
  float *tmp_lse;      // [tiles, H]
  // work description
  const int32_t *request_indices;  // [tiles] or nullptr (tile == seq, chunk 0)
  const int32_t *kv_tile_indices;  // [tiles] or nullptr
  const uint8_t *block_valid_mask; // [tiles] or nullptr
  const int32_t *kv_chunk_size_ptr; // device scalar or nullptr
  int kv_chunk_size;               // used when ptr is null; <=0 -> whole context
  // page table: CSR (HND API) or dense block table (vLLM API)
  const int32_t *kv_indptr, *kv_indices, *kv_last_page_len;
  const int32_t *block_tables, *context_lens;
  int max_blocks_per_seq;
  int64_t kv_block_stride, kv_head_stride;  // elements
  int num_heads, num_kv_heads, page_size;
  int64_t q_stride_n, q_stride_h;
  float sm_scale, softcap;  // softcap <= 0: disabled
  float k_scale, v_scale;   // FP8 cache: per-tensor dequantisation scales (1 for 16/32-bit caches)
  const float *k_scale_ptr, *v_scale_ptr;   // the same as device scalars (vLLM-style API); override the values
  int window_left;          // < 0: disabled
  const float *alibi_slopes, *sinks;
  int tiles_are_partitions; // vLLM v2: tile index = seq * num_partitions + partition
  int num_partitions;
  int heads_per_cta;        // GQA group may be processed in sub-groups (blockIdx.z)
  int batch_size;           // sequences in this launch (0: unknown)
  int pdl;                  // launched with programmatic stream serialisation
  // FUSED (mrs_paged_decode_fused): un-rotated new-token K/V, RoPE tables, slots, merge counters
  const void *k_new, *v_new;
  int64_t kv_new_stride;
  const void *rope_cos, *rope_sin;
  int rope_interleaved;     // 0: rotate-half (NeoX) pairing, 1: interleaved pairs (GGUF llama files)
  const int32_t *positions;
  const int64_t *slot_mapping;
  const int32_t *o_indptr;
  int *counters;
  int q_len;                // mrs_paged_decode_fused_multi: query rows per sequence (q, k_new, v_new, out: [B * q_len, ...])
};

template <typename T> struct Vec8;
template <> struct Vec8<__half> {
  __device__ static __forceinline__ void load(const __half *p, float *f) {
    const uint4 v = *(const uint4 *)p;
    const __half2 *h = (const __half2 *)&v;
#pragma unroll
    for (int i = 0; i < 4; i++) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  __device__ static __forceinline__ float one(const __half *p) { return __half2float(*p); }
  __device__ static __forceinline__ void store(__half *p, const float *f) {
    uint4 v;
    __half2 *h = (__half2 *)&v;
#pragma unroll
    for (int i = 0; i < 4; i++) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    *(uint4 *)p = v;
  }
};
template <> struct Vec8<__nv_bfloat16> {
  __device__ static __forceinline__ void load(const __nv_bfloat16 *p, float *f) {
    const uint4 v = *(const uint4 *)p;
    const __nv_bfloat162 *h = (const __nv_bfloat162 *)&v;
#pragma unroll
    for (int i = 0; i < 4; i++) { const float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  __device__ static __forceinline__ float one(const __nv_bfloat16 *p) { return __bfloat162float(*p); }
  __device__ static __forceinline__ void store(__nv_bfloat16 *p, const float *f) {
    uint4 v;
    __nv_bfloat162 *h = (__nv_bfloat162 *)&v;
#pragma unroll
    for (int i = 0; i < 4; i++) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    *(uint4 *)p = v;
  }
};
template <> struct Vec8<float> {
  __device__ static __forceinline__ void load(const float *p, float *f) {
    const float4 a = *(const float4 *)p, b = *(const float4 *)(p + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  __device__ static __forceinline__ float one(const float *p) { return *p; }
  __device__ static __forceinline__ void store(float *p, const float *f) {
    *(float4 *)p = make_float4(f[0], f[1], f[2], f[3]);
    *(float4 *)(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
  }
};
// FP8-E4M3 cache bytes (cache_dtype 3, REF mistralrs-paged-attn/src/cuda/ffi.rs dtype codes): value = float(e4m3);
// the per-tensor scales are folded into the logits (k_scale) and the output (v_scale)
struct fp8_t { uint8_t b; };
__device__ __forceinline__ float fp8_to_float(uint8_t b) {
  const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)b, __NV_E4M3);
  return __half2float(*(const __half *)&h);
}
template <> struct Vec8<fp8_t> {
  __device__ static __forceinline__ void load(const fp8_t *p, float *f) {
    const uint2 v = *(const uint2 *)p;
    const uint8_t *b = (const uint8_t *)&v;
#pragma unroll
    for (int i = 0; i < 8; i++) f[i] = fp8_to_float(b[i]);
  }
  __device__ static __forceinline__ float one(const fp8_t *p) { return fp8_to_float(p->b); }
};

// round through T (what storing a tensor of dtype T would do)
template <typename T> __device__ __forceinline__ float rnd(float v);
template <> __device__ __forceinline__ float rnd<__half>(float v) { return __half2float(__float2half_rn(v)); }
template <> __device__ __forceinline__ float rnd<__nv_bfloat16>(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
template <> __device__ __forceinline__ float rnd<float>(float v) { return v; }
template <typename T> __device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ float from_float<float>(float v) { return v; }

// NeoX RoPE of the 8-element slice held by lane `gl` (elements d0..d0+7 of a head), with the
// reference kernel's per-operation rounding in T (rotary.cu:10-34).  The partner slice
// (d +- D/2) lives in lane gl ^ (LPT/2).
template <typename T, int D>
__device__ __forceinline__ void rope_slice(float *x, const T *cosp, const T *sinp, int gl) {
  constexpr int LPT = D / 8;
  const bool upper = gl >= LPT / 2;
  const int o0 = (upper ? gl - LPT / 2 : gl) * 8;  // rot offset of this slice
  float c[8], sn[8];
  Vec8<T>::load(cosp + o0, c);
  Vec8<T>::load(sinp + o0, sn);
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const float other = __shfl_xor_sync(0xffffffffu, x[i], LPT / 2);
    // out_x = fma(x, cos, -T(y*sin)); out_y = fma(y, cos, T(x*sin)) with one rounding in T, as the
    // reference kernel is compiled (tests/golden/ref_golden.npz)
    const float b = rnd<T>(other * sn[i]);     // y*sin (lower) / x*sin (upper)
    x[i] = (float)__hfma((T)x[i], (T)c[i], (T)(upper ? b : -b));
  }
}
// GPT-J / GGUF-llama pairing: (x[2i], x[2i+1]) rotate together and both live in this lane's slice;
// cos/sin index d/2.  Same per-operation rounding as rope_slice (REF rotary.cu:10-34, is_neox = 0).
template <typename T, int D>
__device__ __forceinline__ void rope_slice_interleaved(float *x, const T *cosp, const T *sinp, int gl) {
  const int o0 = gl * 4;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const float c = Vec8<T>::one(cosp + o0 + i), sn = Vec8<T>::one(sinp + o0 + i);
    const float xv = x[2 * i], yv = x[2 * i + 1];
    const float ys = rnd<T>(yv * sn), xs = rnd<T>(xv * sn);
    x[2 * i] = (float)__hfma((T)xv, (T)c, (T)(-ys));
    x[2 * i + 1] = (float)__hfma((T)yv, (T)c, (T)xs);
  }
}
template <typename T, int D>
__device__ __forceinline__ void rope_any(float *x, const T *cosp, const T *sinp, int gl, bool interleaved) {
  if (interleaved) rope_slice_interleaved<T, D>(x, cosp, sinp, gl);
  else rope_slice<T, D>(x, cosp, sinp, gl);
}

constexpr int pa_next_pow2(int v) { return v <= 8 ? 8 : (v <= 16 ? 16 : 32); }

// LAYOUT 0: vLLM (K [NB,KVH,D/x,BS,x] with x = 16 / sizeof(cache element), V [NB,KVH,D,BS]); 1: HND ([NB,KVH,BS,D])
// T: query / output dtype; CT: cache element (T, or fp8_t for the FP8-E4M3 cache).
// Head sizes that are not 8 x a power of two (80, 96, 112, 192) run with the next power-of-two lane count and
// idle lanes; 512 gives every lane 16 elements.
// FUSED (16-bit caches, D in {64,128,256}): q/k/v of the new token arrive un-rotated; the kernel applies RoPE,
// writes the new K/V row into the cache (the tile that owns the last position) and merges split-KV partials
// itself ("last tile done" counter) — one launch instead of rope + reshape_and_cache + decode + merge.
template <typename T, typename CT, int D, int G, int LAYOUT, bool FUSED>
__global__ void __launch_bounds__(PA_THREADS) paged_decode_kernel(const PagedParams p) {
  constexpr int EPL = (D > 256) ? 16 : 8;              // elements per lane
  constexpr int NV = EPL / 8;                          // 8-element vectors per lane
  constexpr int LPT_RAW = (D + EPL - 1) / EPL;         // lanes that hold data
  constexpr int LPT = pa_next_pow2(LPT_RAW);           // lanes per token (power of two: shuffle reductions)
  constexpr int NGRP = PA_THREADS / LPT;               // token groups per CTA
  constexpr int UNROLL = (EPL == 16) ? 1 : PA_UNROLL;
  constexpr int XK = 16 / (int)sizeof(CT);             // vLLM K-cache inner width
  static_assert(!FUSED || (EPL == 8 && LPT_RAW == LPT && sizeof(CT) == sizeof(T)), "fused path: plain 16-bit heads");
  const int tile = blockIdx.x, kvh = blockIdx.y;
  const int tid = threadIdx.x;
  const int grp = tid / LPT, gl = tid % LPT;  // group, lane within group
  const int d0 = gl * EPL;
  const bool act = gl < LPT_RAW;              // lane holds elements d0 .. d0+EPL-1 (all < D: D % EPL == 0)

  if (p.pdl && tid == 0) pdl_launch_dependents();  // downstream GEMV may start prefetching its weights
  if (p.block_valid_mask != nullptr && p.block_valid_mask[tile] == 0) return;
  int seq, chunk_idx;
  if (p.tiles_are_partitions) { seq = tile / p.num_partitions; chunk_idx = tile % p.num_partitions; }
  else if (p.request_indices != nullptr) { seq = p.request_indices[tile]; chunk_idx = p.kv_tile_indices[tile]; }
  else { seq = tile; chunk_idx = 0; }

  // context length and page list of this sequence
  int kv_len;
  const int32_t *pages;
  if (p.kv_indptr != nullptr) {
    const int p0 = p.kv_indptr[seq], p1 = p.kv_indptr[seq + 1];
    pages = p.kv_indices + p0;
    kv_len = (p1 > p0) ? (p1 - p0 - 1) * p.page_size + p.kv_last_page_len[seq] : 0;
  } else {
    pages = p.block_tables + (int64_t)seq * p.max_blocks_per_seq;
    kv_len = p.context_lens[seq];
  }
  int chunk = p.kv_chunk_size_ptr ? *p.kv_chunk_size_ptr : p.kv_chunk_size;
  if (chunk <= 0) chunk = kv_len > 0 ? kv_len : 1;
  const int t_begin = chunk_idx * chunk;
  int t_end = min(kv_len, t_begin + chunk);
  const bool partial = p.tmp_o != nullptr;

  const int group = p.num_heads / p.num_kv_heads;
  const int h0 = kvh * group + blockIdx.z * p.heads_per_cta;      // first query head of this CTA
  const int gsize = min(p.heads_per_cta, group - (int)blockIdx.z * p.heads_per_cta);  // heads here (<= G)

  // q slice of this lane for all heads of the group; filled after the page copies are in flight and after
  // griddepcontrol.wait (q/k_new/v_new come from the upstream kernel)
  float qf[G][EPL];
  const T *cosp = nullptr, *sinp = nullptr;
  float slope[G];
#pragma unroll
  for (int g = 0; g < G; g++) slope[g] = (p.alibi_slopes != nullptr && g < gsize) ? p.alibi_slopes[h0 + g] : 0.f;

  float m[G], l[G], o[G][EPL];
#pragma unroll
  for (int g = 0; g < G; g++) {
    m[g] = -INFINITY; l[g] = 0.f;
#pragma unroll
    for (int i = 0; i < EPL; i++) o[g][i] = 0.f;
  }

  const CT *kc = (const CT *)p.kc, *vc = (const CT *)p.vc;
  const int win_lo = (p.window_left >= 0) ? max(0, kv_len - 1 - p.window_left) : 0;

  auto load_q = [&]() {
    if (p.pdl) pdl_wait();
    if constexpr (FUSED) {
      const int64_t pos = p.positions[seq];
      cosp = (const T *)p.rope_cos + pos * (D / 2);
      sinp = (const T *)p.rope_sin + pos * (D / 2);
    }
#pragma unroll
    for (int g = 0; g < G; g++) {
      if (g < gsize && act) {
#pragma unroll
        for (int v = 0; v < NV; v++)
          Vec8<T>::load((const T *)p.q + (int64_t)seq * p.q_stride_n + (int64_t)(h0 + g) * p.q_stride_h + d0 + 8 * v, qf[g] + 8 * v);
      } else {
#pragma unroll
        for (int i = 0; i < EPL; i++) qf[g][i] = 0.f;
      }
      if constexpr (FUSED) rope_any<T, D>(qf[g], cosp, sinp, gl, p.rope_interleaved != 0);
#pragma unroll
      for (int i = 0; i < EPL; i++) qf[g][i] *= p.sm_scale * (p.k_scale_ptr ? *p.k_scale_ptr : p.k_scale);
    }
  };

  // one token's contribution to the running softmax state of this token group
  auto update = [&](const float *kf, const float *vf, int t, bool live) {
    float s[G];
#pragma unroll
    for (int g = 0; g < G; g++) {
      float a = 0.f;
#pragma unroll
      for (int i = 0; i < EPL; i++) a = fmaf(qf[g][i], kf[i], a);
      s[g] = a;
    }
#pragma unroll
    for (int mask = LPT / 2; mask > 0; mask >>= 1)
#pragma unroll
      for (int g = 0; g < G; g++) s[g] += __shfl_xor_sync(0xffffffffu, s[g], mask);
    const bool in_window = t >= win_lo && live;
#pragma unroll
    for (int g = 0; g < G; g++) {
      float x = s[g];
      if (p.softcap > 0.f) x = p.softcap * tanhf(x / p.softcap);
      // REF pagedattention.cuh:138,283: `context_len` is a uint32_t there, so `token_idx - context_len + 1`
      // is evaluated in unsigned arithmetic and wraps for every token but the last; restated as is
      // (tests/golden pins it against the reference kernel's output)
      if (slope[g] != 0.f) x += slope[g] * (float)(uint32_t)(t - kv_len + 1);
      if (!in_window) x = -INFINITY;
      const float mn = fmaxf(m[g], x);
      if (mn > -INFINITY) {
        const float corr = __expf(m[g] - mn);
        const float pv = __expf(x - mn);
        l[g] = l[g] * corr + pv;
#pragma unroll
        for (int i = 0; i < EPL; i++) o[g][i] = fmaf(pv, vf[i], o[g][i] * corr);
        m[g] = mn;
      }
    }
  };

  // FUSED: the tile that owns the last position takes the new token from registers
  bool owns_new = false;
  if constexpr (FUSED) {
    owns_new = kv_len > 0 && (kv_len - 1) >= t_begin && (kv_len - 1) < t_end;
    if (owns_new) t_end = kv_len - 1;  // the cache loop stops before the new token
  }

  if constexpr (LAYOUT == 1) {
    // ---- HND: stage the chunk's pages through shared memory with the TMA engine.  A page is a
    // contiguous [page_size, D] slab per KV head, so one cp.async.bulk per (page, K|V) moves it;
    // all copies of a sub-chunk are in flight at once (one HBM latency per sub-chunk
    // instead of one per 4 tokens), double buffered.
    extern __shared__ __align__(128) uint8_t pa_stage[];
    constexpr int ROWB = D * (int)sizeof(CT);                         // bytes per cached row
    constexpr int SUB = (ROWB <= 256) ? 128 : (ROWB <= 512 ? 64 : 32);  // tokens per sub-chunk
    constexpr int SUB_BYTES = SUB * ROWB;                              // per K or V buffer
    __shared__ __align__(8) uint64_t st_full[2];
    CT *st_k[2] = {(CT *)pa_stage, (CT *)(pa_stage + 2 * SUB_BYTES)};
    CT *st_v[2] = {(CT *)(pa_stage + SUB_BYTES), (CT *)(pa_stage + 3 * SUB_BYTES)};
    if (tid == 0) { mbar_init(&st_full[0], 1); mbar_init(&st_full[1], 1); fence_mbar_init(); }
    __syncthreads();
    const int nsub = (t_end > t_begin) ? (t_end - t_begin + SUB - 1) / SUB : 0;
    // page ids of the chunk -> shared memory in one parallel round (a serial walk by the
    // issuing thread would pay one L2 latency per page)
    __shared__ int st_pages[2048 / 8 + 2];
    const int pg0 = t_begin / p.page_size;
    const int npg = (t_end > t_begin) ? (t_end - 1) / p.page_size - pg0 + 1 : 0;
    for (int i = tid; i < npg && i < (int)(sizeof(st_pages) / sizeof(int)); i += PA_THREADS) st_pages[i] = pages[pg0 + i];
    __syncthreads();
    const bool pages_in_smem = npg <= (int)(sizeof(st_pages) / sizeof(int));
    auto issue = [&](int si) {  // thread 0 only
      const int s0 = t_begin + si * SUB, s1 = min(t_end, s0 + SUB);
      const int b = si & 1;
      mbar_arrive_expect_tx(&st_full[b], (uint32_t)(2 * (s1 - s0) * ROWB));
      for (int t = s0; t < s1;) {
        const int off = t % p.page_size;
        const int n = min(p.page_size - off, s1 - t);   // tokens of this page inside the sub-chunk
        const int pgi = t / p.page_size;
        const int64_t pg = pages_in_smem ? st_pages[pgi - pg0] : pages[pgi];
        const int64_t base = pg * p.kv_block_stride + (int64_t)kvh * p.kv_head_stride + (int64_t)off * D;
        const uint32_t bytes = (uint32_t)(n * ROWB);
        bulk_g2s(st_k[b] + (size_t)(t - s0) * D, kc + base, bytes, &st_full[b]);
        bulk_g2s(st_v[b] + (size_t)(t - s0) * D, vc + base, bytes, &st_full[b]);
        t += n;
      }
    };
    if (tid == 0 && nsub > 0) issue(0);
    load_q();
    for (int si = 0; si < nsub; si++) {
      const int b = si & 1;
      if (tid == 0 && si + 1 < nsub) issue(si + 1);   // buffer (si+1)&1 was released by the barrier below
      mbar_wait(&st_full[b], (uint32_t)((si >> 1) & 1));
      const int s0 = t_begin + si * SUB, s1 = min(t_end, s0 + SUB);
      // trip count is uniform across the CTA (the shuffles need every lane of the warp)
      for (int tb0 = s0; tb0 < s1; tb0 += NGRP * UNROLL) {
        const int tb = tb0 + grp;
        float kf[UNROLL][EPL], vf[UNROLL][EPL];
        bool ok[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; u++) {
          const int t = tb + u * NGRP;
          ok[u] = t < s1;
#pragma unroll
          for (int i = 0; i < EPL; i++) { kf[u][i] = 0.f; vf[u][i] = 0.f; }
          if (ok[u] && act) {
#pragma unroll
            for (int v = 0; v < NV; v++) {
              Vec8<CT>::load(st_k[b] + (size_t)(t - s0) * D + d0 + 8 * v, kf[u] + 8 * v);
              Vec8<CT>::load(st_v[b] + (size_t)(t - s0) * D + d0 + 8 * v, vf[u] + 8 * v);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; u++) update(kf[u], vf[u], tb + u * NGRP, ok[u]);
      }
      __syncthreads();  // everyone is done with buffer b before it is refilled
    }
  } else {
  load_q();
  // trip count is uniform across the CTA (the shuffles need every lane of the warp)
  for (int tb0 = t_begin; tb0 < t_end; tb0 += NGRP * UNROLL) {
    const int tb = tb0 + grp;
    float kf[UNROLL][EPL], vf[UNROLL][EPL];
    bool ok[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; u++) {
      const int t = tb + u * NGRP;
      ok[u] = t < t_end;
#pragma unroll
      for (int i = 0; i < EPL; i++) { kf[u][i] = 0.f; vf[u][i] = 0.f; }
      if (ok[u] && act) {
        const int64_t page = pages[t / p.page_size];
        const int off = t % p.page_size;
        const int64_t base = page * p.kv_block_stride + (int64_t)kvh * p.kv_head_stride;
        // K [D/XK][BS][XK]: this lane's EPL consecutive d's are EPL/XK whole groups, or part of one group
        if constexpr (EPL >= XK) {
#pragma unroll
          for (int c = 0; c < EPL / XK; c++) {
            const CT *src = kc + base + ((int64_t)(d0 / XK + c) * p.page_size + off) * XK;
            if constexpr (XK == 8) Vec8<CT>::load(src, kf[u] + 8 * c);
            else {                                       // XK == 4 (f32 cache)
#pragma unroll
              for (int i = 0; i < XK; i++) kf[u][XK * c + i] = Vec8<CT>::one(src + i);
            }
          }
        } else {                                          // XK == 16 (fp8 cache), EPL == 8
          Vec8<CT>::load(kc + base + ((int64_t)(d0 / XK) * p.page_size + off) * XK + (d0 % XK), kf[u]);
        }
#pragma unroll
        for (int i = 0; i < EPL; i++) vf[u][i] = Vec8<CT>::one(vc + base + (int64_t)(d0 + i) * p.page_size + off);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; u++) update(kf[u], vf[u], tb + u * NGRP, ok[u]);
  }
  }

  if constexpr (FUSED) {
    if (owns_new) {  // CTA-uniform
      // every token group computes the rotated key (cheap) so the shuffles stay warp-uniform;
      // group 0 contributes it to the softmax and (sub-group 0 only) writes the cache row
      float kn[8], vn[8];
      Vec8<T>::load((const T *)p.k_new + (int64_t)seq * p.kv_new_stride + (int64_t)kvh * D + d0, kn);
      Vec8<T>::load((const T *)p.v_new + (int64_t)seq * p.kv_new_stride + (int64_t)kvh * D + d0, vn);
      rope_any<T, D>(kn, cosp, sinp, gl, p.rope_interleaved != 0);
      update(kn, vn, kv_len - 1, grp == 0);
      const int64_t slot = p.slot_mapping[seq];
      if (grp == 0 && blockIdx.z == 0 && slot >= 0) {
        const int64_t page = slot / p.page_size;
        const int off = (int)(slot % p.page_size);
        const int64_t base = page * p.kv_block_stride + (int64_t)kvh * p.kv_head_stride;
        T *kcw = (T *)p.kc, *vcw = (T *)p.vc;
        if constexpr (LAYOUT == 1) {
          Vec8<T>::store(kcw + base + (int64_t)off * D + d0, kn);
          Vec8<T>::store(vcw + base + (int64_t)off * D + d0, vn);
        } else {
          Vec8<T>::store(kcw + base + ((int64_t)gl * p.page_size + off) * 8, kn);
#pragma unroll
          for (int i = 0; i < 8; i++) vcw[base + (int64_t)(d0 + i) * p.page_size + off] = from_float<T>(vn[i]);
        }
      }
    }
  }

  // ---------------------------------------------------------------- merge the token groups
  constexpr int NSTATE = PA_THREADS / 32;  // one softmax state per warp after the pre-merge
  static_assert(LPT <= 16 || NGRP == NSTATE, "one token group per warp when LPT == 32");
  __shared__ float sm_m[NSTATE][G], sm_l[NSTATE][G];
  __shared__ float sm_o[NSTATE][G][D];
  __shared__ int sm_last;
  // pairwise pre-merge inside a warp when several groups share one (LPT < 32)
  if constexpr (LPT <= 16) {
#pragma unroll
    for (int mask = LPT; mask < 32; mask <<= 1) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const float mo = __shfl_xor_sync(0xffffffffu, m[g], mask);
        const float lo = __shfl_xor_sync(0xffffffffu, l[g], mask);
        const float mn = fmaxf(m[g], mo);
        const float ca = (mn > -INFINITY) ? __expf(m[g] - mn) : 0.f;
        const float cb = (mn > -INFINITY) ? __expf(mo - mn) : 0.f;
#pragma unroll
        for (int i = 0; i < EPL; i++) {
          const float oo = __shfl_xor_sync(0xffffffffu, o[g][i], mask);
          o[g][i] = o[g][i] * ca + oo * cb;
        }
        l[g] = l[g] * ca + lo * cb;
        m[g] = mn;
      }
    }
  }
  constexpr int WG = NSTATE;
  const int warp = tid >> 5, lane = tid & 31;
  const int sidx = warp;
  const bool writer = lane < LPT;
  if (writer) {
#pragma unroll
    for (int g = 0; g < G; g++) {
      if (gl == 0) { sm_m[sidx][g] = m[g]; sm_l[sidx][g] = l[g]; }
      if (act) {
#pragma unroll
        for (int i = 0; i < EPL; i++) sm_o[sidx][g][d0 + i] = o[g][i];
      }
    }
  }
  __syncthreads();
  // final: thread per (head, d)
  for (int idx = tid; idx < G * D; idx += PA_THREADS) {
    const int g = idx / D, d = idx % D;
    if (g >= gsize) continue;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < WG; w++) M = fmaxf(M, sm_m[w][g]);
    const bool use_sink = (p.sinks != nullptr) && !partial;
    if (use_sink) M = fmaxf(M, p.sinks[h0 + g]);
    float L = 0.f, acc = 0.f;
    if (M > -INFINITY) {
#pragma unroll
      for (int w = 0; w < WG; w++) {
        const float c = __expf(sm_m[w][g] - M);
        L += sm_l[w][g] * c;
        acc += sm_o[w][g][d] * c;
      }
    }
    if (use_sink) L += __expf(p.sinks[h0 + g] - M);
    const float val = (L > 0.f) ? acc / L * (p.v_scale_ptr ? *p.v_scale_ptr : p.v_scale) : 0.f;
    if (partial) {
      ((T *)p.tmp_o)[((int64_t)tile * p.num_heads + h0 + g) * D + d] = from_float<T>(val);
      if (d == 0) p.tmp_lse[(int64_t)tile * p.num_heads + h0 + g] = (L > 0.f) ? M + __logf(L) : -INFINITY;
    } else {
      ((T *)p.out)[((int64_t)seq * p.num_heads + h0 + g) * D + d] = from_float<T>(val);
    }
  }

  if constexpr (FUSED) {
    if (partial) {
      // last tile of this (sequence, kv head, sub-group) merges the partials in place of a
      // second launch.  counters are zero on entry and left zero.
      const int t0 = p.o_indptr[seq], t1 = p.o_indptr[seq + 1];
      __threadfence();
      __syncthreads();
      if (tid == 0) {
        int *ctr = p.counters + ((int64_t)seq * p.num_kv_heads + kvh) * gridDim.z + blockIdx.z;
        const int old = atomicAdd(ctr, 1);
        sm_last = (old == (t1 - t0) - 1);
        if (sm_last) *ctr = 0;
      }
      __syncthreads();
      if (sm_last) {
        __threadfence();
        for (int idx = tid; idx < G * D; idx += PA_THREADS) {
          const int g = idx / D, d = idx % D;
          if (g >= gsize) continue;
          const int h = h0 + g;
          float M = -INFINITY;
#pragma unroll 4
          for (int t = t0; t < t1; t++) M = fmaxf(M, __ldcg(p.tmp_lse + (int64_t)t * p.num_heads + h));
          float W = 0.f, acc = 0.f;
          if (M > -INFINITY) {
#pragma unroll 4
            for (int t = t0; t < t1; t++) {
              const float w = __expf(__ldcg(p.tmp_lse + (int64_t)t * p.num_heads + h) - M);
              const unsigned short raw = __ldcg((const unsigned short *)p.tmp_o + ((int64_t)t * p.num_heads + h) * D + d);
              T tv;
              memcpy(&tv, &raw, 2);
              W += w;
              acc += w * (float)tv;
            }
          }
          ((T *)p.out)[((int64_t)seq * p.num_heads + h) * D + d] = from_float<T>((W > 0.f) ? acc / W : 0.f);
        }
      }
    }
  }
}

// merge split-KV partials: out[s,h,:] = sum_p w_p o_p / sum_p w_p, w_p = exp(lse_p - max lse)
// tiles of sequence s are [o_indptr[s], o_indptr[s+1]) (HND API) or s*P .. s*P+P-1 (vLLM v2)
template <typename T>
__global__ void merge_partials_kernel(const T *__restrict__ tmp_o, const float *__restrict__ tmp_lse,
                                      T *__restrict__ out, const int32_t *__restrict__ o_indptr, int num_partitions,
                                      int num_heads, int D, const float *__restrict__ sinks,
                                      const int32_t *__restrict__ context_lens, int partition_size) {
  const int s = blockIdx.x, h = blockIdx.y;
  int t0, t1;
  if (o_indptr != nullptr) { t0 = o_indptr[s]; t1 = o_indptr[s + 1]; }
  else {
    t0 = s * num_partitions;
    const int np = (context_lens[s] + partition_size - 1) / partition_size;
    t1 = t0 + max(np, 0);
  }
  float M = -INFINITY;
  for (int t = t0; t < t1; t++) M = fmaxf(M, tmp_lse[(int64_t)t * num_heads + h]);
  if (sinks != nullptr) M = fmaxf(M, sinks[h]);
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float W = 0.f, acc = 0.f;
    if (M > -INFINITY) {
      for (int t = t0; t < t1; t++) {
        const float w = __expf(tmp_lse[(int64_t)t * num_heads + h] - M);
        W += w;
        acc += w * (float)tmp_o[((int64_t)t * num_heads + h) * D + d];
      }
      if (sinks != nullptr) W += __expf(sinks[h] - M);
    }
    out[((int64_t)s * num_heads + h) * D + d] = (T)((W > 0.f) ? acc / W : 0.f);
  }
}

}  // namespace mrs
#include "paged_attn_mma.cuh"
namespace mrs {

static int g_pa_flags = 0;   // bit 0: keep HND decode on the SIMT kernel (A/B, debugging)

template <typename K>
static cudaError_t launch_pa(K kern, dim3 grid, const PagedParams &p, cudaStream_t st, size_t dyn_smem, int threads = PA_THREADS) {
  if (dyn_smem > 0) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem);
  return launch_pdl(kern, grid, dim3(threads), dyn_smem, st, p.pdl, p);
}

// the split tiles of one sequence as one thread-block cluster (merge through DSMEM).  Returns false, launching nothing,
// when the device cannot schedule that cluster shape: asked once per shape through `feasible` (0 unknown, 1 yes,
// -1 no), because a failed launch inside a stream capture would poison the capture
template <typename K>
static bool launch_pm_cluster(K kern, dim3 grid, const PagedParams &p, cudaStream_t st, size_t dyn, int *feasible, cudaError_t *err) {
  const int tiles = (int)grid.x;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(PM_THREADS); cfg.dynamicSmemBytes = dyn; cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = tiles; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  if (feasible[tiles] == 0) {
    int ncl = 0;
    const cudaError_t qe = cudaOccupancyMaxActiveClusters(&ncl, kern, &cfg);
    feasible[tiles] = (qe == cudaSuccess && ncl >= 1) ? 1 : -1;
    if (qe != cudaSuccess) (void)cudaGetLastError();
  }
  if (feasible[tiles] != 1) return false;
  cfg.numAttrs = p.pdl ? 2 : 1;
  *err = cudaLaunchKernelEx(&cfg, kern, p);
  return true;
}

template <typename T, typename CT, int D, int LAYOUT, bool FUSED>
static cudaError_t launch_decode_g(PagedParams p, int tiles, cudaStream_t st) {
  const int group = p.num_heads / p.num_kv_heads;
  if constexpr (LAYOUT == 1 && (D == 64 || D == 128) && sizeof(T) == 2 && sizeof(CT) == 2) {
    // HND 16-bit cache: the GQA group is an MMA tile (paged_attn_mma.cuh); ALiBi / sinks are vLLM-layout features
    if (!(g_pa_flags & 1) && p.alibi_slopes == nullptr && p.sinks == nullptr && p.kv_indptr != nullptr && !p.tiles_are_partitions) {
      const int nsub = (group + 15) / 16;
      p.heads_per_cta = (group + nsub - 1) / nsub;
      dim3 grid(tiles, p.num_kv_heads, nsub);
      if constexpr (FUSED) {
        // one sequence split into <= 8 tiles: the tiles form a cluster and merge through DSMEM
        // (batch > 1 plans are compacted per sequence, so a fixed cluster size would straddle sequences)
        if (!(g_pa_flags & 2) && p.tmp_o != nullptr && p.batch_size == 1 && tiles <= PM_CL_MAX && nsub == 1 && p.heads_per_cta <= PM_CL_G) {
          static int feasible[PM_CL_MAX + 1] = {};
          cudaError_t e;
          if (launch_pm_cluster(paged_decode_mma_kernel<T, D, true, true>, grid, p, st, pm_smem_bytes<D>(true, true), feasible, &e)) return e;
        }
      }
      return launch_pa(paged_decode_mma_kernel<T, D, FUSED, false>, grid, p, st, pm_smem_bytes<D>(FUSED, false), PM_THREADS);
    }
  }
  constexpr int GMAX = (D <= 128) ? 8 : (D <= 256 ? 4 : 2);  // static smem budget: 8 states x G x D floats
  const int nsub = (group + GMAX - 1) / GMAX;
  const int per = (group + nsub - 1) / nsub;
  p.heads_per_cta = per;
  dim3 grid(tiles, p.num_kv_heads, nsub);
  // HND: two double-buffered (K, V) sub-chunk stages sized by the cached row (see the kernel)
  constexpr int ROWB = D * (int)sizeof(CT);
  constexpr int SUB = (ROWB <= 256) ? 128 : (ROWB <= 512 ? 64 : 32);
  const size_t dyn = (LAYOUT == 1) ? (size_t)4 * SUB * ROWB : 0;
  if (per <= 1) return launch_pa(paged_decode_kernel<T, CT, D, 1, LAYOUT, FUSED>, grid, p, st, dyn);
  if (per <= 2) return launch_pa(paged_decode_kernel<T, CT, D, 2, LAYOUT, FUSED>, grid, p, st, dyn);
  if constexpr (D <= 256) {
    if (per <= 4) return launch_pa(paged_decode_kernel<T, CT, D, 4, LAYOUT, FUSED>, grid, p, st, dyn);
  }
  if constexpr (D <= 128) return launch_pa(paged_decode_kernel<T, CT, D, 8, LAYOUT, FUSED>, grid, p, st, dyn);
  return cudaErrorInvalidValue;
}

// multi-query fused decode: the MMA rows of a KV head are its group x q_len (query, head) pairs, in slices of <= 16
// over blockIdx.z.  The cluster merge buffer holds a whole 16-row slice (PM_CL_GM), so every one-slice batch-1 split
// plan merges through DSMEM; larger shapes merge through the counter.
template <typename T, int D>
static cudaError_t launch_decode_multi(PagedParams p, int tiles, cudaStream_t st) {
  if (tiles <= 0) return cudaSuccess;
  const int rows = p.num_heads / p.num_kv_heads * p.q_len;
  const int nsub = (rows + 15) / 16;
  p.heads_per_cta = (rows + nsub - 1) / nsub;
  dim3 grid(tiles, p.num_kv_heads, nsub);
  if (!(g_pa_flags & 2) && p.tmp_o != nullptr && p.batch_size == 1 && tiles <= PM_CL_MAX && nsub == 1) {
    static int feasible[PM_CL_MAX + 1] = {};
    cudaError_t e;
    if (launch_pm_cluster(paged_decode_mma_multi_kernel<T, D, true>, grid, p, st, pm_smem_bytes<D>(true, true, PM_CL_GM), feasible, &e)) return e;
  }
  return launch_pa(paged_decode_mma_multi_kernel<T, D, false>, grid, p, st, pm_smem_bytes<D>(true, false), PM_THREADS);
}

// head sizes: REF pagedattention.cuh:718-739 (64, 80, 96, 112, 128, 192, 256) + 512 (flashinfer/mod.rs:262)
template <typename T, typename CT, int LAYOUT, bool FUSED = false>
static cudaError_t launch_decode(const PagedParams &p, int head_size, int tiles, cudaStream_t st) {
  if (tiles <= 0) return cudaSuccess;
  if (p.num_heads % p.num_kv_heads) return cudaErrorInvalidValue;
  switch (head_size) {
  case 64: return launch_decode_g<T, CT, 64, LAYOUT, FUSED>(p, tiles, st);
  case 128: return launch_decode_g<T, CT, 128, LAYOUT, FUSED>(p, tiles, st);
  case 256: return launch_decode_g<T, CT, 256, LAYOUT, FUSED>(p, tiles, st);
  default: break;
  }
  if constexpr (!FUSED) {
    switch (head_size) {
    case 80: return launch_decode_g<T, CT, 80, LAYOUT, false>(p, tiles, st);
    case 96: return launch_decode_g<T, CT, 96, LAYOUT, false>(p, tiles, st);
    case 112: return launch_decode_g<T, CT, 112, LAYOUT, false>(p, tiles, st);
    case 192: return launch_decode_g<T, CT, 192, LAYOUT, false>(p, tiles, st);
    case 512: return launch_decode_g<T, CT, 512, LAYOUT, false>(p, tiles, st);
    default: break;
    }
  }
  return cudaErrorInvalidValue;
}

// dtype: 0 f16, 1 bf16, 2 f32; cache_dtype: same codes, or 3 = FP8-E4M3 bytes (REF ffi.rs dtype codes)
template <int LAYOUT>
static cudaError_t launch_decode_any(const PagedParams &p, uint32_t dtype, uint32_t cache_dtype, int head_size, int tiles, cudaStream_t st) {
  if (cache_dtype == 3) {
    if (dtype == 0) return launch_decode<__half, fp8_t, LAYOUT>(p, head_size, tiles, st);
    if (dtype == 1) return launch_decode<__nv_bfloat16, fp8_t, LAYOUT>(p, head_size, tiles, st);
    if (dtype == 2) return launch_decode<float, fp8_t, LAYOUT>(p, head_size, tiles, st);
    return cudaErrorInvalidValue;
  }
  if (cache_dtype != dtype) return cudaErrorInvalidValue;
  if (dtype == 0) return launch_decode<__half, __half, LAYOUT>(p, head_size, tiles, st);
  if (dtype == 1) return launch_decode<__nv_bfloat16, __nv_bfloat16, LAYOUT>(p, head_size, tiles, st);
  if (dtype == 2) return launch_decode<float, float, LAYOUT>(p, head_size, tiles, st);
  return cudaErrorInvalidValue;
}

}  // namespace mrs

using namespace mrs;

// ---------------------------------------------------------------- flashinfer_decode (HND)
extern "C" int32_t flashinfer_decode(void *q, void *key_cache, void *value_cache, const int32_t *kv_indptr,
                                     const int32_t *kv_indices, const int32_t *kv_last_page_len,
                                     const int32_t *request_indices, const int32_t *kv_tile_indices,
                                     const int32_t *o_indptr, const int32_t *kv_chunk_size_ptr,
                                     const bool *block_valid_mask, void *o, void *tmp_v, void *tmp_s,
                                     int32_t batch_size, int32_t padded_batch_size, int32_t num_qo_heads,
                                     int32_t num_kv_heads, int32_t head_size, int32_t page_size, int32_t q_stride_n,
                                     int32_t q_stride_h, float sm_scale, int32_t window_left, float logits_soft_cap,
                                     float k_scale, float v_scale, uint32_t dtype, uint32_t cache_dtype,
                                     cudaStream_t stream) {
  if (dtype > 2 || (cache_dtype != dtype && cache_dtype != 3)) {
    fprintf(stderr, "mrs_b200: flashinfer_decode: unsupported query / cache dtype codes %u / %u\n", dtype, cache_dtype);
    return (int32_t)cudaErrorInvalidValue;
  }
  PagedParams p = {};
  // FP8-E4M3 cache: k_scale folds into the logits, v_scale into the output (REF flashinfer_decode.cu: sm_scale * k_scale, v_scale)
  p.k_scale = (cache_dtype == 3) ? k_scale : 1.f; p.v_scale = (cache_dtype == 3) ? v_scale : 1.f;
  p.batch_size = batch_size;
  p.q = q; p.kc = key_cache; p.vc = value_cache; p.out = o;
  const bool split = tmp_v != nullptr && padded_batch_size > batch_size;
  p.tmp_o = split ? tmp_v : nullptr; p.tmp_lse = split ? (float *)tmp_s : nullptr;
  p.request_indices = request_indices; p.kv_tile_indices = kv_tile_indices;
  p.block_valid_mask = (const uint8_t *)block_valid_mask;
  p.kv_chunk_size_ptr = split ? kv_chunk_size_ptr : nullptr;  // unsplit plans carry chunk = page_size
  p.kv_chunk_size = 0;
  p.kv_indptr = kv_indptr; p.kv_indices = kv_indices; p.kv_last_page_len = kv_last_page_len;
  p.kv_block_stride = (int64_t)num_kv_heads * page_size * head_size; p.kv_head_stride = (int64_t)page_size * head_size;
  p.num_heads = num_qo_heads; p.num_kv_heads = num_kv_heads; p.page_size = page_size;
  p.q_stride_n = q_stride_n; p.q_stride_h = q_stride_h; p.sm_scale = sm_scale;
  p.softcap = logits_soft_cap; p.window_left = window_left;
  if (!split) {
    // one tile per request, whole context (tile list may still be given: request i, tile 0)
    p.request_indices = nullptr; p.kv_tile_indices = nullptr; p.block_valid_mask = nullptr;
  }
  const int tiles = split ? padded_batch_size : batch_size;
  cudaError_t e = launch_decode_any<1>(p, dtype, cache_dtype, head_size, tiles, stream);
  if (e != cudaSuccess) { fprintf(stderr, "mrs_b200: flashinfer_decode failed: %s\n", cudaGetErrorString(e)); return (int32_t)e; }
  if (split) {
    dim3 grid(batch_size, num_qo_heads);
    if (dtype == 0) merge_partials_kernel<__half><<<grid, 128, 0, stream>>>((const __half *)tmp_v, (const float *)tmp_s, (__half *)o, o_indptr, 0, num_qo_heads, head_size, nullptr, nullptr, 0);
    else if (dtype == 1) merge_partials_kernel<__nv_bfloat16><<<grid, 128, 0, stream>>>((const __nv_bfloat16 *)tmp_v, (const float *)tmp_s, (__nv_bfloat16 *)o, o_indptr, 0, num_qo_heads, head_size, nullptr, nullptr, 0);
    else merge_partials_kernel<float><<<grid, 128, 0, stream>>>((const float *)tmp_v, (const float *)tmp_s, (float *)o, o_indptr, 0, num_qo_heads, head_size, nullptr, nullptr, 0);
    e = cudaGetLastError();
  }
  return (int32_t)e;
}

// ---------------------------------------------------------------- paged_attention v1 / v2 (vLLM)
static void vllm_common(PagedParams &p, void *out, void *query, void *key_cache, void *value_cache, void *alibi,
                        int num_kv_heads, float scale, float softcapping, const int32_t *block_tables,
                        const int32_t *context_lens, int block_size, int num_heads, int head_size,
                        int max_num_blocks_per_seq, int q_stride, int kv_block_stride, int kv_head_stride,
                        const float *sinks) {
  p.q = query; p.kc = key_cache; p.vc = value_cache; p.out = out;
  p.block_tables = block_tables; p.context_lens = context_lens; p.max_blocks_per_seq = max_num_blocks_per_seq;
  p.kv_block_stride = kv_block_stride; p.kv_head_stride = kv_head_stride;
  p.num_heads = num_heads; p.num_kv_heads = num_kv_heads; p.page_size = block_size;
  p.q_stride_n = q_stride; p.q_stride_h = head_size; p.sm_scale = scale;
  p.softcap = (softcapping != 1.0f) ? softcapping : 0.f;  // REF pagedattention.cuh:276-279
  p.window_left = -1; p.alibi_slopes = (const float *)alibi; p.sinks = sinks;
  p.k_scale = 1.f; p.v_scale = 1.f;
}
// FP8 cache: the vLLM-style API hands the per-tensor scales as DEVICE pointers (REF pagedattention.cuh
// `*k_scale`); a one-thread kernel would cost a launch, so the attention kernel reads them itself
static void vllm_scales(PagedParams &p, uint32_t cache_dtype, const float *k_scale, const float *v_scale) {
  p.k_scale_ptr = (cache_dtype == 3) ? k_scale : nullptr;
  p.v_scale_ptr = (cache_dtype == 3) ? v_scale : nullptr;
}

static void die_if(cudaError_t e, const char *what) {
  if (e != cudaSuccess) {  // REF pagedattention.cuh:46-56: report and exit
    fprintf(stderr, "mrs_b200: %s failed: %s\n", what, cudaGetErrorString(e));
    exit((int)e);
  }
}

static void paged_v1(uint32_t dtype, void *out, void *query, void *key_cache, void *value_cache, void *alibi, int num_kv_heads,
                     float scale, float softcapping, const int32_t *block_tables, const int32_t *context_lens,
                     int block_size, int num_seqs, int num_heads, int head_size, int max_num_blocks_per_seq,
                     int q_stride, int kv_block_stride, int kv_head_stride, cudaStream_t stream, uint32_t cache_dtype,
                     const float *k_scale, const float *v_scale, const float *sinks) {
  PagedParams p = {};
  vllm_common(p, out, query, key_cache, value_cache, alibi, num_kv_heads, scale, softcapping, block_tables,
              context_lens, block_size, num_heads, head_size, max_num_blocks_per_seq, q_stride, kv_block_stride,
              kv_head_stride, sinks);
  vllm_scales(p, cache_dtype, k_scale, v_scale);
  die_if(launch_decode_any<0>(p, dtype, cache_dtype, head_size, num_seqs, stream), "paged_attention_v1");
}

static void paged_v2(uint32_t dtype, void *out, float *exp_sums, float *max_logits, void *tmp_out, void *query, void *key_cache,
                     void *value_cache, void *alibi, int num_kv_heads, float scale, float softcapping,
                     const int32_t *block_tables, const int32_t *context_lens, int block_size, int max_context_len,
                     int num_seqs, int num_heads, int head_size, int max_num_blocks_per_seq, int q_stride,
                     int kv_block_stride, int kv_head_stride, cudaStream_t stream, uint32_t cache_dtype,
                     const float *k_scale, const float *v_scale, const float *sinks) {
  (void)exp_sums;
  constexpr int PARTITION = 512;  // REF backend/paged_attention.rs:302
  const int num_partitions = (max_context_len + PARTITION - 1) / PARTITION;
  PagedParams p = {};
  vllm_common(p, out, query, key_cache, value_cache, alibi, num_kv_heads, scale, softcapping, block_tables,
              context_lens, block_size, num_heads, head_size, max_num_blocks_per_seq, q_stride, kv_block_stride,
              kv_head_stride, nullptr);
  vllm_scales(p, cache_dtype, k_scale, v_scale);
  p.tmp_o = tmp_out; p.tmp_lse = max_logits;  // scratch is opaque to the caller: lse lives in max_logits
  p.kv_chunk_size = PARTITION; p.tiles_are_partitions = 1; p.num_partitions = num_partitions;
  die_if(launch_decode_any<0>(p, dtype, cache_dtype, head_size, num_seqs * num_partitions, stream), "paged_attention_v2");
  dim3 grid(num_seqs, num_heads);
  if (dtype == 0) merge_partials_kernel<__half><<<grid, 128, 0, stream>>>((const __half *)tmp_out, max_logits, (__half *)out, nullptr, num_partitions, num_heads, head_size, sinks, context_lens, PARTITION);
  else if (dtype == 1) merge_partials_kernel<__nv_bfloat16><<<grid, 128, 0, stream>>>((const __nv_bfloat16 *)tmp_out, max_logits, (__nv_bfloat16 *)out, nullptr, num_partitions, num_heads, head_size, sinks, context_lens, PARTITION);
  else merge_partials_kernel<float><<<grid, 128, 0, stream>>>((const float *)tmp_out, max_logits, (float *)out, nullptr, num_partitions, num_heads, head_size, sinks, context_lens, PARTITION);
  die_if(cudaGetLastError(), "paged_attention_v2 reduce");
}

#define MRS_PAGED(tag, DT)                                                                                      \
  extern "C" void paged_attention_v1_##tag(void *out, void *query, void *key_cache, void *value_cache,          \
      void *alibi_slopes, int32_t num_kv_heads, float scale, float softcapping, uint32_t *block_tables,         \
      uint32_t *context_lens, int32_t block_size, int32_t max_context_len, int32_t num_seqs, int32_t num_heads, \
      int32_t head_size, int32_t max_num_blocks_per_seq, int32_t q_stride, int32_t kv_block_stride,             \
      int32_t kv_head_stride, cudaStream_t stream, uint32_t cache_dtype, float *k_scale, float *v_scale,        \
      const float *sinks) {                                                                                     \
    (void)max_context_len;                                                                                      \
    paged_v1(DT, out, query, key_cache, value_cache, alibi_slopes, num_kv_heads, scale, softcapping,            \
             (const int32_t *)block_tables, (const int32_t *)context_lens, block_size, num_seqs, num_heads,     \
             head_size, max_num_blocks_per_seq, q_stride, kv_block_stride, kv_head_stride, stream,              \
             cache_dtype, k_scale, v_scale, sinks);                                                             \
  }                                                                                                             \
  extern "C" void paged_attention_v2_##tag(void *out, float *exp_sums, float *max_logits, void *tmp_out,        \
      void *query, void *key_cache, void *value_cache, void *alibi_slopes, int32_t num_kv_heads, float scale,   \
      float softcapping, uint32_t *block_tables, uint32_t *context_lens, int32_t block_size,                    \
      int32_t max_context_len, int32_t num_seqs, int32_t num_heads, int32_t head_size,                          \
      int32_t max_num_blocks_per_seq, int32_t q_stride, int32_t kv_block_stride, int32_t kv_head_stride,        \
      cudaStream_t stream, uint32_t cache_dtype, float *k_scale, float *v_scale, const float *sinks) {          \
    paged_v2(DT, out, exp_sums, max_logits, tmp_out, query, key_cache, value_cache, alibi_slopes, num_kv_heads, \
             scale, softcapping, (const int32_t *)block_tables, (const int32_t *)context_lens, block_size,      \
             max_context_len, num_seqs, num_heads, head_size, max_num_blocks_per_seq, q_stride,                 \
             kv_block_stride, kv_head_stride, stream, cache_dtype, k_scale, v_scale, sinks);                    \
  }
MRS_PAGED(f16, 0u)
MRS_PAGED(bf16, 1u)
MRS_PAGED(f32, 2u)

// ---------------------------------------------------------------- native fused decode attention
// the PagedParams of the fused decode entry points; the split-KV tiles (tmp_o != nullptr) are used only when the plan
// has more tiles than sequences
static PagedParams fused_decode_params(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                                       const void *rope_cos, const void *rope_sin, const int32_t *positions,
                                       const int64_t *slot_mapping, const int32_t *kv_indptr, const int32_t *kv_indices,
                                       const int32_t *kv_last_page_len, const int32_t *request_indices,
                                       const int32_t *kv_tile_indices, const int32_t *o_indptr,
                                       const int32_t *kv_chunk_size_ptr, const uint8_t *block_valid_mask, void *o,
                                       void *tmp_v, float *tmp_s, int32_t *counters, int32_t batch_size,
                                       int32_t padded_batch_size, int32_t num_qo_heads, int32_t num_kv_heads,
                                       int32_t head_size, int32_t page_size, float sm_scale, int32_t pdl,
                                       int64_t q_stride_n, int64_t kv_new_stride) {
  PagedParams p = {};
  p.q = q; p.kc = key_cache; p.vc = value_cache; p.out = o;
  const bool split = tmp_v != nullptr && padded_batch_size > batch_size;
  p.tmp_o = split ? tmp_v : nullptr; p.tmp_lse = split ? tmp_s : nullptr;
  if (split) {
    p.request_indices = request_indices; p.kv_tile_indices = kv_tile_indices;
    p.block_valid_mask = block_valid_mask; p.kv_chunk_size_ptr = kv_chunk_size_ptr;
  }
  p.kv_indptr = kv_indptr; p.kv_indices = kv_indices; p.kv_last_page_len = kv_last_page_len;
  p.kv_block_stride = (int64_t)num_kv_heads * page_size * head_size; p.kv_head_stride = (int64_t)page_size * head_size;
  p.num_heads = num_qo_heads; p.num_kv_heads = num_kv_heads; p.page_size = page_size;
  p.q_stride_n = q_stride_n; p.q_stride_h = head_size; p.sm_scale = sm_scale;
  p.window_left = -1; p.pdl = pdl & 1; p.rope_interleaved = (pdl >> 1) & 1;
  p.k_new = k_new; p.v_new = v_new; p.kv_new_stride = kv_new_stride;
  p.rope_cos = rope_cos; p.rope_sin = rope_sin; p.positions = positions; p.slot_mapping = slot_mapping;
  p.o_indptr = o_indptr; p.counters = counters; p.batch_size = batch_size;
  p.k_scale = 1.f; p.v_scale = 1.f;
  return p;
}

// RoPE(q, k_new) + KV-cache write + paged decode attention + split-KV merge in ONE launch over
// the HND cache.  q [B, H*D], k_new/v_new [B, KVH*D] are the raw QKV GEMV outputs; cos/sin
// [max_pos, D/2]; positions [B] i32; slot_mapping [B] i64; counters: zeroed int32
// [B * KVH * ceil(group/8)] scratch (left zero).  `pdl`: bit 0 = launched with programmatic stream
// serialisation, bit 1 = interleaved RoPE pairing (GGUF llama files; default rotate-half).  Same arithmetic as the separate
// rotary_embedding_positions -> reshape_and_cache_flashinfer -> flashinfer_decode chain.
// q rows are q_stride_n elements apart, k_new / v_new rows kv_new_stride (a fused QKV GEMM writes
// [B, (H + 2 KVH) D] and hands three pointers into it)
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
                                          int64_t q_stride_n, int64_t kv_new_stride, void *stream) {
  if (dtype != 0 && dtype != 1) return (int32_t)cudaErrorInvalidValue;
  const PagedParams p = fused_decode_params(q, k_new, v_new, key_cache, value_cache, rope_cos, rope_sin, positions,
                                            slot_mapping, kv_indptr, kv_indices, kv_last_page_len, request_indices,
                                            kv_tile_indices, o_indptr, kv_chunk_size_ptr, block_valid_mask, o, tmp_v, tmp_s,
                                            counters, batch_size, padded_batch_size, num_qo_heads, num_kv_heads, head_size,
                                            page_size, sm_scale, pdl, q_stride_n, kv_new_stride);
  const int tiles = p.tmp_o != nullptr ? padded_batch_size : batch_size;
  const cudaError_t e = (dtype == 0) ? launch_decode<__half, __half, 1, true>(p, head_size, tiles, (cudaStream_t)stream)
                                     : launch_decode<__nv_bfloat16, __nv_bfloat16, 1, true>(p, head_size, tiles, (cudaStream_t)stream);
  if (e != cudaSuccess) fprintf(stderr, "mrs_b200: mrs_paged_decode_fused failed: %s\n", cudaGetErrorString(e));
  return (int32_t)e;
}

extern "C" int32_t mrs_paged_decode_fused(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                                          const void *rope_cos, const void *rope_sin, const int32_t *positions,
                                          const int64_t *slot_mapping, const int32_t *kv_indptr,
                                          const int32_t *kv_indices, const int32_t *kv_last_page_len,
                                          const int32_t *request_indices, const int32_t *kv_tile_indices,
                                          const int32_t *o_indptr, const int32_t *kv_chunk_size_ptr,
                                          const uint8_t *block_valid_mask, void *o, void *tmp_v, float *tmp_s,
                                          int32_t *counters, int32_t batch_size, int32_t padded_batch_size,
                                          int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size,
                                          int32_t page_size, float sm_scale, uint32_t dtype, int32_t pdl,
                                          void *stream) {
  return mrs_paged_decode_fused_strided(q, k_new, v_new, key_cache, value_cache, rope_cos, rope_sin, positions, slot_mapping,
                                        kv_indptr, kv_indices, kv_last_page_len, request_indices, kv_tile_indices, o_indptr,
                                        kv_chunk_size_ptr, block_valid_mask, o, tmp_v, tmp_s, counters, batch_size,
                                        padded_batch_size, num_qo_heads, num_kv_heads, head_size, page_size, sm_scale, dtype,
                                        pdl, (int64_t)num_qo_heads * head_size, (int64_t)num_kv_heads * head_size, stream);
}

// Multi-query form of mrs_paged_decode_fused (speculative verify): q_len rows per sequence at positions
// kv_len - q_len .. kv_len - 1, laid out [B * q_len, ...] in q / k_new / v_new / positions / slot_mapping / o;
// partials tmp_v / tmp_s [padded_batch_size, q_len * num_qo_heads]; counters [B * KVH * ceil(group * q_len / 16)].
// Head size 64 | 128, q_len 1..8, 16-bit dtypes.  A sequence needs kv_len >= q_len.
// q rows are q_stride_n elements apart, k_new / v_new rows kv_new_stride (the [B * q_len, (H + 2 KVH) D] rows of a
// fused QKV GEMM, as for mrs_paged_decode_fused_strided); o stays contiguous
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
                                                        void *stream) {
  if ((dtype != 0 && dtype != 1) || (head_size != 64 && head_size != 128) || q_len < 1 || q_len > 8 || num_kv_heads < 1 ||
      num_qo_heads % num_kv_heads)
    return (int32_t)cudaErrorInvalidValue;
  PagedParams p = fused_decode_params(q, k_new, v_new, key_cache, value_cache, rope_cos, rope_sin, positions, slot_mapping,
                                      kv_indptr, kv_indices, kv_last_page_len, request_indices, kv_tile_indices,
                                      o_indptr, kv_chunk_size_ptr, block_valid_mask, o, tmp_v, tmp_s, counters,
                                      batch_size, padded_batch_size, num_qo_heads, num_kv_heads, head_size,
                                      page_size, sm_scale, pdl, q_stride_n, kv_new_stride);
  p.q_len = q_len;
  const int tiles = p.tmp_o != nullptr ? padded_batch_size : batch_size;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e;
  if (dtype == 0) e = head_size == 64 ? launch_decode_multi<__half, 64>(p, tiles, st) : launch_decode_multi<__half, 128>(p, tiles, st);
  else e = head_size == 64 ? launch_decode_multi<__nv_bfloat16, 64>(p, tiles, st) : launch_decode_multi<__nv_bfloat16, 128>(p, tiles, st);
  if (e != cudaSuccess) fprintf(stderr, "mrs_b200: mrs_paged_decode_fused_multi failed: %s\n", cudaGetErrorString(e));
  return (int32_t)e;
}

extern "C" int32_t mrs_paged_decode_fused_multi(void *q, void *k_new, void *v_new, void *key_cache, void *value_cache,
                                                const void *rope_cos, const void *rope_sin, const int32_t *positions,
                                                const int64_t *slot_mapping, const int32_t *kv_indptr,
                                                const int32_t *kv_indices, const int32_t *kv_last_page_len,
                                                const int32_t *request_indices, const int32_t *kv_tile_indices,
                                                const int32_t *o_indptr, const int32_t *kv_chunk_size_ptr,
                                                const uint8_t *block_valid_mask, void *o, void *tmp_v, float *tmp_s,
                                                int32_t *counters, int32_t batch_size, int32_t padded_batch_size,
                                                int32_t num_qo_heads, int32_t num_kv_heads, int32_t head_size,
                                                int32_t page_size, float sm_scale, uint32_t dtype, int32_t pdl,
                                                int32_t q_len, void *stream) {
  return mrs_paged_decode_fused_multi_strided(q, k_new, v_new, key_cache, value_cache, rope_cos, rope_sin, positions,
                                              slot_mapping, kv_indptr, kv_indices, kv_last_page_len, request_indices,
                                              kv_tile_indices, o_indptr, kv_chunk_size_ptr, block_valid_mask, o, tmp_v, tmp_s,
                                              counters, batch_size, padded_batch_size, num_qo_heads, num_kv_heads, head_size,
                                              page_size, sm_scale, dtype, pdl, q_len, (int64_t)num_qo_heads * head_size,
                                              (int64_t)num_kv_heads * head_size, stream);
}

// bit 0: keep HND decode attention on the SIMT kernel instead of the tensor-core one; bit 1: no cluster/DSMEM
// merge of split-KV tiles (A/B, debugging)
extern "C" void mrs_set_attn_flags(int32_t flags) { mrs::g_pa_flags = flags; }
