// cache_ops.cu — paged KV-cache data movement behind the reference's C symbols
// (REF: mistralrs-paged-attn/src/cuda/ffi.rs:96-116,159-176,212-268 and the kernels in
//  reshape_and_cache_kernel.cu:32-87, flashinfer_decode.cu:20-100, gather_kv_cache_kernel.cu,
//  copy_blocks_kernel.cu).
//
// Two cache layouts, both the reference's:
//   vLLM      K [NB, KVH, D/x, BS, x]   V [NB, KVH, D, BS]
//   HND       K,V [NB, KVH, BS, D]      (FlashInfer; the default for Llama/Mistral shapes)
// dtype codes 0=f16 1=bf16 2=f32 3=fp8_e4m3 (cache only).  16-bit types are moved as raw
// uint16 (bit-exact); FP8 follows the reference's scaled conversion.
#include "common.cuh"

#include <cuda_fp8.h>
#include <stdio.h>
#include <stdlib.h>

namespace mrs {

template <typename T> struct Conv;
template <> struct Conv<uint16_t> {  // raw 16-bit (f16 or bf16: pure copy)
  __device__ static __forceinline__ uint16_t id(uint16_t v) { return v; }
};

// value -> float for the fp8 paths
template <int DT> __device__ __forceinline__ float widen(const void *p, int64_t i) {
  if constexpr (DT == MRS_F16) return __half2float(((const __half *)p)[i]);
  else if constexpr (DT == MRS_BF16) return __bfloat162float(((const __nv_bfloat16 *)p)[i]);
  else return ((const float *)p)[i];
}
template <int DT> __device__ __forceinline__ void narrow(void *p, int64_t i, float v) {
  if constexpr (DT == MRS_F16) ((__half *)p)[i] = __float2half_rn(v);
  else if constexpr (DT == MRS_BF16) ((__nv_bfloat16 *)p)[i] = __float2bfloat16_rn(v);
  else ((float *)p)[i] = v;
}

// ---------------------------------------------------------------- reshape_and_cache
// LAYOUT 0 vLLM, 1 HND.  ESZ: element bytes of a same-dtype copy (2 or 4); FP8: cache is e4m3.
template <int LAYOUT, typename E>
__global__ void reshape_and_cache_copy(const E *__restrict__ key, const E *__restrict__ value, E *__restrict__ kc,
                                       E *__restrict__ vc, const int64_t *__restrict__ slot_mapping, int key_stride,
                                       int value_stride, int num_heads, int head_size, int block_size, int x) {
  const int64_t t = blockIdx.x;
  const int64_t slot = slot_mapping[t];
  if (slot < 0) return;  // padding token (REF reshape_and_cache_kernel.cu:45-48)
  const int64_t blk = slot / block_size, off = slot % block_size;
  const int n = num_heads * head_size;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int h = i / head_size, d = i - h * head_size;
    int64_t ki, vi;
    if constexpr (LAYOUT == 0) {
      ki = blk * num_heads * head_size * block_size + (int64_t)h * head_size * block_size +
           (int64_t)(d / x) * block_size * x + off * x + (d % x);
      vi = blk * num_heads * head_size * block_size + (int64_t)h * head_size * block_size + (int64_t)d * block_size + off;
    } else {
      ki = vi = ((blk * num_heads + h) * block_size + off) * head_size + d;
    }
    kc[ki] = key[t * key_stride + i];
    vc[vi] = value[t * value_stride + i];
  }
}

template <int LAYOUT, int DT>
__global__ void reshape_and_cache_fp8(const void *__restrict__ key, const void *__restrict__ value,
                                      __nv_fp8_e4m3 *__restrict__ kc, __nv_fp8_e4m3 *__restrict__ vc,
                                      const int64_t *__restrict__ slot_mapping, int key_stride, int value_stride,
                                      int num_heads, int head_size, int block_size, int x, float k_scale, float v_scale,
                                      const float *k_scale_p, const float *v_scale_p) {
  const int64_t t = blockIdx.x;
  const int64_t slot = slot_mapping[t];
  if (slot < 0) return;
  if (k_scale_p != nullptr) { k_scale = *k_scale_p; v_scale = *v_scale_p; }
  const int64_t blk = slot / block_size, off = slot % block_size;
  const int n = num_heads * head_size;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int h = i / head_size, d = i - h * head_size;
    int64_t ki, vi;
    if constexpr (LAYOUT == 0) {
      ki = blk * num_heads * head_size * block_size + (int64_t)h * head_size * block_size +
           (int64_t)(d / x) * block_size * x + off * x + (d % x);
      vi = blk * num_heads * head_size * block_size + (int64_t)h * head_size * block_size + (int64_t)d * block_size + off;
    } else {
      ki = vi = ((blk * num_heads + h) * block_size + off) * head_size + d;
    }
    kc[ki] = __nv_fp8_e4m3(widen<DT>(key, t * key_stride + i) / k_scale);
    vc[vi] = __nv_fp8_e4m3(widen<DT>(value, t * value_stride + i) / v_scale);
  }
}

template <int LAYOUT>
static void launch_reshape_and_cache(void *key, void *value, void *kc, void *vc, const int64_t *slot_mapping,
                                     int num_tokens, int num_heads, int head_size, int block_size, int x,
                                     int key_stride, int value_stride, uint32_t dtype, uint32_t cache_dtype,
                                     float k_scale, float v_scale, const float *ksp, const float *vsp,
                                     cudaStream_t st) {
  if (num_tokens <= 0) return;
  dim3 grid(num_tokens);
  int threads = num_heads * head_size;
  threads = threads < 512 ? ((threads + 31) / 32) * 32 : 512;
  if (cache_dtype == 3) {
    auto K = (__nv_fp8_e4m3 *)kc;
    auto V = (__nv_fp8_e4m3 *)vc;
    if (dtype == 0) reshape_and_cache_fp8<LAYOUT, MRS_F16><<<grid, threads, 0, st>>>(key, value, K, V, slot_mapping, key_stride, value_stride, num_heads, head_size, block_size, x, k_scale, v_scale, ksp, vsp);
    else if (dtype == 1) reshape_and_cache_fp8<LAYOUT, MRS_BF16><<<grid, threads, 0, st>>>(key, value, K, V, slot_mapping, key_stride, value_stride, num_heads, head_size, block_size, x, k_scale, v_scale, ksp, vsp);
    else if (dtype == 2) reshape_and_cache_fp8<LAYOUT, MRS_F32><<<grid, threads, 0, st>>>(key, value, K, V, slot_mapping, key_stride, value_stride, num_heads, head_size, block_size, x, k_scale, v_scale, ksp, vsp);
  } else if (dtype == cache_dtype && (dtype == 0 || dtype == 1)) {
    reshape_and_cache_copy<LAYOUT, uint16_t><<<grid, threads, 0, st>>>((const uint16_t *)key, (const uint16_t *)value, (uint16_t *)kc, (uint16_t *)vc, slot_mapping, key_stride, value_stride, num_heads, head_size, block_size, x);
  } else if (dtype == 2 && cache_dtype == 2) {
    reshape_and_cache_copy<LAYOUT, uint32_t><<<grid, threads, 0, st>>>((const uint32_t *)key, (const uint32_t *)value, (uint32_t *)kc, (uint32_t *)vc, slot_mapping, key_stride, value_stride, num_heads, head_size, block_size, x);
  } else {
    fprintf(stderr, "mrs_b200: reshape_and_cache received unsupported dtype pair %u/%u\n", dtype, cache_dtype);
  }
}

// ---------------------------------------------------------------- gather (paged -> dense)
// One block per output token; cu_seq_lens [num_seqs+1] locates the sequence
// (REF flashinfer_decode.cu:56-100, gather_kv_cache_kernel.cu).
template <int LAYOUT, typename E>
__global__ void gather_kv_copy(const E *__restrict__ kc, const E *__restrict__ vc, E *__restrict__ k_out,
                               E *__restrict__ v_out, const int32_t *__restrict__ block_table,
                               const int32_t *__restrict__ cu_seq_lens, int num_tokens, int num_seqs, int block_size,
                               int block_table_stride, int num_kv_heads, int head_size, int x) {
  const int t = blockIdx.x;
  if (t >= num_tokens) return;
  int lo = 0, hi = num_seqs;  // largest seq with cu[seq] <= t
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cu_seq_lens[mid] <= t) lo = mid; else hi = mid;
  }
  const int seq = lo;
  const int so = t - cu_seq_lens[seq];
  const int64_t blk = block_table[(int64_t)seq * block_table_stride + so / block_size];
  const int off = so % block_size;
  const int n = num_kv_heads * head_size;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int h = i / head_size, d = i - h * head_size;
    int64_t ki, vi;
    if constexpr (LAYOUT == 0) {
      ki = blk * num_kv_heads * head_size * block_size + (int64_t)h * head_size * block_size +
           (int64_t)(d / x) * block_size * x + (int64_t)off * x + (d % x);
      vi = blk * num_kv_heads * head_size * block_size + (int64_t)h * head_size * block_size + (int64_t)d * block_size + off;
    } else {
      ki = vi = ((blk * num_kv_heads + h) * block_size + off) * head_size + d;
    }
    k_out[(int64_t)t * n + i] = kc[ki];
    v_out[(int64_t)t * n + i] = vc[vi];
  }
}

template <int LAYOUT, int DT>
__global__ void gather_kv_fp8(const __nv_fp8_e4m3 *__restrict__ kc, const __nv_fp8_e4m3 *__restrict__ vc,
                              void *__restrict__ k_out, void *__restrict__ v_out,
                              const int32_t *__restrict__ block_table, const int32_t *__restrict__ cu_seq_lens,
                              int num_tokens, int num_seqs, int block_size, int block_table_stride, int num_kv_heads,
                              int head_size, int x, float k_scale, float v_scale, const float *k_scale_p,
                              const float *v_scale_p) {
  const int t = blockIdx.x;
  if (t >= num_tokens) return;
  if (k_scale_p != nullptr) { k_scale = *k_scale_p; v_scale = *v_scale_p; }
  int lo = 0, hi = num_seqs;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cu_seq_lens[mid] <= t) lo = mid; else hi = mid;
  }
  const int seq = lo;
  const int so = t - cu_seq_lens[seq];
  const int64_t blk = block_table[(int64_t)seq * block_table_stride + so / block_size];
  const int off = so % block_size;
  const int n = num_kv_heads * head_size;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int h = i / head_size, d = i - h * head_size;
    int64_t ki, vi;
    if constexpr (LAYOUT == 0) {
      ki = blk * num_kv_heads * head_size * block_size + (int64_t)h * head_size * block_size +
           (int64_t)(d / x) * block_size * x + (int64_t)off * x + (d % x);
      vi = blk * num_kv_heads * head_size * block_size + (int64_t)h * head_size * block_size + (int64_t)d * block_size + off;
    } else {
      ki = vi = ((blk * num_kv_heads + h) * block_size + off) * head_size + d;
    }
    narrow<DT>(k_out, (int64_t)t * n + i, (float)kc[ki] * k_scale);
    narrow<DT>(v_out, (int64_t)t * n + i, (float)vc[vi] * v_scale);
  }
}

template <int LAYOUT>
static void launch_gather(void *kc, void *vc, void *k_out, void *v_out, const int32_t *block_table,
                          const int32_t *cu_seq_lens, int num_tokens, int num_seqs, int block_size,
                          int block_table_stride, int num_kv_heads, int head_size, int x, uint32_t out_dtype,
                          uint32_t cache_dtype, float k_scale, float v_scale, const float *ksp, const float *vsp,
                          cudaStream_t st) {
  if (num_tokens <= 0) return;
  dim3 grid(num_tokens);
  int threads = num_kv_heads * head_size;
  threads = threads < 512 ? ((threads + 31) / 32) * 32 : 512;
  if (cache_dtype == 3) {
    auto K = (const __nv_fp8_e4m3 *)kc;
    auto V = (const __nv_fp8_e4m3 *)vc;
    if (out_dtype == 0) gather_kv_fp8<LAYOUT, MRS_F16><<<grid, threads, 0, st>>>(K, V, k_out, v_out, block_table, cu_seq_lens, num_tokens, num_seqs, block_size, block_table_stride, num_kv_heads, head_size, x, k_scale, v_scale, ksp, vsp);
    else if (out_dtype == 1) gather_kv_fp8<LAYOUT, MRS_BF16><<<grid, threads, 0, st>>>(K, V, k_out, v_out, block_table, cu_seq_lens, num_tokens, num_seqs, block_size, block_table_stride, num_kv_heads, head_size, x, k_scale, v_scale, ksp, vsp);
    else if (out_dtype == 2) gather_kv_fp8<LAYOUT, MRS_F32><<<grid, threads, 0, st>>>(K, V, k_out, v_out, block_table, cu_seq_lens, num_tokens, num_seqs, block_size, block_table_stride, num_kv_heads, head_size, x, k_scale, v_scale, ksp, vsp);
  } else if (out_dtype == cache_dtype && (out_dtype == 0 || out_dtype == 1)) {
    gather_kv_copy<LAYOUT, uint16_t><<<grid, threads, 0, st>>>((const uint16_t *)kc, (const uint16_t *)vc, (uint16_t *)k_out, (uint16_t *)v_out, block_table, cu_seq_lens, num_tokens, num_seqs, block_size, block_table_stride, num_kv_heads, head_size, x);
  } else if (out_dtype == 2 && cache_dtype == 2) {
    gather_kv_copy<LAYOUT, uint32_t><<<grid, threads, 0, st>>>((const uint32_t *)kc, (const uint32_t *)vc, (uint32_t *)k_out, (uint32_t *)v_out, block_table, cu_seq_lens, num_tokens, num_seqs, block_size, block_table_stride, num_kv_heads, head_size, x);
  } else {
    fprintf(stderr, "mrs_b200: gather_kv_cache received unsupported dtype pair %u/%u\n", out_dtype, cache_dtype);
  }
}

// ---------------------------------------------------------------- copy_blocks (copy-on-write)
// key/value_cache_ptrs: device arrays of per-layer cache base addresses; block_mapping
// [num_pairs, 2] int64 (src, dst).  Grid (layers, pairs) — REF copy_blocks_kernel.cu:1-37.
template <typename E>
__global__ void copy_blocks_kernel(int64_t *key_cache_ptrs, int64_t *value_cache_ptrs,
                                   const int64_t *__restrict__ block_mapping, int numel_key, int numel_value) {
  E *kc = (E *)key_cache_ptrs[blockIdx.x];
  E *vc = (E *)value_cache_ptrs[blockIdx.x];
  const int64_t src = block_mapping[2 * blockIdx.y], dst = block_mapping[2 * blockIdx.y + 1];
  for (int i = threadIdx.x; i < numel_key; i += blockDim.x) kc[dst * numel_key + i] = kc[src * numel_key + i];
  for (int i = threadIdx.x; i < numel_value; i += blockDim.x) vc[dst * numel_value + i] = vc[src * numel_value + i];
}

}  // namespace mrs

using namespace mrs;

extern "C" void reshape_and_cache(void *key, void *value, void *key_cache, void *value_cache, int64_t *slot_mapping,
                                  int32_t num_tokens, int32_t num_heads, int32_t head_size, int32_t block_size,
                                  int32_t x, int32_t key_stride, int32_t value_stride, cudaStream_t stream,
                                  uint32_t dtype, uint32_t cache_dtype, float *k_scale, float *v_scale) {
  // vLLM-layout ABI: FP8 scales are device pointers, dereferenced inside the kernel
  launch_reshape_and_cache<0>(key, value, key_cache, value_cache, slot_mapping, num_tokens, num_heads, head_size,
                              block_size, x, key_stride, value_stride, dtype, cache_dtype, 1.f, 1.f, k_scale, v_scale,
                              stream);
}

extern "C" void reshape_and_cache_flashinfer(void *key, void *value, void *key_cache, void *value_cache,
                                             int64_t *slot_mapping, int32_t num_tokens, int32_t num_heads,
                                             int32_t head_size, int32_t block_size, int32_t key_stride,
                                             int32_t value_stride, float k_scale, float v_scale, uint32_t dtype,
                                             uint32_t cache_dtype, cudaStream_t stream) {
  launch_reshape_and_cache<1>(key, value, key_cache, value_cache, slot_mapping, num_tokens, num_heads, head_size,
                              block_size, 1, key_stride, value_stride, dtype, cache_dtype, k_scale, v_scale, nullptr, nullptr, stream);
}

extern "C" void gather_kv_cache_flashinfer(void *key_cache, void *value_cache, void *k_out, void *v_out,
                                           const int32_t *block_table, const int32_t *cu_seq_lens, int32_t num_tokens,
                                           int32_t num_seqs, int32_t block_size, int32_t block_table_stride,
                                           int32_t num_kv_heads, int32_t head_size, uint32_t out_dtype,
                                           uint32_t cache_dtype, float k_scale, float v_scale, cudaStream_t stream) {
  launch_gather<1>(key_cache, value_cache, k_out, v_out, block_table, cu_seq_lens, num_tokens, num_seqs, block_size,
                   block_table_stride, num_kv_heads, head_size, 1, out_dtype, cache_dtype, k_scale, v_scale, nullptr, nullptr, stream);
}

extern "C" void gather_kv_cache(void *key_cache, void *value_cache, void *k_out, void *v_out, const float *k_scale,
                                const float *v_scale, const int32_t *block_table, const int32_t *cu_seq_lens,
                                int32_t num_tokens, int32_t num_seqs, int32_t block_size, int32_t block_table_stride,
                                int32_t num_kv_heads, int32_t head_size, int32_t x, cudaStream_t stream,
                                uint32_t out_dtype, uint32_t cache_dtype) {
  launch_gather<0>(key_cache, value_cache, k_out, v_out, block_table, cu_seq_lens, num_tokens, num_seqs, block_size,
                   block_table_stride, num_kv_heads, head_size, x, out_dtype, cache_dtype, 1.f, 1.f, k_scale, v_scale,
                   stream);
}

#define MRS_COPY_BLOCKS(tag, E)                                                                              \
  extern "C" void copy_blocks_##tag(int64_t *key_cache_ptrs, int64_t *value_cache_ptrs,                      \
                                    const int64_t *block_mapping, int32_t num_layers, int32_t num_pairs,     \
                                    int32_t numel_per_block_key, int32_t numel_per_block_value,              \
                                    int64_t stream) {                                                        \
    if (num_layers <= 0 || num_pairs <= 0) return;                                                           \
    dim3 grid(num_layers, num_pairs);                                                                        \
    copy_blocks_kernel<E><<<grid, 512, 0, (cudaStream_t)stream>>>(key_cache_ptrs, value_cache_ptrs,          \
                                                                  block_mapping, numel_per_block_key,        \
                                                                  numel_per_block_value);                    \
  }
MRS_COPY_BLOCKS(f32, uint32_t)
MRS_COPY_BLOCKS(f16, uint16_t)
MRS_COPY_BLOCKS(bf16, uint16_t)
MRS_COPY_BLOCKS(u8, uint8_t)

// ---------------------------------------------------------------- update_kv_scales (FP8 scale tracking)
// k_scale = max(k_scale, absmax(k) / 240), same for v — REF update_kvscales.cu:45-124 (one scalar per
// cache; 240 leaves headroom below e4m3's 448).  Here: 16-byte loads where the pointers allow, shuffle
// + shared-memory reduction, and one integer atomicMax per CTA (non-negative floats order like their
// bit patterns) instead of the reference's CAS loop.  NaNs are ignored, as in the reference's `>` scan;
// the reference is built with --use_fast_math, hence the approximate division.
template <typename T> __device__ __forceinline__ float kv_abs(T x);
template <> __device__ __forceinline__ float kv_abs<float>(float x) { return fabsf(x); }
template <> __device__ __forceinline__ float kv_abs<__half>(__half x) { return fabsf(__half2float(x)); }
template <> __device__ __forceinline__ float kv_abs<__nv_bfloat16>(__nv_bfloat16 x) { return fabsf(__bfloat162float(x)); }

template <typename T>
__device__ __forceinline__ float absmax_stream(const T *__restrict__ p, int64_t n, int64_t tid, int64_t nthreads) {
  constexpr int VEC = 16 / (int)sizeof(T);
  float m = 0.f;
  int64_t head = 0;  // elements before the first 16-byte boundary
  const uintptr_t mis = (uintptr_t)p & 15;
  if (mis) head = (int64_t)((16 - mis) / sizeof(T));
  if (head > n) head = n;
  for (int64_t i = tid; i < head; i += nthreads) m = fmaxf(m, kv_abs<T>(p[i]));
  const int64_t nvec = (n - head) / VEC;
  const uint4 *pv = (const uint4 *)(p + head);
  for (int64_t i = tid; i < nvec; i += nthreads) {
    const uint4 raw = pv[i];
    const T *e = (const T *)&raw;
#pragma unroll
    for (int k = 0; k < VEC; k++) m = fmaxf(m, kv_abs<T>(e[k]));
  }
  for (int64_t i = head + nvec * VEC + tid; i < n; i += nthreads) m = fmaxf(m, kv_abs<T>(p[i]));
  return m;
}

template <typename T>
__global__ void __launch_bounds__(256) update_kv_scales_kernel(const T *__restrict__ k, const T *__restrict__ v, int64_t n,
                                                                 float *__restrict__ k_scale, float *__restrict__ v_scale) {
  __shared__ float red[2][8];
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (int64_t)gridDim.x * blockDim.x;
  float mk = absmax_stream<T>(k, n, tid, nthreads);
  float mv = absmax_stream<T>(v, n, tid, nthreads);
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    mk = fmaxf(mk, __shfl_xor_sync(0xffffffffu, mk, s));
    mv = fmaxf(mv, __shfl_xor_sync(0xffffffffu, mv, s));
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red[0][warp] = mk; red[1][warp] = mv; }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int w = 1; w < 8; w++) { mk = fmaxf(mk, red[0][w]); mv = fmaxf(mv, red[1][w]); }
    const float ck = __fdividef(mk, 240.0f), cv = __fdividef(mv, 240.0f);
    if (ck > 0.0f) atomicMax((int *)k_scale, __float_as_int(ck));
    if (cv > 0.0f) atomicMax((int *)v_scale, __float_as_int(cv));
  }
}

template <typename T>
static void launch_update_kv_scales(void *k, void *v, long n, float *k_scales, float *v_scales, int64_t stream) {
  if (n <= 0) return;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long blocks = (n + 256 * 16 - 1) / (256 * 16);  // >= 16 elements per thread before adding CTAs
  if (blocks < 1) blocks = 1;
  if (blocks > 8L * sms) blocks = 8L * sms;
  update_kv_scales_kernel<T><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const T *)k, (const T *)v, (int64_t)n,
                                                                              k_scales, v_scales);
}

extern "C" void update_kv_scales_f32(void *k, void *v, const long num_elements, float *k_scales, float *v_scales, int64_t stream) {
  launch_update_kv_scales<float>(k, v, num_elements, k_scales, v_scales, stream);
}
extern "C" void update_kv_scales_f16(void *k, void *v, const long num_elements, float *k_scales, float *v_scales, int64_t stream) {
  launch_update_kv_scales<__half>(k, v, num_elements, k_scales, v_scales, stream);
}
extern "C" void update_kv_scales_bf16(void *k, void *v, const long num_elements, float *k_scales, float *v_scales, int64_t stream) {
  launch_update_kv_scales<__nv_bfloat16>(k, v, num_elements, k_scales, v_scales, stream);
}

// ---------------------------------------------------------------- swap_blocks
// REF backend/cache.rs:194-300 (`swap_blocks`): for every (src_block -> dst_block) copy one cache
// block between two caches on the same device, or between a host cache and a device cache (swap
// out / swap in).  The reference loops over memcpy_dtod / htod / dtoh in Rust; this is the same loop
// behind one C call, asynchronous on `stream` (host memory must be pinned for true overlap).
// pairs: host array [n_pairs][2] of (src_block, dst_block).  Returns a cudaError_t.
extern "C" int32_t mrs_swap_blocks(const void *src, void *dst, int64_t block_bytes, const int64_t *pairs,
                                   int64_t n_pairs, void *stream) {
  if (block_bytes <= 0 || n_pairs < 0 || (n_pairs > 0 && pairs == nullptr)) return (int32_t)cudaErrorInvalidValue;
  for (int64_t i = 0; i < n_pairs; i++) {
    const int64_t s = pairs[2 * i], d = pairs[2 * i + 1];
    if (s < 0 || d < 0) return (int32_t)cudaErrorInvalidValue;
    const cudaError_t e = cudaMemcpyAsync((uint8_t *)dst + d * block_bytes, (const uint8_t *)src + s * block_bytes,
                                          (size_t)block_bytes, cudaMemcpyDefault, (cudaStream_t)stream);
    if (e != cudaSuccess) return (int32_t)e;
  }
  return 0;
}
