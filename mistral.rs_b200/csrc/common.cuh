// common.cuh — shared device helpers for the sm_90a hot-path kernels.
//
// Block layouts follow the ggml formats the reference consumes
// (REF: mistralrs-quant/kernels/mmvq_gguf/mmvq_gguf.cu:134-225).  Everything here is
// written for sm_90a only: mbarrier + cp.async.bulk (TMA engine, SASS UBLKCP), PDL
// (griddepcontrol), 32-wide shuffles.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define MRS_WARP 32

// host: return a failing call's error code from the enclosing function, naming the call on stderr
#define MRS_TRY(expr)                                               \
  do {                                                              \
    const int _e = (int)(expr);                                     \
    if (_e != 0) {                                                  \
      fprintf(stderr, "mrs_b200: %s -> cudaError %d\n", #expr, _e); \
      return _e;                                                    \
    }                                                               \
  } while (0)

// host: launch `kernel` on `stream`, as a programmatic dependent of the previous launch when `pdl` is set
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     bool pdl, Args &&...args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<Args &&>(args)...);
}

// ggml dtype codes (candle GgmlDType numbering used by the reference's Rust side)
enum : int {
  MRS_Q4_0 = 2, MRS_Q4_1 = 3, MRS_Q5_0 = 6, MRS_Q5_1 = 7, MRS_Q8_0 = 8, MRS_Q8_1 = 9,
  MRS_Q2_K = 10, MRS_Q3_K = 11, MRS_Q4_K = 12, MRS_Q5_K = 13, MRS_Q6_K = 14
};
// activation dtype codes of the reference C ABI (paged-attn ffi.rs / rotary ffi.rs)
enum : int { MRS_F16 = 0, MRS_BF16 = 1, MRS_F32 = 2 };

// block_q8_1: REF mmvq_gguf.cu:146-152
struct __align__(4) block_q8_1 {
  __half2 ds;
  int8_t qs[32];
};
static_assert(sizeof(block_q8_1) == 36, "q8_1 layout");

// ---------------------------------------------------------------- small utilities
__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) x += __shfl_xor_sync(0xffffffffu, x, m);
  return x;
}
__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, m));
  return x;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// dtype-generic loads/stores of activations (dtype codes above)
__device__ __forceinline__ float load_act(const void *p, int64_t i, int dtype) {
  if (dtype == MRS_BF16) return __bfloat162float(((const __nv_bfloat16 *)p)[i]);
  if (dtype == MRS_F16) return __half2float(((const __half *)p)[i]);
  return ((const float *)p)[i];
}
__device__ __forceinline__ void store_act(void *p, int64_t i, float v, int dtype) {
  if (dtype == MRS_BF16) ((__nv_bfloat16 *)p)[i] = __float2bfloat16_rn(v);
  else if (dtype == MRS_F16) ((__half *)p)[i] = __float2half_rn(v);
  else ((float *)p)[i] = v;
}
// 8 consecutive activations (index multiple of 8): one 16-byte load for the 16-bit dtypes
__device__ __forceinline__ void load_act8(const void *p, int64_t i, int dtype, float *out) {
  if (dtype == MRS_BF16) {
    const uint4 v = *(const uint4 *)((const __nv_bfloat16 *)p + i);
    const __nv_bfloat162 *h = (const __nv_bfloat162 *)&v;
#pragma unroll
    for (int k = 0; k < 4; k++) { const float2 t = __bfloat1622float2(h[k]); out[2 * k] = t.x; out[2 * k + 1] = t.y; }
  } else if (dtype == MRS_F16) {
    const uint4 v = *(const uint4 *)((const __half *)p + i);
    const __half2 *h = (const __half2 *)&v;
#pragma unroll
    for (int k = 0; k < 4; k++) { const float2 t = __half22float2(h[k]); out[2 * k] = t.x; out[2 * k + 1] = t.y; }
  } else {
    const float4 a = *(const float4 *)((const float *)p + i), b = *(const float4 *)((const float *)p + i + 4);
    out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w; out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
  }
}
// 8 activations of a 16-bit dtype already held as one 16-byte register quad
__device__ __forceinline__ void unpack_act8(const uint4 &v, int dtype, float *out) {
  if (dtype == MRS_BF16) {
    const __nv_bfloat162 *h = (const __nv_bfloat162 *)&v;
#pragma unroll
    for (int k = 0; k < 4; k++) { const float2 t = __bfloat1622float2(h[k]); out[2 * k] = t.x; out[2 * k + 1] = t.y; }
  } else {
    const __half2 *h = (const __half2 *)&v;
#pragma unroll
    for (int k = 0; k < 4; k++) { const float2 t = __half22float2(h[k]); out[2 * k] = t.x; out[2 * k + 1] = t.y; }
  }
}
// round an f32 through the activation dtype (what materialising a tensor would do)
__device__ __forceinline__ float round_act(float v, int dtype) {
  if (dtype == MRS_BF16) return __bfloat162float(__float2bfloat16_rn(v));
  if (dtype == MRS_F16) return __half2float(__float2half_rn(v));
  return v;
}

// GLU activations with the reference's --use_fast_math semantics made explicit
// (REF: mmvq_gguf.cu:52-88, ops.cu:806-847; build flag mistralrs-quant/build.rs:38).
__device__ __forceinline__ float glu_activation(float x, int act) {
  switch (act) {
  case 1: {  // GELU tanh approximation
    const float x3 = x * x * x;
    const float inner = 0.7978845608f * (x + 0.044715f * x3);
    float th;  // the reference's tanhf under --use_fast_math is tanh.approx.f32
    asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(inner));
    return 0.5f * x * (1.0f + th);
  }
  case 2: return fmaxf(x, 0.0f);
  case 3: return x * normcdff(x);
  case 4: return __fdividef(1.0f, 1.0f + __expf(-x));
  case 0:
  default: return __fdividef(x, 1.0f + __expf(-x));
  }
}

// ---------------------------------------------------------------- mbarrier / bulk copy / PDL
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra.uni WAIT_DONE;\n\t"
      "bra.uni WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D bulk async copy global -> shared through the TMA engine; completion counted in bytes
// on `bar`.  src/dst/bytes must all be multiples of 16.
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes,
                                         uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// Programmatic dependent launch: wait for the producer grid's memory / let dependents start.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// explicit shared-space accesses through 32-bit shared addresses: a pointer derived from a kernel's dynamic
// shared memory by byte arithmetic is "generic" to the compiler (SASS LD.E / ST.E with an address-space
// check, accounted as long-scoreboard traffic); these force LDS / STS
__device__ __forceinline__ uint4 lds128(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
  return v;
}
__device__ __forceinline__ uint32_t lds_u16s(uint32_t saddr) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(saddr));
  return (uint32_t)v;
}
__device__ __forceinline__ void sts128(uint32_t saddr, const uint4 &v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory");
}

// unaligned 32-bit read from shared memory (addr has any byte alignment)
__device__ __forceinline__ uint32_t lds_u32_unaligned(const uint8_t *p) {
  const uintptr_t a = (uintptr_t)p;
  const uint32_t *w = (const uint32_t *)(a & ~(uintptr_t)3);
  const uint32_t sh = (uint32_t)(a & 3) * 8;
  return __funnelshift_r(w[0], w[1], sh);
}
// n consecutive unaligned words: n+1 aligned loads + n funnel shifts
template <int N>
__device__ __forceinline__ void lds_words_unaligned(const uint8_t *p, uint32_t (&out)[N]) {
  const uintptr_t a = (uintptr_t)p;
  const uint32_t *w = (const uint32_t *)(a & ~(uintptr_t)3);
  const uint32_t sh = (uint32_t)(a & 3) * 8;
  uint32_t t[N + 1];
#pragma unroll
  for (int i = 0; i <= N; i++) t[i] = w[i];
#pragma unroll
  for (int i = 0; i < N; i++) out[i] = __funnelshift_r(t[i], t[i + 1], sh);
}
// 16-bit read from shared memory: AL = 2-byte aligned, otherwise any byte alignment (a weight row at an odd address)
template <bool AL> __device__ __forceinline__ uint32_t lds_u16(const uint8_t *p) {
  if constexpr (AL) return *(const uint16_t *)p;
  else return (uint32_t)p[0] | ((uint32_t)p[1] << 8);
}

__device__ __forceinline__ float half_bits_to_float(uint32_t h16) {
  return __half2float(__ushort_as_half((unsigned short)h16));
}
