// fused_ops.cu — the small elementwise / normalisation ops between the GEMVs, behind the
// reference's C symbols:
//   rotary_embedding, rotary_embedding_positions   REF mistralrs-quant/kernels/rotary/rotary.cu:110-196
//                                                  (ffi: mistralrs-quant/src/rotary/ffi.rs:4-43)
//   fused_glu_{f16,bf16,f32}, fused_split_glu_*    REF mistralrs-quant/kernels/ops/ops.cu:848-1060
//                                                  (ffi: mistralrs-quant/src/utils/ffi.rs:274-330)
//   add_rms_norm_{f32,f16,bf16}                    REF mistralrs-core/src/cuda/sort.cu:403-461,701-727
//   mrs_rms_norm                                   plain RMSNorm (the reference falls through to
//                                                  candle_nn::ops::rms_norm — core/src/layers.rs:403-413)
// In the decode chain these are normally folded into the GEMV prologue/epilogue
// (mrs_mmvq_fused) or the attention kernel; the standalone launchers exist so the library is a
// drop-in for the reference's FFI and for the prefill path.
#include "common.cuh"

#include <stdio.h>

namespace mrs {

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// products/sums rounded in T at every step, like the scalar_t operators of the reference
template <typename T> __device__ __forceinline__ T mul_t(T a, T b) { return from_f<T>(to_f(a) * to_f(b)); }
template <typename T> __device__ __forceinline__ T add_t(T a, T b) { return from_f<T>(to_f(a) + to_f(b)); }
template <typename T> __device__ __forceinline__ T sub_t(T a, T b) { return from_f<T>(to_f(a) - to_f(b)); }
// a*b + c with ONE rounding in T (native fma.rn.{f16,bf16,f32})
__device__ __forceinline__ float fma_t(float a, float b, float c) { return fmaf(a, b, c); }
__device__ __forceinline__ __half fma_t(__half a, __half b, __half c) { return __hfma(a, b, c); }
__device__ __forceinline__ __nv_bfloat16 fma_t(__nv_bfloat16 a, __nv_bfloat16 b, __nv_bfloat16 c) { return __hfma(a, b, c); }
template <typename T> __device__ __forceinline__ T neg_t(T a) { return from_f<T>(-to_f(a)); }

// ------------------------------------------------------------------ RoPE
template <typename T, bool NEOX>
__device__ __forceinline__ void rope_pair(T *arr, const T *cosp, const T *sinp, int off, int rot_half) {
  const int xi = NEOX ? off : 2 * off;
  const int yi = NEOX ? rot_half + off : 2 * off + 1;
  const T c = cosp[off], s = sinp[off];
  const T x = arr[xi], y = arr[yi];
  // as the reference kernel is compiled (checked against its outputs, tests/golden/ref_golden.npz):
  // the second product is rounded, the first is fused into the add -> fma(x, cos, -T(y*sin))
  arr[xi] = fma_t(x, c, neg_t(mul_t(y, s)));
  arr[yi] = fma_t(y, c, mul_t(x, s));
}

template <typename T, bool NEOX>
__global__ void rotary_kernel(T *__restrict__ q, T *__restrict__ k, const T *__restrict__ cosb,
                              const T *__restrict__ sinb, const uint32_t *__restrict__ positions, int rot_half,
                              int64_t q_stride, int64_t k_stride, int num_heads, int num_kv_heads, int head_size) {
  const int64_t t = blockIdx.x;
  const int64_t pos = positions ? (int64_t)positions[t] : t;
  const T *cp = cosb + pos * rot_half, *sp = sinb + pos * rot_half;
  const int nq = num_heads * rot_half, nk = num_kv_heads * rot_half;
  for (int i = threadIdx.x; i < nq + nk; i += blockDim.x) {
    const bool isq = i < nq;
    const int ii = isq ? i : i - nq;
    const int h = ii / rot_half, off = ii - h * rot_half;
    T *base = isq ? q + t * q_stride + (int64_t)h * head_size : k + t * k_stride + (int64_t)h * head_size;
    rope_pair<T, NEOX>(base, cp, sp, off, rot_half);
  }
}

template <typename T>
static void launch_rotary(void *q, void *k, void *c, void *s, void *pos, int is_neox, int head_size, int64_t tokens,
                          int rot_half, int nh, int nkv, int64_t qs, int64_t ks, cudaStream_t st) {
  if (tokens <= 0) return;
  int threads = (nh + nkv) * rot_half;
  threads = threads < 512 ? ((threads + 31) / 32) * 32 : 512;
  if (is_neox)
    rotary_kernel<T, true><<<(unsigned)tokens, threads, 0, st>>>((T *)q, (T *)k, (const T *)c, (const T *)s,
                                                                  (const uint32_t *)pos, rot_half, qs, ks, nh, nkv, head_size);
  else
    rotary_kernel<T, false><<<(unsigned)tokens, threads, 0, st>>>((T *)q, (T *)k, (const T *)c, (const T *)s,
                                                                   (const uint32_t *)pos, rot_half, qs, ks, nh, nkv, head_size);
}

// ------------------------------------------------------------------ GLU
template <typename T>
__global__ void glu_kernel(const T *__restrict__ a, const T *__restrict__ b, T *__restrict__ out, uint32_t cols,
                           uint32_t a_stride, uint32_t b_stride, uint64_t n, int act, int pdl) {
  if (pdl) { pdl_launch_dependents(); pdl_wait(); }   // inputs come from the upstream kernel; the next one may start its prologue
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t row = i / cols;
  const uint32_t col = (uint32_t)(i - row * cols);
  // activation in f32, cast to T, then the product in T (REF ops.cu:866-870: candle's two-step)
  const T activated = from_f<T>(glu_activation(to_f(a[row * a_stride + col]), act));
  out[i] = mul_t(activated, b[row * b_stride + col]);
}

template <typename T>
static void launch_glu(const void *a, const void *b, void *out, uint32_t rows, uint32_t cols, uint32_t as, uint32_t bs,
                       int act, cudaStream_t st, int pdl = 0) {
  if (rows == 0 || cols == 0) return;
  const uint64_t n = (uint64_t)rows * cols;
  launch_pdl(glu_kernel<T>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, pdl, (const T *)a, (const T *)b, (T *)out,
             cols, as, bs, n, act, pdl);
}

// ------------------------------------------------------------------ RMSNorm
__device__ __forceinline__ float block_sum(float v, float *red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (l < nw) ? red[l] : 0.f;
  t = warp_sum(t);
  return t;
}

// out = T(x * inv_rms * w); when `res` != nullptr: sum = T(x + res) is written to sum_out and
// normalised from its rounded value (REF sort.cu:403-428).
template <typename T>
__global__ void rms_norm_kernel(const T *__restrict__ x, const T *__restrict__ res, const T *__restrict__ w,
                                T *__restrict__ sum_out, T *__restrict__ out, int cols, float eps, int pdl) {
  __shared__ float red[32];
  if (pdl) { pdl_launch_dependents(); pdl_wait(); }
  const int64_t off = (int64_t)blockIdx.x * cols;
  float ss = 0.f;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    float v;
    if (res != nullptr) {
      const T s = from_f<T>(to_f(x[off + c]) + to_f(res[off + c]));
      sum_out[off + c] = s;
      v = to_f(s);
    } else {
      v = to_f(x[off + c]);
    }
    ss += v * v;
  }
  const float inv = rsqrtf(block_sum(ss, red) / (float)cols + eps);
  const T *src = (res != nullptr) ? sum_out : x;
  for (int c = threadIdx.x; c < cols; c += blockDim.x)
    out[off + c] = from_f<T>(to_f(src[off + c]) * inv * to_f(w[c]));
}

template <typename T>
static void launch_rms(const void *x, const void *res, const void *w, void *sum_out, void *out, int rows, int cols,
                       float eps, cudaStream_t st, int pdl = 0) {
  if (rows <= 0 || cols <= 0) return;
  const int block = cols < 1024 ? 128 : 512;
  launch_pdl(rms_norm_kernel<T>, dim3(rows), dim3(block), 0, st, pdl, (const T *)x, (const T *)res, (const T *)w,
             (T *)sum_out, (T *)out, cols, eps, pdl);
}

// rms_norm_kernel with its normed output in the order of an act-order linear: out[j] = (the plain kernel's out)[perm[j]],
// bit for bit (same block size, same per-thread sums, same rounding points); sum_out stays in natural order.  Thread j
// reads element perm[j], which another thread loaded, so the row (the rounded sum when `res` is set) is staged in shared
// memory: x may alias out (the prompt step normalises h in place), and nothing is re-read from global memory.
template <typename T>
__global__ void rms_norm_perm_kernel(const T *x, const T *res, const T *__restrict__ w, const int32_t *__restrict__ perm,
                                     T *sum_out, T *out, int cols, float eps, int pdl) {
  extern __shared__ __align__(16) unsigned char rms_row_smem[];
  T *row = (T *)rms_row_smem;
  __shared__ float red[32];
  if (pdl) { pdl_launch_dependents(); pdl_wait(); }
  const int64_t off = (int64_t)blockIdx.x * cols;
  float ss = 0.f;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    T s;
    if (res != nullptr) {
      s = from_f<T>(to_f(x[off + c]) + to_f(res[off + c]));
      sum_out[off + c] = s;
    } else {
      s = x[off + c];
    }
    row[c] = s;
    const float v = to_f(s);
    ss += v * v;
  }
  // block_sum's barriers also order every row[] store and every read of x before the first store to out
  const float inv = rsqrtf(block_sum(ss, red) / (float)cols + eps);
  for (int j = threadIdx.x; j < cols; j += blockDim.x) {
    const int p = perm[j];
    out[off + j] = from_f<T>(to_f(row[p]) * inv * to_f(w[p]));
  }
}

template <typename T>
static cudaError_t launch_rms_perm(const void *x, const void *res, const void *w, const int32_t *perm, void *sum_out, void *out,
                                   int rows, int cols, float eps, cudaStream_t st, int pdl) {
  if (rows <= 0 || cols <= 0) return cudaSuccess;
  const size_t smem = (size_t)cols * sizeof(T);
  if (perm == nullptr || smem > 48 * 1024) return cudaErrorInvalidValue;
  const int block = cols < 1024 ? 128 : 512;     // as launch_rms: the same reduction, so the same inverse RMS
  return launch_pdl(rms_norm_perm_kernel<T>, dim3(rows), dim3(block), smem, st, pdl, (const T *)x, (const T *)res,
                    (const T *)w, perm, (T *)sum_out, (T *)out, cols, eps, pdl);
}

// y[r, j] = x[r, perm[j]] over 16-bit elements: the activations of an act-order linear whose input no norm produces
__global__ void gather_cols_kernel(const uint16_t *__restrict__ x, const int32_t *__restrict__ perm, uint16_t *__restrict__ y,
                                   int cols, int pdl) {
  if (pdl) { pdl_launch_dependents(); pdl_wait(); }
  const int64_t off = (int64_t)blockIdx.x * cols;
  for (int j = threadIdx.x; j < cols; j += blockDim.x) y[off + j] = x[off + perm[j]];
}

// Per-head RMSNorm of a strided [B, H, S, D] view into a contiguous [B, H, S, D] tensor (QK-norm of
// Qwen3 / Gemma-3 style models) — REF sort.cu:619-672 (one CTA per row there).  Here one warp per
// row, eight rows per CTA: D is a head size (64..256), so a shuffle reduction is enough and a
// decode step (a few hundred rows) still fills the SMs.  Same rounding points: f32 sum of squares,
// T(x * inv_rms * w).
template <typename T>
__global__ void __launch_bounds__(256) rms_norm_strided_4d_kernel(const T *__restrict__ x, const T *__restrict__ w,
                                                                  T *__restrict__ dst, int64_t stride_b, int64_t stride_h,
                                                                  int64_t stride_s, int64_t stride_d, int heads,
                                                                  int seq_len, int head_dim, int64_t rows, float eps) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;  // whole warps leave together
  const int lane = threadIdx.x & 31;
  const int seq = (int)(row % seq_len);
  const int64_t t = row / seq_len;
  const int head = (int)(t % heads);
  const int64_t b = t / heads;
  const T *src = x + b * stride_b + head * stride_h + seq * stride_s;
  float ss = 0.f;
  for (int c = lane; c < head_dim; c += 32) {
    const float v = to_f(src[c * stride_d]);
    ss += v * v;
  }
  const float inv = rsqrtf(warp_sum(ss) / (float)head_dim + eps);
  T *out = dst + row * head_dim;
  for (int c = lane; c < head_dim; c += 32) out[c] = from_f<T>(to_f(src[c * stride_d]) * inv * to_f(w[c]));
}

template <typename T>
static void launch_rms_strided_4d(const void *x, const void *w, void *dst, int64_t sb, int64_t sh, int64_t ss, int64_t sd,
                                  int batch, int heads, int seq_len, int head_dim, float eps, cudaStream_t st) {
  if (batch <= 0 || heads <= 0 || seq_len <= 0 || head_dim <= 0) return;
  const int64_t rows = (int64_t)batch * heads * seq_len;
  rms_norm_strided_4d_kernel<T><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>((const T *)x, (const T *)w, (T *)dst, sb, sh, ss,
                                                                           sd, heads, seq_len, head_dim, rows, eps);
}

}  // namespace mrs

using namespace mrs;

// ---- reference-shaped C ABI ----------------------------------------------------------------
extern "C" void rotary_embedding(void *query, void *key, void *cos_cache, void *sin_cache, int32_t is_neox,
                                 int32_t head_size, int64_t num_tokens, int32_t rot_dim, int32_t num_heads,
                                 int32_t num_kv_heads, int64_t query_stride, int64_t key_stride, uint32_t dtype,
                                 int64_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0) launch_rotary<__half>(query, key, cos_cache, sin_cache, nullptr, is_neox, head_size, num_tokens, rot_dim, num_heads, num_kv_heads, query_stride, key_stride, st);
  else if (dtype == 1) launch_rotary<__nv_bfloat16>(query, key, cos_cache, sin_cache, nullptr, is_neox, head_size, num_tokens, rot_dim, num_heads, num_kv_heads, query_stride, key_stride, st);
  else if (dtype == 2) launch_rotary<float>(query, key, cos_cache, sin_cache, nullptr, is_neox, head_size, num_tokens, rot_dim, num_heads, num_kv_heads, query_stride, key_stride, st);
}

extern "C" void rotary_embedding_positions(void *query, void *key, void *cos_cache, void *sin_cache, void *positions,
                                           int32_t is_neox, int32_t head_size, int64_t num_tokens, int32_t rot_dim,
                                           int32_t seq_len, int32_t num_heads, int32_t num_kv_heads,
                                           int64_t query_stride, int64_t key_stride, uint32_t dtype, int64_t stream) {
  (void)seq_len;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0) launch_rotary<__half>(query, key, cos_cache, sin_cache, positions, is_neox, head_size, num_tokens, rot_dim, num_heads, num_kv_heads, query_stride, key_stride, st);
  else if (dtype == 1) launch_rotary<__nv_bfloat16>(query, key, cos_cache, sin_cache, positions, is_neox, head_size, num_tokens, rot_dim, num_heads, num_kv_heads, query_stride, key_stride, st);
  else if (dtype == 2) launch_rotary<float>(query, key, cos_cache, sin_cache, positions, is_neox, head_size, num_tokens, rot_dim, num_heads, num_kv_heads, query_stride, key_stride, st);
}

#define MRS_GLU(tag, T)                                                                                   \
  extern "C" void fused_glu_##tag(const void *a, const void *b, void *output, uint32_t rows, uint32_t cols, \
                                  uint32_t a_row_stride, uint32_t b_row_stride, int activation,           \
                                  cudaStream_t stream) {                                                  \
    launch_glu<T>(a, b, output, rows, cols, a_row_stride, b_row_stride, activation, stream);              \
  }                                                                                                       \
  extern "C" void fused_split_glu_##tag(const void *input, void *output, uint32_t rows, uint32_t split_size, \
                                        int activation, cudaStream_t stream) {                           \
    launch_glu<T>(input, (const T *)input + split_size, output, rows, split_size, 2 * split_size,        \
                  2 * split_size, activation, stream);                                                    \
  }
MRS_GLU(f16, __half)
MRS_GLU(bf16, __nv_bfloat16)
MRS_GLU(f32, float)

#define MRS_RMS(tag, T)                                                                                       \
  extern "C" void add_rms_norm_##tag(const void *x, const void *residual, const void *weight,                 \
                                     void *residual_dst, void *norm_dst, const int nrows, const int ncols,    \
                                     const float eps, int64_t stream) {                                       \
    launch_rms<T>(x, residual, weight, residual_dst, norm_dst, nrows, ncols, eps, (cudaStream_t)stream);      \
  }                                                                                                           \
  extern "C" void mrs_rms_norm_##tag(const void *x, const void *weight, void *dst, const int nrows,           \
                                     const int ncols, const float eps, int64_t stream) {                      \
    launch_rms<T>(x, nullptr, weight, nullptr, dst, nrows, ncols, eps, (cudaStream_t)stream);                 \
  }
MRS_RMS(f16, __half)
MRS_RMS(bf16, __nv_bfloat16)
MRS_RMS(f32, float)

// decode-chain forms (not in the reference's ABI): the same kernels as links of a programmatic-dependent-launch
// chain — they let the next kernel start its prologue at once and wait for the upstream grid before reading
extern "C" void mrs_add_rms_norm_pdl(const void *x, const void *residual, const void *weight, void *residual_dst, void *norm_dst,
                                     int32_t nrows, int32_t ncols, float eps, int32_t dtype, int32_t pdl, void *stream) {
  if (dtype == MRS_F16) launch_rms<__half>(x, residual, weight, residual_dst, norm_dst, nrows, ncols, eps, (cudaStream_t)stream, pdl);
  else if (dtype == MRS_BF16) launch_rms<__nv_bfloat16>(x, residual, weight, residual_dst, norm_dst, nrows, ncols, eps, (cudaStream_t)stream, pdl);
}
// the norms in front of act-order linears (contract: include/mrs_b200_model.h); pdl 0 is the plain stream-ordered form
extern "C" int32_t mrs_rms_norm_perm_pdl(const void *x, const void *weight, const int32_t *perm, void *norm_dst, int32_t nrows,
                                         int32_t ncols, float eps, int32_t dtype, int32_t pdl, void *stream) {
  if (dtype == MRS_F16) return (int32_t)launch_rms_perm<__half>(x, nullptr, weight, perm, nullptr, norm_dst, nrows, ncols, eps, (cudaStream_t)stream, pdl);
  if (dtype == MRS_BF16) return (int32_t)launch_rms_perm<__nv_bfloat16>(x, nullptr, weight, perm, nullptr, norm_dst, nrows, ncols, eps, (cudaStream_t)stream, pdl);
  return (int32_t)cudaErrorInvalidValue;
}
extern "C" int32_t mrs_add_rms_norm_perm_pdl(const void *x, const void *residual, const void *weight, const int32_t *perm,
                                             void *residual_dst, void *norm_dst, int32_t nrows, int32_t ncols, float eps,
                                             int32_t dtype, int32_t pdl, void *stream) {
  if (residual == nullptr || residual_dst == nullptr) return (int32_t)cudaErrorInvalidValue;
  if (dtype == MRS_F16) return (int32_t)launch_rms_perm<__half>(x, residual, weight, perm, residual_dst, norm_dst, nrows, ncols, eps, (cudaStream_t)stream, pdl);
  if (dtype == MRS_BF16) return (int32_t)launch_rms_perm<__nv_bfloat16>(x, residual, weight, perm, residual_dst, norm_dst, nrows, ncols, eps, (cudaStream_t)stream, pdl);
  return (int32_t)cudaErrorInvalidValue;
}
extern "C" int32_t mrs_gather_cols_pdl(const void *x, const int32_t *perm, void *y, int32_t rows, int32_t cols, int32_t pdl,
                                       void *stream) {
  if (x == nullptr || perm == nullptr || y == nullptr || x == y || rows < 0 || cols < 0) return (int32_t)cudaErrorInvalidValue;
  if (rows == 0 || cols == 0) return 0;
  return (int32_t)launch_pdl(gather_cols_kernel, dim3(rows), dim3(256), 0, (cudaStream_t)stream, pdl, (const uint16_t *)x, perm,
                             (uint16_t *)y, cols, pdl);
}
extern "C" void mrs_split_glu_pdl(const void *input, void *output, uint32_t rows, uint32_t split_size, int32_t activation,
                                  int32_t dtype, int32_t pdl, void *stream) {
  if (dtype == MRS_F16)
    launch_glu<__half>(input, (const __half *)input + split_size, output, rows, split_size, 2 * split_size, 2 * split_size, activation, (cudaStream_t)stream, pdl);
  else if (dtype == MRS_BF16)
    launch_glu<__nv_bfloat16>(input, (const __nv_bfloat16 *)input + split_size, output, rows, split_size, 2 * split_size, 2 * split_size, activation, (cudaStream_t)stream, pdl);
}

#define MRS_RMS4D(tag, T)                                                                                     \
  extern "C" void rms_norm_strided_4d_##tag(const void *x, const void *weight, void *dst, int64_t stride_b,   \
                                            int64_t stride_h, int64_t stride_s, int64_t stride_d, int32_t batch, \
                                            int32_t heads, int32_t seq_len, int32_t head_dim, float eps,      \
                                            int64_t stream) {                                                 \
    launch_rms_strided_4d<T>(x, weight, dst, stride_b, stride_h, stride_s, stride_d, batch, heads, seq_len,   \
                             head_dim, eps, (cudaStream_t)stream);                                            \
  }
MRS_RMS4D(f16, __half)
MRS_RMS4D(bf16, __nv_bfloat16)
MRS_RMS4D(f32, float)
