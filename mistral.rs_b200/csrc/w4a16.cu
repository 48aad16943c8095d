// w4a16.cu — small-batch W4A16 (GPTQ / AWQ int4) and dense f16/bf16 linear on the warpgroup tensor cores
// (tc_gemm.cuh), "swap-AB": the WEIGHT rows are the wgmma M (two warpgroups x 64) and the tokens its N (32, 64, 128),
// so a decode batch of 32 fills the instruction instead of a quarter of a 128-token tile.
//
// Replaces the reference's Marlin path behind its own symbols
//   marlin_{gptq,awq}_4bit_{f16,bf16}, {gptq,awq}_marlin_repack     REF mistralrs-quant/src/gptq/marlin_ffi.rs:6-81,
//   kernels/marlin/marlin_kernel.cuh (one kernel for every m), marlin_repack.cu:255,473
// and the dense small-batch lm_head of GPTQ checkpoints (REF kernels/gemv/gemv.cu, candle matmul).
//
// HBM-bound at m <= 64 (Mistral-7B g128: 3.6 GB of packed weights per step).  Per thread = (weight row, 32-weight
// half of a 64-k step): one 16-byte load of packed nibbles (contiguous in the repacked layout) + the group's scale
// (and AWQ zero point) -> exact (q - 8) [(q - z)] in the activation format via the magic-number trick -> x scale (one
// rounding, = the reference's dequant) -> the K-major 128B-swizzled A stage.  Dense weights come in through the TMA.
// When the row tiles alone leave SMs idle, K is split over a thread-block cluster and the partials are added in rank
// order through DSMEM (deterministic, no global scratch).
//
// Repacked weight layout ("mrs int4 tiles", same byte count as the checkpoint tensor so the
// reference's result buffer [K/16, N*16/8] i32 fits): [K/64][N][32 B]; the 32 bytes of (k-step, row)
// hold 64 nibbles, word w = k 8w..8w+7 with nibble j < 4 <-> k = 2j and nibble 4+j <-> k = 2j+1 (so
// that `q & 0x000f000f` yields the f16x2 pair (k, k+1)).
#include "tc_gemm.cuh"

#include <stdio.h>

namespace mrs {

enum { WA_SRC_INT4 = 0, WA_SRC_DENSE = 1 };

// Inverses of the reference's scale-column permutations (REF gptq_cuda.rs:530-540 get_scale_perms):
// permuted[j] = original[perm[j]], so original column r of a 64- (32-) wide chunk sits at inv(r).
//   64-wide: perm[8i + j] = i + 8j                          -> inv(r) = 8 (r % 8) + r / 8
//   32-wide: perm[8i + j] = 2i + {0,1,8,9,16,17,24,25}[j]   -> inv(r) = 8 ((r % 8) / 2) + 2 (r / 8) + r % 2
__host__ __device__ __forceinline__ int inv_scale_perm64(int r) { return 8 * (r & 7) + (r >> 3); }
__host__ __device__ __forceinline__ int inv_scale_perm32(int r) { return 8 * ((r & 7) >> 1) + 2 * (r >> 3) + (r & 1); }

// 8 packed nibbles (layout above) -> four 16-bit pairs of (q - zp) * s in the activation format.
// f16: (q & 0xf) | 0x6400 = 1024 + q exactly; the nibble at bits 4..7 gives 1024 + 16 q, and
// fma(x, 1/16, -(64 + zp)) is exact — REF marlin dequant (kU4B8 / kU4) — then one rounding in x s.
// sub_lo = f16x2(1024 + zp), sub_hi = f16x2(-(64 + zp)) are per-(row, group) constants of the caller.
__device__ __forceinline__ void dequant_word_f16(uint32_t q, uint32_t sub_lo, uint32_t sub_hi, uint32_t s2, uint32_t *out) {
  const uint32_t sixteenth = 0x2c002c00u;
#pragma unroll
  for (int i = 0; i < 2; i++) {
    uint32_t lo, hi;
    asm("lop3.b32 %0, %1, 0x000f000f, 0x64006400, 0xea;" : "=r"(lo) : "r"(q));   // (q & mask) | magic
    asm("lop3.b32 %0, %1, 0x00f000f0, 0x64006400, 0xea;" : "=r"(hi) : "r"(q));
    __half2 a = __hsub2(*(const __half2 *)&lo, *(const __half2 *)&sub_lo);
    __half2 b = __hfma2(*(const __half2 *)&hi, *(const __half2 *)&sixteenth, *(const __half2 *)&sub_hi);
    a = __hmul2(a, *(const __half2 *)&s2);
    b = __hmul2(b, *(const __half2 *)&s2);
    out[2 * i] = *(const uint32_t *)&a;
    out[2 * i + 1] = *(const uint32_t *)&b;
    q >>= 8;
  }
}
// bf16: (q & 0xf) | 0x4300 = 128 + q exactly (the 7-bit mantissa holds the nibble); the subtraction of 128 + zp is
// exact and the product with the bf16 scale rounds once — the same value as (float)(q - zp) * s rounded to bf16
__device__ __forceinline__ void dequant_word_bf16_m(uint32_t q, uint32_t sub2, uint32_t s2, uint32_t *out) {
#pragma unroll
  for (int j = 0; j < 4; j++) {
    uint32_t v;
    asm("lop3.b32 %0, %1, 0x000f000f, 0x43004300, 0xea;" : "=r"(v) : "r"(q));
    __nv_bfloat162 a = __hsub2(*(const __nv_bfloat162 *)&v, *(const __nv_bfloat162 *)&sub2);
    a = __hmul2(a, *(const __nv_bfloat162 *)&s2);
    out[j] = *(const uint32_t *)&a;
    q >>= 4;
  }
}

// ---- weight sources of the warpgroup-MMA GEMM (tc_gemm.cuh) ----------------------------------------
struct Int4TileSrc {
  static constexpr bool kTmaA = false;
  // HBM-bound at decode batch: 16 B per thread and step is 4 KB per CTA; four steps ahead keep 16 KB of weights in flight
  static constexpr int kAhead = 4;
  struct Raw { uint4 q; uint32_t s, zp; };
  const uint8_t *wq;       // repacked int4 [K/64][N][32 B]
  const uint16_t *scales;  // [K/group, N] in the activation dtype (columns possibly Marlin-permuted)
  const int32_t *qzeros;   // AWQ: raw [K/group, N/8] (nibbles in AWQ order) or nullptr (zero point 8)
  int N, group, scale_perm, bf;
  __device__ __forceinline__ void load(Raw &r, int n, int k) const {
    r.q = *(const uint4 *)(wq + ((size_t)(k >> 6) * N + n) * 32 + 16 * ((k >> 5) & 1));
    const int g = k / group;
    int scol = n;
    if (scale_perm == 1) scol = (n & ~63) + inv_scale_perm64(n & 63);
    else if (scale_perm == 2) scol = (n & ~31) + inv_scale_perm32(n & 31);
    r.s = scales[(size_t)g * N + scol];
    r.zp = 8u;
    if (qzeros) {
      const int c7 = n & 7;
      const int zsh = 4 * ((c7 & 1) ? 4 + (c7 >> 1) : (c7 >> 1));   // nibble of column n in AWQ order {0,2,4,6,1,3,5,7}
      r.zp = ((uint32_t)qzeros[(size_t)g * (N >> 3) + (n >> 3)] >> zsh) & 0xFu;
    }
  }
  __device__ __forceinline__ void expand(const Raw &r, int, int, uint32_t *o) const {
    const uint32_t w[4] = {r.q.x, r.q.y, r.q.z, r.q.w};
    const uint32_t s2 = r.s * 0x00010001u;
    if (bf) {
      const uint32_t sub2 = 0x43004300u + r.zp * 0x00010001u;                                  // bf16x2(128 + zp)
#pragma unroll
      for (int c4 = 0; c4 < 4; c4++) dequant_word_bf16_m(w[c4], sub2, s2, o + 4 * c4);
    } else {
      const uint32_t sub_lo = 0x64006400u + r.zp * 0x00010001u;                                // f16x2(1024 + zp)
      const uint32_t sub_hi = (0xD400u + (r.zp << 4)) * 0x00010001u;                           // f16x2(-(64 + zp)): ulp 1/16 in [64, 128)
#pragma unroll
      for (int c4 = 0; c4 < 4; c4++) dequant_word_f16(w[c4], sub_lo, sub_hi, s2, o + 4 * c4);
    }
  }
};
// gate||up int4 tiles (N = 2I weight rows: gate 0 .. I-1, up I .. 2I-1) with the GLU epilogue of tc_gemm.cuh: tile z
// holds gate rows 64 z .. 64 z + 63 in its first 64 rows (warpgroup 0) and the same up rows in its second 64
// (warpgroup 1); y[M, I] = T(silu(T(gate))) * T(up) is written, the [M, 2I] product never is.
struct Int4GluSrc : Int4TileSrc {
  static constexpr int kEpi = 2;
  void *y;
  int I;
  __device__ __forceinline__ int local(int n) const { return (n >> 7) * 64 + (n & 63); }
  __device__ __forceinline__ bool live(int n) const { return local(n) < I; }
  __device__ __forceinline__ void *out(int n, int tok) const { return (uint16_t *)y + (size_t)tok * I + local(n); }
  __device__ __forceinline__ void load(Raw &r, int n, int k) const { Int4TileSrc::load(r, local(n) + ((n >> 6) & 1) * I, k); }
};
// dense 16-bit weights: A tiles straight from the TMA
struct DenseSrc {
  static constexpr bool kTmaA = true;
  static constexpr int kAhead = 1;
  struct Raw {};
  __device__ __forceinline__ void load(Raw &, int, int) const {}
  __device__ __forceinline__ void expand(const Raw &, int, int, uint32_t *) const {}
};

// ---------------------------------------------------------------- repack kernels
// GPTQ checkpoint [K/8, N] i32 (nibble j of word (k8, n) = k 8*k8 + j) -> mrs int4 tiles; `perm`
// (argsort of g_idx, REF gptq_cuda.rs:573-583) gathers source rows exactly like
// gptq_marlin_repack does: packed row k' takes checkpoint row perm[k'].
__global__ void repack_gptq_kernel(const uint32_t *__restrict__ qw, const int32_t *__restrict__ perm, uint32_t *__restrict__ out,
                                   int K, int N) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;   // one output word: (ks, n, w)
  const int64_t total = (int64_t)(K / 64) * N * 8;
  if (idx >= total) return;
  const int w = (int)(idx & 7);
  const int n = (int)((idx >> 3) % N);
  const int ks = (int)((idx >> 3) / N);
  uint32_t o = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int kdst = ks * 64 + w * 8 + j;
    const int ksrc = perm ? perm[kdst] : kdst;
    const uint32_t nib = (qw[(size_t)(ksrc >> 3) * N + n] >> (4 * (ksrc & 7))) & 0xFu;
    const int pos = (j & 1) ? 4 + (j >> 1) : (j >> 1);
    o |= nib << (4 * pos);
  }
  out[idx] = o;
}
// AWQ checkpoint [K, N/8] i32 (nibble i of word (k, c) = column 8c + {0,2,4,6,1,3,5,7}[i]) -> mrs int4 tiles
__global__ void repack_awq_kernel(const uint32_t *__restrict__ qw, uint32_t *__restrict__ out, int K, int N) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)(K / 64) * N * 8;
  if (idx >= total) return;
  const int w = (int)(idx & 7);
  const int n = (int)((idx >> 3) % N);
  const int ks = (int)((idx >> 3) / N);
  const int c7 = n & 7;
  const int ipos = (c7 & 1) ? 4 + (c7 >> 1) : (c7 >> 1);   // inverse of {0,2,4,6,1,3,5,7}
  uint32_t o = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int k = ks * 64 + w * 8 + j;
    const uint32_t nib = (qw[(size_t)k * (N >> 3) + (n >> 3)] >> (4 * ipos)) & 0xFu;
    const int pos = (j & 1) ? 4 + (j >> 1) : (j >> 1);
    o |= nib << (4 * pos);
  }
  out[idx] = o;
}

// ---------------------------------------------------------------- host
// flags: bit 0 a link of a PDL chain, bit 1 never split K, bit 2 (int4 only) the GLU epilogue over gate||up, N = 2I
static cudaError_t run_wa(int src, const void *x, const void *w, const void *scales, const int32_t *qzeros, void *y, int M,
                          int K, int N, int group, int dtype, int scale_perm, cudaStream_t st, int flags = 0) {
  const bool glu = flags & 4, split_k = !(flags & 2);
  const int pdl = flags & 1;
  if ((flags & ~7) || (glu && (src != WA_SRC_INT4 || N % 16 != 0))) return cudaErrorInvalidValue;
  if (M <= 0 || N <= 0) return cudaSuccess;
  if (K % HG_BK != 0 || (dtype != MRS_F16 && dtype != MRS_BF16)) return cudaErrorInvalidValue;
  if (group <= 0) group = K;
  if (src == WA_SRC_INT4 && (group % 32 != 0 || K % group != 0 || N % 8 != 0)) return cudaErrorInvalidValue;
  if (src == WA_SRC_INT4 && qzeros != nullptr && N % 32 != 0) return cudaErrorInvalidValue;
  if (((uintptr_t)x & 15) || ((uintptr_t)w & 15)) return cudaErrorMisalignedAddress;
  if (src == WA_SRC_DENSE) return hg_run(DenseSrc{}, x, w, y, M, N, K, dtype, pdl, st, split_k);
  const Int4TileSrc s = {(const uint8_t *)w, (const uint16_t *)scales, qzeros, N, group, scale_perm, dtype == MRS_BF16};
  if (glu) {
    const int I = N / 2;
    return hg_run(Int4GluSrc{s, y, I}, x, nullptr, nullptr, M, (I + 63) / 64 * HG_BM, K, dtype, pdl, st, split_k);
  }
  return hg_run(s, x, nullptr, y, M, N, K, dtype, pdl, st, split_k);
}

}  // namespace mrs

using namespace mrs;

// ---- native entries ---------------------------------------------------------------------
// Y[M,N] = X[M,K] . W^T, W = repacked int4 (mrs tiles, see gptq_marlin_repack below); scales
// [K/group, N] in dtype (0 f16 / 1 bf16), group <= 0: one group; qzeros: AWQ raw zero points or NULL
// (symmetric, zero point 8); scale_perm: 0 plain, 1/2 Marlin-permuted scale columns.
extern "C" int32_t mrs_w4a16_gemm(const void *x, const void *w_tiles, const void *scales, const int32_t *qzeros, void *y,
                                  int32_t M, int32_t K, int32_t N, int32_t group, int32_t dtype, int32_t scale_perm,
                                  void *stream) {
  return (int32_t)run_wa(WA_SRC_INT4, x, w_tiles, scales, qzeros, y, M, K, N, group, dtype, scale_perm, (cudaStream_t)stream);
}
// Y[M,N] = X[M,K] . W[N,K]^T with dense 16-bit W (the lm_head of GPTQ/AWQ checkpoints at decode batch)
extern "C" int32_t mrs_dense_linear(const void *x, const void *w, void *y, int32_t M, int32_t K, int32_t N, int32_t dtype,
                                    void *stream) {
  return (int32_t)run_wa(WA_SRC_DENSE, x, w, nullptr, nullptr, y, M, K, N, 0, dtype, 0, (cudaStream_t)stream);
}
// the same two as links of a programmatic-dependent-launch chain (decode layer stack): the weight stream starts while
// the upstream kernel is still running; x is read, and y written, only after it has completed.  `pdl` bit 0: that
// link; bit 1: never split K, so a row's result does not depend on M (prompt steps); bit 2 (int4 only): w_tiles is
// gate||up of N = 2I rows and y [M, I] = T(silu(T(X gate^T))) * T(X up^T), as fused_split_glu after the plain GEMM
extern "C" int32_t mrs_w4a16_gemm_pdl(const void *x, const void *w_tiles, const void *scales, const int32_t *qzeros, void *y,
                                      int32_t M, int32_t K, int32_t N, int32_t group, int32_t dtype, int32_t scale_perm,
                                      int32_t pdl, void *stream) {
  return (int32_t)run_wa(WA_SRC_INT4, x, w_tiles, scales, qzeros, y, M, K, N, group, dtype, scale_perm, (cudaStream_t)stream, pdl);
}
extern "C" int32_t mrs_dense_linear_pdl(const void *x, const void *w, void *y, int32_t M, int32_t K, int32_t N, int32_t dtype,
                                        int32_t pdl, void *stream) {
  return (int32_t)run_wa(WA_SRC_DENSE, x, w, nullptr, nullptr, y, M, K, N, 0, dtype, 0, (cudaStream_t)stream, pdl);
}

// ---- the reference's Marlin symbols (REF mistralrs-quant/src/gptq/marlin_ffi.rs:6-81) ----------
// `weight` of the matmuls is what our own *_marlin_repack wrote (the Rust side treats it as opaque);
// `scales` arrive column-permuted by marlin_permute_scales (REF gptq_cuda.rs:542-565): the 64-wide
// permutation when group < K/8 (the reference passes in_dim / pack_factor as size_k), else the
// 32-wide one; `workspace` (Marlin's lock array) is not needed.
static int marlin_common(const void *inputs, const int32_t *weight, const void *scales, const void *zeros, void *out, int m,
                         int k, int n, int groupsize, int dtype, int is_awq, int64_t stream) {
  cudaError_t status = cudaGetLastError();
  if (status != cudaSuccess) return (int)status;
  const int group = groupsize <= 0 ? k : groupsize;
  const int perm_kind = (groupsize > 0 && groupsize < k / 8) ? 1 : 2;
  const cudaError_t e = run_wa(WA_SRC_INT4, inputs, weight, scales, is_awq ? (const int32_t *)zeros : nullptr, out, m, k, n, group,
                               dtype, perm_kind, (cudaStream_t)stream);
  return e == cudaSuccess ? (int)cudaGetLastError() : (int)e;
}
extern "C" int marlin_gptq_4bit_f16(const void *inputs, const int32_t *weight, const void *scales, const void *zeros,
                                    const void *out, int m, int k, int n, const void *workspace, int groupsize, int64_t stream) {
  (void)workspace;
  return marlin_common(inputs, weight, scales, zeros, (void *)out, m, k, n, groupsize, MRS_F16, 0, stream);
}
extern "C" int marlin_gptq_4bit_bf16(const void *inputs, const int32_t *weight, const void *scales, const void *zeros,
                                     const void *out, int m, int k, int n, const void *workspace, int groupsize, int64_t stream) {
  (void)workspace;
  return marlin_common(inputs, weight, scales, zeros, (void *)out, m, k, n, groupsize, MRS_BF16, 0, stream);
}
extern "C" int marlin_awq_4bit_f16(const void *inputs, const int32_t *weight, const void *scales, const void *zeros,
                                   const void *out, int m, int k, int n, const void *workspace, int groupsize, int64_t stream) {
  (void)workspace;
  return marlin_common(inputs, weight, scales, zeros, (void *)out, m, k, n, groupsize, MRS_F16, 1, stream);
}
extern "C" int marlin_awq_4bit_bf16(const void *inputs, const int32_t *weight, const void *scales, const void *zeros,
                                    const void *out, int m, int k, int n, const void *workspace, int groupsize, int64_t stream) {
  (void)workspace;
  return marlin_common(inputs, weight, scales, zeros, (void *)out, m, k, n, groupsize, MRS_BF16, 1, stream);
}

// weight [k/8, n] i32, perm [k] i32 (argsort of g_idx; the reference always passes one), result: k*n/2 bytes
extern "C" void gptq_marlin_repack(const void *weight, const void *perm, const void *result, int k, int n, int bits,
                                   int64_t stream) {
  if (bits != 4 || k % 64 != 0 || n % 8 != 0) {
    fprintf(stderr, "mrs_b200: gptq_marlin_repack supports 4-bit weights with k %% 64 == 0 (got bits %d, k %d, n %d)\n", bits, k, n);
    return;
  }
  const int64_t total = (int64_t)(k / 64) * n * 8;
  repack_gptq_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint32_t *)weight, (const int32_t *)perm,
                                                                                    (uint32_t *)result, k, n);
}
// in [k, n] i32 with n = out_dim / 8 (REF marlin_repack.cu:473-483), perm unused
extern "C" void awq_marlin_repack(const void *in, const void *perm, const void *out, int k, int n, int bits, int64_t stream) {
  (void)perm;
  const int size_n = n * 8;
  if (bits != 4 || k % 64 != 0) {
    fprintf(stderr, "mrs_b200: awq_marlin_repack supports 4-bit weights with k %% 64 == 0 (got bits %d, k %d)\n", bits, k);
    return;
  }
  const int64_t total = (int64_t)(k / 64) * size_n * 8;
  repack_awq_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const uint32_t *)in, (uint32_t *)out, k, size_n);
}
