// mmq_tc.cu — prefill GEMM over ggml quant blocks on the warpgroup tensor cores (wgmma, tc_gemm.cuh).
//
// Replaces the reference's batch>8 path `fast_mmq::plain` (REF mistralrs-quant/src/gguf/
// fast_mmq.rs:762-826 -> launch_mmq_quantize_q8_1_* + launch_mmq_gguf_<q>, int8 `mma.sync`
// m16n8k32 with Q8_1 activations; kernels/mmq_gguf/mmq_gguf.cuh) and the opt-in Marlin repack
// path (gguf/packed_affine.rs:604): Y[M,N] = X[M,K] . W[N,K]^T with W in raw ggml blocks.
//
// This file holds the weight decoders (ggml blocks, GPTQ / AWQ checkpoint tensors, packed-affine payloads) and the
// entry points; the kernel is tc_gemm.cuh's: two threads per weight row read its blocks straight from global / L2,
// expand 32 weights per 64-k step and write them K-major into the 128-byte-swizzled A stage; the TMA brings the
// activation tiles; wgmma m64nNk16 accumulates in registers.
// Numerics: every weight is dequantised with the reference's f32 formula and rounded ONCE to the activations' 16-bit
// format (f16 with f16 activations, bf16 with bf16 ones: the MMA takes one format for both operands); activations are
// used as they are — no activation quantisation — f32 accumulation.  Closer to the exact product than the
// reference's int8-activation MMQ.
#include "affine.cuh"
#include "dequant.cuh"
#include "tc_gemm.cuh"

#include <stdio.h>

namespace mrs {

// ---- register-staged decoding of 32 consecutive weights (two threads share a row's K-step) ----
// load_raw32 only issues loads (so the next K-step's bytes are in flight while the current one
// is expanded); expand32 turns them into 32 floats.
__device__ __forceinline__ void ld_unaligned_words9(const uint8_t *a, uint32_t *w, uint32_t &phase) {
  const uintptr_t u = (uintptr_t)a;
  const uint32_t *a0 = (const uint32_t *)(u & ~(uintptr_t)3);
  phase = (uint32_t)(u & 3) * 8;
#pragma unroll
  for (int i = 0; i < 8; i++) w[i] = a0[i];
  // a 34-byte Q8_0 block that starts on a word boundary ends in the middle of word 8: fetch only
  // its two valid bytes, so the LAST block of a tensor is never read past
  w[8] = (phase != 0) ? a0[8] : (uint32_t)*(const uint16_t *)(a0 + 8);
}
// byte stream starting at the unaligned address: word i of the stream
__device__ __forceinline__ uint32_t stream_word(const uint32_t *w, int i, uint32_t phase) {
  return __funnelshift_r(w[i], (i + 1 < 9) ? w[i + 1] : 0u, phase);
}

template <int TYPE> struct Raw32 { uint32_t w[1]; };
template <> struct Raw32<MRS_Q4_K> { uint4 hdr, q0, q1; };
template <> struct Raw32<MRS_Q8_0> { uint32_t w[9]; uint32_t phase; };
template <> struct Raw32<MRS_Q6_K> { uint32_t ql[9], qh[9]; uint32_t pl, ph; uint32_t sc; uint32_t d; };

template <int TYPE>
__device__ __forceinline__ void load_raw32(const uint8_t *row, int k, Raw32<TYPE> &r) {
  if constexpr (TYPE == MRS_Q4_K) {
    const uint8_t *b = row + (size_t)(k / 256) * 144;
    const int j = ((k % 256) / 32) >> 1;
    r.hdr = *(const uint4 *)b;
    r.q0 = *(const uint4 *)(b + 16 + 32 * j);
    r.q1 = *(const uint4 *)(b + 32 + 32 * j);
  } else if constexpr (TYPE == MRS_Q8_0) {
    ld_unaligned_words9(row + (size_t)(k / 32) * 34, r.w, r.phase);
  } else if constexpr (TYPE == MRS_Q6_K) {
    const uint8_t *b = row + (size_t)(k / 256) * 210;
    const int n = (k % 256) / 128, kk = (k % 128) / 32;
    ld_unaligned_words9(b + 64 * n + 32 * (kk & 1), r.ql, r.pl);
    ld_unaligned_words9(b + 128 + 32 * n, r.qh, r.ph);
    r.sc = *(const uint16_t *)(b + 192 + 8 * n + 2 * kk);
    r.d = *(const uint16_t *)(b + 208);
  }
}

template <int TYPE>
__device__ __forceinline__ void expand32(const Raw32<TYPE> &r, const uint8_t *row, int k, float *out) {
  if constexpr (TYPE == MRS_Q4_K) {
    const int sub = (k % 256) / 32, hi = sub & 1;
    const float d = __half2float(__ushort_as_half((unsigned short)(r.hdr.x & 0xFFFF)));
    const float dmin = __half2float(__ushort_as_half((unsigned short)(r.hdr.x >> 16)));
    // 6-bit scale / min of sub-block `sub` from the 12 scale bytes held in hdr.y/z/w (registers only)
    auto qb = [&](int i) -> int {
      const uint32_t wsel = (i < 4) ? r.hdr.y : ((i < 8) ? r.hdr.z : r.hdr.w);
      return (int)((wsel >> (8 * (i & 3))) & 0xFF);
    };
    int sc, m;
    if (sub < 4) { sc = qb(sub) & 63; m = qb(sub + 4) & 63; }
    else { sc = (qb(sub + 4) & 0xF) | ((qb(sub - 4) >> 6) << 4); m = (qb(sub + 4) >> 4) | ((qb(sub) >> 6) << 4); }
    const float ds = d * (float)sc, om = dmin * (float)m;
    const uint32_t w[8] = {r.q0.x, r.q0.y, r.q0.z, r.q0.w, r.q1.x, r.q1.y, r.q1.z, r.q1.w};
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const uint32_t v = hi ? (w[i] >> 4) : w[i];
#pragma unroll
      for (int b = 0; b < 4; b++) out[4 * i + b] = ds * (float)((v >> (8 * b)) & 0xF) - om;
    }
  } else if constexpr (TYPE == MRS_Q8_0) {
    const uint32_t s0 = stream_word(r.w, 0, r.phase);
    const float d = __half2float(__ushort_as_half((unsigned short)(s0 & 0xFFFF)));
#pragma unroll
    for (int i = 0; i < 8; i++) {
      // qs word i = stream bytes 2+4i .. 5+4i = high half of stream word i, low half of word i+1
      const uint32_t lo = stream_word(r.w, i, r.phase), hi2 = stream_word(r.w, i + 1, r.phase);
      const uint32_t q = __funnelshift_r(lo, hi2, 16);
#pragma unroll
      for (int b = 0; b < 4; b++) out[4 * i + b] = d * (float)(int8_t)((q >> (8 * b)) & 0xFF);
    }
  } else if constexpr (TYPE == MRS_Q6_K) {
    const int kk = (k % 128) / 32, hs = kk >> 1;   // hs: 1 -> high nibbles, qh bits shift by 4
    const float d = __half2float(__ushort_as_half((unsigned short)r.d));
    const float d0 = d * (float)(int8_t)(r.sc & 0xFF), d1 = d * (float)(int8_t)(r.sc >> 8);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const uint32_t l = stream_word(r.ql, i, r.pl), h = stream_word(r.qh, i, r.ph);
#pragma unroll
      for (int b = 0; b < 4; b++) {
        const uint32_t lb = (l >> (8 * b)) & 0xFF, hb = (h >> (8 * b)) & 0xFF;
        const int q = (int)((hs ? (lb >> 4) : (lb & 0xF)) | (((hb >> (2 * kk)) & 3) << 4)) - 32;
        out[4 * i + b] = ((4 * i + b) < 16 ? d0 : d1) * (float)q;
      }
    }
  } else {
    // other ggml types: exact per-element decode (correct, not tuned)
    const int be = (TYPE >= MRS_Q2_K) ? 256 : 32;
    constexpr int bb = (TYPE == MRS_Q4_0) ? 18 : (TYPE == MRS_Q4_1) ? 20 : (TYPE == MRS_Q5_0) ? 22 : (TYPE == MRS_Q5_1) ? 24
                     : (TYPE == MRS_Q2_K) ? 84 : (TYPE == MRS_Q3_K) ? 110 : (TYPE == MRS_Q5_K) ? 176 : 1;
    for (int i = 0; i < 32; i++) {
      const int e = k + i;
      out[i] = dequant_elem(TYPE, row + (size_t)(e / be) * bb, e % be);
    }
  }
}

// "checkpoint" types: weights are not ggml blocks addressed by row_bytes but separate arrays read through dequant32_ckpt
struct TcParams {
  int N, K, out_dtype;
  // GPTQ / AWQ int4 checkpoints (TYPE_GPTQ4 / TYPE_AWQ4): raw HF tensors, no Marlin repack
  const int32_t *qweight;   // GPTQ [K/8, N] (nibbles along K); AWQ [K, N/8] (nibbles along N, order 0,2,4,6,1,3,5,7)
  const __half *scales;     // [K/group, N]
  const int32_t *qzeros;    // AWQ [K/group, N/8]; GPTQ: ignored (symmetric, w = (q-8)*s — REF marlin kU4B8)
  const int32_t *g_idx;     // GPTQ act-order group of each k, or nullptr (k / group)
  int group;
  // packed-affine ggml weights (TYPE_AFF4 / TYPE_AFF8; layout in affine.cuh): w = scale * q - offset, group 16 or 32
  const uint8_t *aff_payload;
  const uint16_t *aff_scales, *aff_offsets;
  int aff_bf16;             // 16-bit format of scales / offsets
};
constexpr int TYPE_GPTQ4 = 100, TYPE_AWQ4 = 101, TYPE_AFF4 = 102, TYPE_AFF8 = 103;

template <int TYPE>
__device__ __forceinline__ void dequant32_ckpt(const TcParams &p, int n, int k0, float *out) {
  if constexpr (TYPE == TYPE_AFF4 || TYPE == TYPE_AFF8) {
    affine::dequant32(p.aff_payload, p.aff_scales, p.aff_offsets, TYPE == TYPE_AFF4 ? 4 : 8, p.group, p.aff_bf16 != 0, p.K, n, k0, out);
  } else if constexpr (TYPE == TYPE_GPTQ4) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint32_t w = (uint32_t)p.qweight[(size_t)(k0 / 8 + i) * p.N + n];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int k = k0 + 8 * i + j;
        const int g = p.g_idx ? p.g_idx[k] : k / p.group;
        out[8 * i + j] = (float)((int)((w >> (4 * j)) & 0xF) - 8) * __half2float(p.scales[(size_t)g * p.N + n]);
      }
    }
  } else {
    const int sh = 4 * ((n & 7) == 0 ? 0 : (n & 7) == 1 ? 4 : (n & 7) == 2 ? 1 : (n & 7) == 3 ? 5 : (n & 7) == 4 ? 2 : (n & 7) == 5 ? 6 : (n & 7) == 6 ? 3 : 7);
#pragma unroll 8
    for (int i = 0; i < 32; i++) {
      const int k = k0 + i, g = k / p.group;
      const int q = (int)(((uint32_t)p.qweight[(size_t)k * (p.N / 8) + n / 8] >> sh) & 0xF);
      const int z = (int)(((uint32_t)p.qzeros[(size_t)g * (p.N / 8) + n / 8] >> sh) & 0xF);
      out[i] = (float)(q - z) * __half2float(p.scales[(size_t)g * p.N + n]);
    }
  }
}

// ---- weight sources of the warpgroup-MMA GEMM (tc_gemm.cuh) --------------------------------------
// ggml blocks addressed by row_bytes: raw words of the next step are loaded while the current one is expanded
template <int TYPE> struct GgmlSrc {
  static constexpr bool kTmaA = false;
  static constexpr int kAhead = 1;
  using Raw = Raw32<TYPE>;
  const uint8_t *w;
  int row_bytes, bf;
  __device__ __forceinline__ void load(Raw &r, int row, int k) const { load_raw32<TYPE>(w + (size_t)row * row_bytes, k, r); }
  __device__ __forceinline__ void expand(const Raw &r, int row, int k, uint32_t *o) const {
    float v[32];
    expand32<TYPE>(r, w + (size_t)row * row_bytes, k, v);
#pragma unroll
    for (int i = 0; i < 16; i++) o[i] = pack_act2(v[2 * i], v[2 * i + 1], bf != 0);
  }
};
// up to three ggml matrices of one type over the same X and K (q|k|v, gate|up), each in its own buffer with its own
// output [M, rows_m].  Grouped (GLU false): global weight row n runs through matrix 0, then 1, then 2; a 128-row tile
// may straddle two matrices, so every row is mapped on its own.  GLU: tile z holds gate rows 64 z .. 64 z + 63 in its
// first 64 rows and the same up rows in its second 64 (warpgroup 0 / 1); only the gate rows' outputs are written.
template <int TYPE, bool GLU> struct GgmlGroupSrc {
  static constexpr bool kTmaA = false;
  static constexpr int kAhead = 1;
  static constexpr int kEpi = GLU ? 2 : 1;
  using Raw = Raw32<TYPE>;
  const uint8_t *w0, *w1, *w2;
  void *y0, *y1, *y2;
  int r0, r1, r2;          // rows (output widths) of the matrices; 0 for an absent one
  int row_bytes, bf;
  __device__ __forceinline__ int mat(int n) const { return GLU ? (n >> 6) & 1 : (n >= r0) + (n >= r0 + r1); }
  __device__ __forceinline__ int local(int n, int m) const {
    return GLU ? (n >> 7) * 64 + (n & 63) : n - (m == 0 ? 0 : m == 1 ? r0 : r0 + r1);
  }
  __device__ __forceinline__ bool live(int n) const {
    const int m = mat(n);
    return local(n, m) < (m == 0 ? r0 : m == 1 ? r1 : r2);
  }
  __device__ __forceinline__ const uint8_t *wrow(int n) const {
    const int m = mat(n);
    return (m == 0 ? w0 : m == 1 ? w1 : w2) + (size_t)local(n, m) * row_bytes;
  }
  __device__ __forceinline__ void *out(int n, int tok) const {
    const int m = mat(n);
    const int width = m == 0 ? r0 : m == 1 ? r1 : r2;
    return (uint16_t *)(m == 0 ? y0 : m == 1 ? y1 : y2) + (size_t)tok * width + local(n, m);
  }
  __device__ __forceinline__ void load(Raw &r, int row, int k) const { load_raw32<TYPE>(wrow(row), k, r); }
  __device__ __forceinline__ void expand(const Raw &r, int row, int k, uint32_t *o) const {
    float v[32];
    expand32<TYPE>(r, wrow(row), k, v);
#pragma unroll
    for (int i = 0; i < 16; i++) o[i] = pack_act2(v[2 * i], v[2 * i + 1], bf != 0);
  }
};
// GPTQ / AWQ checkpoints and packed-affine weights: separate arrays read through dequant32_ckpt
template <int TYPE> struct CkptSrc {
  static constexpr bool kTmaA = false;
  static constexpr int kAhead = 1;
  struct Raw {};
  TcParams p;
  __device__ __forceinline__ void load(Raw &, int, int) const {}
  __device__ __forceinline__ void expand(const Raw &, int row, int k, uint32_t *o) const {
    float v[32];
    dequant32_ckpt<TYPE>(p, row, k, v);
#pragma unroll
    for (int i = 0; i < 16; i++) o[i] = pack_act2(v[2 * i], v[2 * i + 1], p.out_dtype == MRS_BF16);
  }
};

}  // namespace mrs

using namespace mrs;

static int tc_row_bytes(int type, int K) {
  switch (type) {
  case MRS_Q4_0: return K / 32 * 18; case MRS_Q4_1: return K / 32 * 20; case MRS_Q5_0: return K / 32 * 22;
  case MRS_Q5_1: return K / 32 * 24; case MRS_Q8_0: return K / 32 * 34; case MRS_Q2_K: return K / 256 * 84;
  case MRS_Q3_K: return K / 256 * 110; case MRS_Q4_K: return K / 256 * 144; case MRS_Q5_K: return K / 256 * 176;
  case MRS_Q6_K: return K / 256 * 210; default: return 0;
  }
}

// Y[M, N] (dtype) = X[M, K] (dtype, row-major contiguous) . W[N, K]^T (ggml blocks).
// dtype 0 = f16, 1 = bf16.  K must be a multiple of 64 (and of the type's block size).
extern "C" int32_t mrs_mmq_gguf(int32_t ggml_type, const void *w, const void *x, void *y, int32_t M, int32_t N,
                                int32_t K, int32_t dtype, void *stream) {
  if (M <= 0 || N <= 0) return 0;
  const int rb = tc_row_bytes(ggml_type, K);
  if (rb == 0 || K % 64 != 0 || (dtype != 0 && dtype != 1)) return (int32_t)cudaErrorInvalidValue;
  if (ggml_type >= MRS_Q2_K && K % 256 != 0) return (int32_t)cudaErrorInvalidValue;
  if (((uintptr_t)w & 15) || ((uintptr_t)x & 15) || ((uintptr_t)y & 1)) return (int32_t)cudaErrorMisalignedAddress;
  cudaStream_t st = (cudaStream_t)stream;
#define MRS_G(T) return (int32_t)hg_run(GgmlSrc<T>{(const uint8_t *)w, rb, dtype}, x, nullptr, y, M, N, K, dtype, 0, st)
  switch (ggml_type) {
  case MRS_Q4_0: MRS_G(MRS_Q4_0);
  case MRS_Q4_1: MRS_G(MRS_Q4_1);
  case MRS_Q5_0: MRS_G(MRS_Q5_0);
  case MRS_Q5_1: MRS_G(MRS_Q5_1);
  case MRS_Q8_0: MRS_G(MRS_Q8_0);
  case MRS_Q2_K: MRS_G(MRS_Q2_K);
  case MRS_Q3_K: MRS_G(MRS_Q3_K);
  case MRS_Q4_K: MRS_G(MRS_Q4_K);
  case MRS_Q5_K: MRS_G(MRS_Q5_K);
  case MRS_Q6_K: MRS_G(MRS_Q6_K);
  default: return (int32_t)cudaErrorInvalidValue;
  }
#undef MRS_G
}

template <bool GLU>
static cudaError_t mmq_group_run(int type, const GgmlGroupSrc<MRS_Q4_0, GLU> &a, const void *x, int M, int N, int K, int dtype,
                                 int pdl, bool split_k, cudaStream_t st) {
  // one field layout for every type: only the decoder differs
#define MRS_GG(T) return hg_run(GgmlGroupSrc<T, GLU>{a.w0, a.w1, a.w2, a.y0, a.y1, a.y2, a.r0, a.r1, a.r2, a.row_bytes, a.bf}, \
                                x, nullptr, nullptr, M, N, K, dtype, pdl, st, split_k)
  switch (type) {
  case MRS_Q4_0: MRS_GG(MRS_Q4_0);
  case MRS_Q4_1: MRS_GG(MRS_Q4_1);
  case MRS_Q5_0: MRS_GG(MRS_Q5_0);
  case MRS_Q5_1: MRS_GG(MRS_Q5_1);
  case MRS_Q8_0: MRS_GG(MRS_Q8_0);
  case MRS_Q2_K: MRS_GG(MRS_Q2_K);
  case MRS_Q3_K: MRS_GG(MRS_Q3_K);
  case MRS_Q4_K: MRS_GG(MRS_Q4_K);
  case MRS_Q5_K: MRS_GG(MRS_Q5_K);
  case MRS_Q6_K: MRS_GG(MRS_Q6_K);
  default: return cudaErrorInvalidValue;
  }
#undef MRS_GG
}

// The GEMM over n_mats (1..3) ggml matrices of one type that share X [M, K]: Y_m [M, rows[m]] = X . W_m^T, one launch
// (q|k|v, gate|up, or a single matrix as a link of a PDL chain).  glu != 0: n_mats == 2, W_0 = gate and W_1 = up of
// equal rows, and only y[0] = T(silu(T(X . W_0^T))) * T(X . W_1^T) (in T, as fused_glu) is written.  pdl != 0: a link
// of a programmatic-dependent-launch chain (weights stream before the upstream grid completes; x is read and y written
// after).  Same numerics and checks as mrs_mmq_gguf.
extern "C" int32_t mrs_mmq_gguf_grouped(int32_t ggml_type, int32_t n_mats, const void **w, const int32_t *rows,
                                        void **y, const void *x, int32_t M, int32_t K, int32_t dtype, int32_t glu,
                                        int32_t pdl, void *stream) {
  if (n_mats < 1 || n_mats > 3 || w == nullptr || rows == nullptr || y == nullptr) return (int32_t)cudaErrorInvalidValue;
  const bool split_k = !(pdl & 2);
  pdl &= 1;
  if (glu && (n_mats != 2 || rows[0] != rows[1])) return (int32_t)cudaErrorInvalidValue;
  if (M <= 0) return 0;
  const int rb = tc_row_bytes(ggml_type, K);
  if (rb == 0 || K % 64 != 0 || (dtype != 0 && dtype != 1)) return (int32_t)cudaErrorInvalidValue;
  if (ggml_type >= MRS_Q2_K && K % 256 != 0) return (int32_t)cudaErrorInvalidValue;
  if ((uintptr_t)x & 15) return (int32_t)cudaErrorMisalignedAddress;
  int64_t total = 0;
  for (int m = 0; m < n_mats; m++) {
    if (rows[m] <= 0 || w[m] == nullptr || (y[m] == nullptr && !(glu && m == 1))) return (int32_t)cudaErrorInvalidValue;
    if (((uintptr_t)w[m] & 15) || ((uintptr_t)y[m] & 1)) return (int32_t)cudaErrorMisalignedAddress;
    total += rows[m];
  }
  if (total > (int64_t)1 << 30) return (int32_t)cudaErrorInvalidValue;
  const int n = n_mats;
  GgmlGroupSrc<MRS_Q4_0, false> a{(const uint8_t *)w[0], n > 1 ? (const uint8_t *)w[1] : nullptr, n > 2 ? (const uint8_t *)w[2] : nullptr,
                                  y[0], n > 1 ? y[1] : nullptr, n > 2 ? y[2] : nullptr, rows[0], n > 1 ? rows[1] : 0,
                                  n > 2 ? rows[2] : 0, rb, dtype};
  cudaStream_t st = (cudaStream_t)stream;
  if (glu) {
    const GgmlGroupSrc<MRS_Q4_0, true> g{a.w0, a.w1, nullptr, a.y0, a.y1, nullptr, a.r0, a.r1, 0, rb, dtype};
    return (int32_t)mmq_group_run<true>(ggml_type, g, x, M, (rows[0] + 63) / 64 * HG_BM, K, dtype, pdl, split_k, st);
  }
  return (int32_t)mmq_group_run<false>(ggml_type, a, x, M, (int)total, K, dtype, pdl, split_k, st);
}

// GPTQ / AWQ int4 linear on the tensor cores, straight from the checkpoint tensors (no Marlin
// repack): Y[M,N] f16 = X[M,K] f16 . W, W[k,n] = (q-8)*s (GPTQ, symmetric) or (q-z)*s (AWQ).
// Mirrors GptqLayer::forward_raw -> marlin_matmul (REF mistralrs-quant/src/gptq/gptq_cuda.rs:357-398,
// marlin_backend.rs); activations are f16 (`quantized_act_type`), bits == 4 only.
extern "C" int32_t mrs_gptq_gemm(const void *x, const int32_t *qweight, const void *scales, const int32_t *qzeros,
                                 const int32_t *g_idx, void *y, int32_t M, int32_t K, int32_t N, int32_t group_size,
                                 int32_t is_awq, void *stream) {
  if (M <= 0 || N <= 0) return 0;
  if (K % 64 != 0 || N % 8 != 0 || group_size <= 0 || K % group_size != 0) return (int32_t)cudaErrorInvalidValue;
  if (is_awq && qzeros == nullptr) return (int32_t)cudaErrorInvalidValue;
  TcParams p = {};
  p.N = N; p.K = K; p.out_dtype = MRS_F16;
  p.qweight = qweight; p.scales = (const __half *)scales; p.qzeros = qzeros; p.g_idx = g_idx; p.group = group_size;
  cudaStream_t st = (cudaStream_t)stream;
  return (int32_t)(is_awq ? hg_run(CkptSrc<TYPE_AWQ4>{p}, x, nullptr, y, M, N, K, MRS_F16, 0, st)
                          : hg_run(CkptSrc<TYPE_GPTQ4>{p}, x, nullptr, y, M, N, K, MRS_F16, 0, st));
}

// Packed-affine ggml linear (a5): Y[m, n] = X[m, k] . W^T with W held as unsigned 4- / 8-bit payload + per-group 16-bit
// scale and offset, as mrs_gguf_affine_repack_* (affine.cu) wrote them.  Behind the reference's symbols
// `marlin_affine_{u4,u8}_{f16,bf16}` (REF mistralrs-quant/src/gguf/packed_affine.rs:1458-1509 declarations, :697-752 call
// site: n is the PADDED width, the output is [m, padded_n]; `workspace` is the reference kernel's lock array — unused here).
// Same kernel as the checkpoint-layout int4 GEMM: each weight is fma(q, scale, -offset) in f32, rounded once to the
// activations' 16-bit format, f32 accumulation.  0 ok, -1 bad shape, else a cudaError.
static int32_t affine_gemm(const void *x, const void *payload, const void *scales, const void *offsets, void *y, int m, int k, int n, int group,
                           int bits, int dtype, cudaStream_t st) {
  if (m <= 0 || n <= 0) return 0;
  if (k <= 0 || k % 64 != 0 || (group != 16 && group != 32) || n % 8 != 0) return -1;
  if (x == nullptr || payload == nullptr || scales == nullptr || offsets == nullptr || y == nullptr) return -1;
  if (((uintptr_t)x & 15) || ((uintptr_t)payload & 15) || ((uintptr_t)y & 15) || ((uintptr_t)scales & 1) || ((uintptr_t)offsets & 1))
    return (int32_t)cudaErrorMisalignedAddress;
  TcParams p = {};
  p.N = n; p.K = k; p.out_dtype = dtype; p.group = group;
  p.aff_payload = (const uint8_t *)payload; p.aff_scales = (const uint16_t *)scales; p.aff_offsets = (const uint16_t *)offsets;
  p.aff_bf16 = dtype == MRS_BF16;
  return (int32_t)(bits == 4 ? hg_run(CkptSrc<TYPE_AFF4>{p}, x, nullptr, y, m, n, k, dtype, 0, st)
                             : hg_run(CkptSrc<TYPE_AFF8>{p}, x, nullptr, y, m, n, k, dtype, 0, st));
}
#define MRS_AFFINE_ENTRY(NAME, BITS, DT)                                                                                                      \
  extern "C" int32_t NAME(const void *input, const void *weight, void *scales, void *offsets, void *output, int32_t m, int32_t k, int32_t n,   \
                          int32_t group_size, void *workspace, int64_t stream) {                                                              \
    (void)workspace;                                                                                                                          \
    return affine_gemm(input, weight, scales, offsets, output, m, k, n, group_size, BITS, DT, (cudaStream_t)stream);                          \
  }
MRS_AFFINE_ENTRY(marlin_affine_u4_f16, 4, MRS_F16)
MRS_AFFINE_ENTRY(marlin_affine_u4_bf16, 4, MRS_BF16)
MRS_AFFINE_ENTRY(marlin_affine_u8_f16, 8, MRS_F16)
MRS_AFFINE_ENTRY(marlin_affine_u8_bf16, 8, MRS_BF16)
