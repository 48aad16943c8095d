// prefill_attn_tc.cu — causal (var-len) prompt attention on the warpgroup tensor cores (wgmma), head size 128.
//
// Same contract and arithmetic class as prefill_attn.cu (REF mistralrs-core/src/paged_attention/layers/
// paged_attention.rs:1413-1475 -> flash_attn_varlen; SURVEY §8(f) rank 1): S = QK^T and O = PV on 16-bit MMAs with
// f32 accumulation, online softmax in f32 (base-2 exponent, scale folded), P rounded to the activation dtype before
// the second GEMM.  mrs_prefill_attention routes here for head_dim 128 without window / softcap; prefill_attn.cu
// (mma.sync) keeps every other case.
//
// One CTA = 128 query rows of one (sequence, head), 128-token K/V tiles, 256 threads (two warpgroups, so that each
// thread may hold the 64 S, 64 O and 32 P registers of its rows without spilling):
//   thread 0        TMA: Q once (two SWIZZLE_128B boxes of 64 d), K and V tiles through two 2-stage rings; the
//                   tiles of step j + 2 are issued once both warpgroups are done with step j;
//   warpgroups 0, 1 64 query rows each:
//                     S_j  = Q K_j^T   wgmma m64n128k16 x 8, both operands K-major in shared memory
//                     softmax on the S accumulators in registers (a row lives in the four threads of a quad)
//                     O   += P_j V_j   wgmma m64n128k16 x 8 with P as the register A operand (the S accumulator
//                                      layout IS the A fragment layout) and V straight from its row-major
//                                      [token][d] tile as an MN-major SWIZZLE_128B operand (no transpose pass)
//                   then O / l -> global.
//
// PAGED = true is the same kernel over the HND page cache [num_blocks, KVH, page, D] (mrs_prefill_attention_paged):
// each cache is one 2-D tensor map of [num_blocks * KVH * page rows, D], and a 128-token K or V tile arrives as
// 128 / page boxes of [page rows][64 d] per d half, box p at row p * page of the stage, issued by the lanes of warp 0
// (one box each, so that no thread serialises up to 64 block-id reads and TMA issues between its MMAs).  The 128-byte swizzle is a
// function of the shared-memory address over 8-row / 1 KB atoms and page * 128 B is a multiple of 1 KB, so the stage
// holds exactly the bytes one [128 rows][64 d] box would: every MMA descriptor is unchanged.  Pages at or past
// ceil(kv_len / page) are never looked up nor loaded; the V rows at or past kv_len in the last tile (stale cache rows
// of the last page, or whatever the stage held) are zeroed before the PV MMAs, because P = 0 times a NaN is NaN.
// Query i of a sequence sits at key position kv_len - q_len + i (causal mask aligned bottom-right).
#include "tc_common.cuh"

#include <math.h>
#include <stdio.h>

namespace mrs {

constexpr int FT_BM = 128, FT_BN = 128, FT_D = 128;
constexpr int FT_THREADS = 256;
constexpr int FT_TILE_BYTES = FT_BN * FT_D * 2;                       // 32 KB: two boxes [128 rows][64 d]
constexpr int FT_STAGES = 2;
constexpr int FT_SMEM = 1024 + (1 + 2 * FT_STAGES) * FT_TILE_BYTES + 256;   // Q + K ring + V ring + barriers

struct FtParams {
  void *o;
  const int32_t *cu_seqlens;   // [B + 1] or nullptr (single sequence of length T); query rows when paged
  int T, H, KVH;
  int64_t o_stride;            // elements between consecutive tokens of the output
  float scale_log2;            // softmax_scale * log2(e)
  int causal, bf16;
  uint32_t v_lbo, v_sbo;       // MN-major descriptor strides of the V operand, bytes
  const int32_t *cu_seqlens_k; // paged: [B + 1] cumulative key counts
  const int32_t *block_table;  // paged: [B][bt_stride] page ids
  int bt_stride, page;         // paged
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <bool BF, bool PAGED>
__global__ void __launch_bounds__(FT_THREADS, 1)
prefill_attn_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_v, const FtParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t *q_s = smem, *k_s = smem + FT_TILE_BYTES, *v_s = smem + (1 + FT_STAGES) * FT_TILE_BYTES;
  uint64_t *bars = (uint64_t *)(smem + (1 + 2 * FT_STAGES) * FT_TILE_BYTES);
  uint64_t *q_full = bars, *k_full = bars + 1, *k_empty = bars + 3, *v_full = bars + 5, *v_empty = bars + 7;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y;
  const int kvh = h / (p.H / p.KVH);
  int seq0 = 0, len = p.T;
  if (p.cu_seqlens != nullptr) { seq0 = p.cu_seqlens[b]; len = p.cu_seqlens[b + 1] - seq0; }
  int kv_len = len;                                  // keys of the sequence; query i sits at key kv_len - len + i
  if constexpr (PAGED) kv_len = p.cu_seqlens_k[b + 1] - p.cu_seqlens_k[b];
  const int off = kv_len - len;
  const int ntile_q = (len + FT_BM - 1) / FT_BM;
  const int qt = ntile_q - 1 - (int)blockIdx.x;      // heavy (late) query tiles first
  if (qt < 0) return;
  const int q0 = qt * FT_BM;
  const int q_hi = min(len, q0 + FT_BM) - 1;
  const int kv_end = p.causal ? (off + q_hi + 1) : kv_len;
  const int nt = (kv_end + FT_BN - 1) / FT_BN;

  if (tid == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < FT_STAGES; s++) {
      mbar_init(&k_full[s], 1); mbar_init(&v_full[s], 1); mbar_init(&k_empty[s], 2); mbar_init(&v_empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  // K_j and V_j of one step into ring stage j % 2 (TMA; fresh: thread 0, paged: all of warp 0)
  auto load_kv = [&](int j) {
    const int s = j % FT_STAGES;
    uint8_t *ks = k_s + (size_t)s * FT_TILE_BYTES, *vs = v_s + (size_t)s * FT_TILE_BYTES;
    if constexpr (PAGED) {
      // the tile's n pages that hold keys (< ceil(kv_len / page)); 2 n boxes per cache (page x d half), one K and one
      // V box per lane: 2 n <= 32, so each lane reads at most one block id and issues its two loads
      const int per = FT_BN / p.page, pg0 = j * per, n = min(per, (kv_len + p.page - 1) / p.page - pg0);
      const uint32_t box = (uint32_t)p.page * 128u;   // bytes of one [page rows][64 d] box
      if (lane == 0) {
        mbar_arrive_expect_tx(&k_full[s], 2u * (uint32_t)n * box);
        mbar_arrive_expect_tx(&v_full[s], 2u * (uint32_t)n * box);
      }
      __syncwarp();
      if (lane < 2 * n) {
        const int pg = lane >> 1, hf = lane & 1;
        const int row = (p.block_table[(int64_t)b * p.bt_stride + pg0 + pg] * p.KVH + kvh) * p.page;
        const uint32_t dst = (uint32_t)hf * (FT_TILE_BYTES / 2) + (uint32_t)pg * box;
        tma_load_2d(ks + dst, &tmap_k, 64 * hf, row, &k_full[s]);
        tma_load_2d(vs + dst, &tmap_v, 64 * hf, row, &v_full[s]);
      }
    } else {
      const int row = seq0 + j * FT_BN;
      mbar_arrive_expect_tx(&k_full[s], FT_TILE_BYTES);
      tma_load_2d(ks, &tmap_k, kvh * FT_D, row, &k_full[s]);
      tma_load_2d(ks + FT_TILE_BYTES / 2, &tmap_k, kvh * FT_D + 64, row, &k_full[s]);
      mbar_arrive_expect_tx(&v_full[s], FT_TILE_BYTES);
      tma_load_2d(vs, &tmap_v, kvh * FT_D, row, &v_full[s]);
      tma_load_2d(vs + FT_TILE_BYTES / 2, &tmap_v, kvh * FT_D + 64, row, &v_full[s]);
    }
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(q_full, FT_TILE_BYTES);
    tma_load_2d(q_s, &tmap_q, h * FT_D, seq0 + q0, q_full);
    tma_load_2d(q_s + FT_TILE_BYTES / 2, &tmap_q, h * FT_D + 64, seq0 + q0, q_full);
    if constexpr (!PAGED)
      for (int j = 0; j < min(nt, FT_STAGES); j++) load_kv(j);
  }
  if constexpr (PAGED) {
    if (warp == 0)
      for (int j = 0; j < min(nt, FT_STAGES); j++) load_kv(j);
  }

  // ===================== warpgroups: S, softmax, PV, epilogue =====================
  const int g = warp >> 2, t = tid & 127;
  const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2);   // this thread's rows r0 and r0 + 8 of the tile
  const int qg0 = q0 + r0, qg1 = qg0 + 8;
  const int cq = 2 * (lane & 3);                           // column pair of the accumulator fragments
  const uint32_t qs = smem_u32(q_s) + (uint32_t)(64 * g) * 128u;
  float o[64], sacc[64];
#pragma unroll
  for (int i = 0; i < 64; i++) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  mbar_wait(q_full, 0);
  for (int j = 0; j < nt; j++) {
    const int s = j % FT_STAGES, ph = (j / FT_STAGES) & 1;
    const uint32_t ks = smem_u32(k_s) + (uint32_t)s * FT_TILE_BYTES, vs = smem_u32(v_s) + (uint32_t)s * FT_TILE_BYTES;
    mbar_wait(&k_full[s], ph);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const uint32_t off = (uint32_t)(c >> 2) * (FT_TILE_BYTES / 2);
      wgmma_ss<128, BF>(sacc, wgmma_desc_sw128(qs + off) + (uint64_t)(2 * (c & 3)), wgmma_desc_sw128(ks + off) + (uint64_t)(2 * (c & 3)),
                        c ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold<64>(sacc);
    if (t == 0) mbar_arrive(&k_empty[s]);

    const int kv0 = j * FT_BN;
    const int lim0 = min(p.causal ? off + qg0 : kv_len - 1, kv_len - 1) - kv0;
    const int lim1 = min(p.causal ? off + qg1 : kv_len - 1, kv_len - 1) - kv0;
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 16; jj++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int col = 8 * jj + cq + e;
        mx0 = fmaxf(mx0, col <= lim0 ? sacc[4 * jj + e] : -INFINITY);
        mx1 = fmaxf(mx1, col <= lim1 ? sacc[4 * jj + 2 + e] : -INFINITY);
      }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0 * p.scale_log2), mn1 = fmaxf(m1, mx1 * p.scale_log2);   // (scale > 0)
    const float corr0 = (mn0 == m0) ? 1.f : ex2_approx(m0 - mn0), corr1 = (mn1 == m1) ? 1.f : ex2_approx(m1 - mn1);
    const float ms0 = (mn0 == -INFINITY) ? 0.f : mn0, ms1 = (mn1 == -INFINITY) ? 0.f : mn1;
    m0 = mn0; m1 = mn1;
    // p = 2^(s * scale - m), row sums in f32, P rounded to the activation format as the A fragments of the PV MMAs
    uint32_t pa[32];
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int jj = 0; jj < 16; jj++) {
      const int col = 8 * jj + cq;
      const float p00 = (col <= lim0) ? ex2_approx(fmaf(sacc[4 * jj], p.scale_log2, -ms0)) : 0.f;
      const float p01 = (col + 1 <= lim0) ? ex2_approx(fmaf(sacc[4 * jj + 1], p.scale_log2, -ms0)) : 0.f;
      const float p10 = (col <= lim1) ? ex2_approx(fmaf(sacc[4 * jj + 2], p.scale_log2, -ms1)) : 0.f;
      const float p11 = (col + 1 <= lim1) ? ex2_approx(fmaf(sacc[4 * jj + 3], p.scale_log2, -ms1)) : 0.f;
      rs0 += p00 + p01;
      rs1 += p10 + p11;
      // k16 step c = jj / 2: a0 (r0, k lo), a1 (r1, k lo), a2 (r0, k hi), a3 (r1, k hi)
      pa[4 * (jj >> 1) + 2 * (jj & 1)] = pack_act2_t<BF>(p00, p01);
      pa[4 * (jj >> 1) + 2 * (jj & 1) + 1] = pack_act2_t<BF>(p10, p11);
    }
    rs0 += __shfl_xor_sync(0xffffffffu, rs0, 1); rs0 += __shfl_xor_sync(0xffffffffu, rs0, 2);
    rs1 += __shfl_xor_sync(0xffffffffu, rs1, 1); rs1 += __shfl_xor_sync(0xffffffffu, rs1, 2);
    l0 = l0 * corr0 + rs0;
    l1 = l1 * corr1 + rs1;
#pragma unroll
    for (int jj = 0; jj < 16; jj++) {
      o[4 * jj] *= corr0; o[4 * jj + 1] *= corr0; o[4 * jj + 2] *= corr1; o[4 * jj + 3] *= corr1;
    }
    mbar_wait(&v_full[s], ph);
    if constexpr (PAGED) {
      if (kv0 + FT_BN > kv_len) {   // last tile: zero V rows kv_len - kv0 .. 127 of both d halves (CTA-uniform branch)
        const int nz = (kv0 + FT_BN - kv_len) * 8;   // 16-byte chunks per half; a swizzled row stays in its 128 B
        uint8_t *vz = v_s + (size_t)s * FT_TILE_BYTES + (size_t)(kv_len - kv0) * 128;
        for (int i = tid; i < 2 * nz; i += FT_THREADS)
          *(uint4 *)(vz + (i >= nz ? FT_TILE_BYTES / 2 : 0) + (size_t)(i >= nz ? i - nz : i) * 16) = make_uint4(0, 0, 0, 0);
        fence_proxy_async();        // generic-proxy stores -> visible to the wgmma reads
        __syncthreads();
      }
    }
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 8; c++)     // 16 tokens per MMA: two 8-row groups of 1024 B
      wgmma_rs_pv<BF>(o, pa + 4 * c, wgmma_desc_sw128_ex(vs + (uint32_t)c * 2048u, p.v_lbo, p.v_sbo));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold<64>(o);
    if (t == 0) mbar_arrive(&v_empty[s]);
    if constexpr (PAGED) {
      if (warp == 0 && j + FT_STAGES < nt) {
        if (lane == 0) { mbar_wait(&k_empty[s], ph); mbar_wait(&v_empty[s], ph); }
        __syncwarp();
        load_kv(j + FT_STAGES);
      }
    } else if (tid == 0 && j + FT_STAGES < nt) {   // both warpgroups are past step j: its stage takes step j + 2
      mbar_wait(&k_empty[s], ph);
      mbar_wait(&v_empty[s], ph);
      load_kv(j + FT_STAGES);
    }
  }
  // epilogue: O / l -> global, 4-byte pairs
  const float inv0 = (l0 > 0.f) ? 1.f / l0 : 0.f, inv1 = (l1 > 0.f) ? 1.f / l1 : 0.f;
#pragma unroll
  for (int half = 0; half < 2; half++) {
    const int qg = half ? qg1 : qg0;
    if (qg >= len) continue;
    const float inv = half ? inv1 : inv0;
    uint32_t *orow = (uint32_t *)((uint8_t *)p.o + ((int64_t)(seq0 + qg) * p.o_stride + (int64_t)h * FT_D) * 2);
#pragma unroll
    for (int jj = 0; jj < 16; jj++) orow[(8 * jj + cq) >> 1] = pack_act2_t<BF>(o[4 * jj + 2 * half] * inv, o[4 * jj + 2 * half + 1] * inv);
  }
}

}  // namespace mrs

using namespace mrs;

static uint32_t g_ft_lbo = 16384u, g_ft_sbo = 1024u;
static int g_ft_enable = 1;
// dev knobs: MN-major descriptor strides of V (bytes); enable = 0 keeps mrs_prefill_attention on prefill_attn.cu
extern "C" void mrs_prefill_attn_tc_debug(int32_t enable, uint32_t lbo, uint32_t sbo) {
  g_ft_enable = enable;
  if (lbo) g_ft_lbo = lbo;
  if (sbo) g_ft_sbo = sbo;
}

template <bool PAGED>
static int32_t launch_ft(const CUtensorMap &tq, const CUtensorMap &tk, const CUtensorMap &tv, const FtParams &p, dim3 grid,
                         cudaStream_t st) {
  if (p.bf16) {
    cudaFuncSetAttribute(prefill_attn_tc_kernel<true, PAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, FT_SMEM);
    prefill_attn_tc_kernel<true, PAGED><<<grid, FT_THREADS, FT_SMEM, st>>>(tq, tk, tv, p);
  } else {
    cudaFuncSetAttribute(prefill_attn_tc_kernel<false, PAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, FT_SMEM);
    prefill_attn_tc_kernel<false, PAGED><<<grid, FT_THREADS, FT_SMEM, st>>>(tq, tk, tv, p);
  }
  return (int32_t)cudaGetLastError();
}

// 2-D tensor map over [rows, cols] 16-bit elements with a row stride, box [box_rows][64], SWIZZLE_128B
static bool ft_make_map(CUtensorMap *m, const void *base, int64_t rows, int64_t cols, int64_t stride, uint32_t box_rows,
                        uint32_t dtype) {
  PFN_encodeTiled enc = tc_get_encode();
  if (enc == nullptr) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)stride * 2};
  const cuuint32_t box[2] = {64u, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return enc(m, dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(base), dims,
             strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// returns cudaErrorNotSupported when the call does not fit this kernel (the caller falls back to prefill_attn.cu)
extern "C" int32_t mrs_prefill_attention_tc(const void *q, const void *k, const void *v, void *out, const int32_t *cu_seqlens,
                                            int32_t batch, int32_t total_tokens, int32_t max_seqlen, int32_t num_heads,
                                            int32_t num_kv_heads, int32_t head_dim, int64_t q_stride, int64_t kv_stride,
                                            int64_t o_stride, float softmax_scale, int32_t causal, int32_t window_left,
                                            float softcap, uint32_t dtype, void *stream) {
  if (!g_ft_enable || head_dim != 128 || window_left >= 0 || softcap > 0.f || (dtype != 0 && dtype != 1)) return (int32_t)cudaErrorNotSupported;
  if (total_tokens <= 0) return 0;
  if (num_kv_heads <= 0 || num_heads % num_kv_heads || (q_stride | kv_stride | o_stride) % 8) return (int32_t)cudaErrorNotSupported;
  if (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15) return (int32_t)cudaErrorNotSupported;
  if (q_stride < (int64_t)num_heads * 128 || kv_stride < (int64_t)num_kv_heads * 128) return (int32_t)cudaErrorNotSupported;
  CUtensorMap tq, tk, tv;
  if (!ft_make_map(&tq, q, total_tokens, (int64_t)num_heads * 128, q_stride, 128, dtype) ||
      !ft_make_map(&tk, k, total_tokens, (int64_t)num_kv_heads * 128, kv_stride, 128, dtype) ||
      !ft_make_map(&tv, v, total_tokens, (int64_t)num_kv_heads * 128, kv_stride, 128, dtype))
    return (int32_t)cudaErrorNotSupported;
  FtParams p = {};
  p.o = out; p.cu_seqlens = cu_seqlens; p.T = total_tokens; p.H = num_heads; p.KVH = num_kv_heads; p.o_stride = o_stride;
  p.scale_log2 = softmax_scale * 1.4426950408889634f; p.causal = causal; p.bf16 = (dtype == 1);
  p.v_lbo = g_ft_lbo; p.v_sbo = g_ft_sbo;
  const int nb = cu_seqlens ? batch : 1, ml = cu_seqlens ? max_seqlen : total_tokens;
  return launch_ft<false>(tq, tk, tv, p, dim3((ml + FT_BM - 1) / FT_BM, num_heads, nb), (cudaStream_t)stream);
}

// the same kernel over the HND page cache (contract: include/mrs_b200_paged_attn.h, mrs_prefill_attention_paged);
// cudaErrorNotSupported when the call does not fit, including a cache whose row index would not fit the TMA's int32
extern "C" int32_t mrs_prefill_attention_paged_tc(const void *q, const void *key_cache, const void *value_cache, void *out,
                                                  const int32_t *block_table, int32_t block_table_stride,
                                                  const int32_t *cu_seqlens_q, const int32_t *cu_seqlens_k, int32_t batch,
                                                  int32_t total_q, int32_t max_seqlen_q, int32_t max_seqlen_k, int32_t num_blocks,
                                                  int32_t num_heads, int32_t num_kv_heads, int32_t head_dim, int32_t page_size,
                                                  int64_t q_stride, int64_t o_stride, float softmax_scale, int32_t causal,
                                                  int32_t window_left, float softcap, uint32_t dtype, void *stream) {
  (void)max_seqlen_k;
  if (!g_ft_enable || head_dim != 128 || window_left >= 0 || softcap > 0.f || (dtype != 0 && dtype != 1)) return (int32_t)cudaErrorNotSupported;
  if (total_q <= 0 || batch <= 0) return 0;
  if (num_kv_heads <= 0 || num_heads % num_kv_heads || (q_stride | o_stride) % 8) return (int32_t)cudaErrorNotSupported;
  if (page_size != 8 && page_size != 16 && page_size != 32) return (int32_t)cudaErrorNotSupported;
  if (((uintptr_t)q | (uintptr_t)key_cache | (uintptr_t)value_cache | (uintptr_t)out) & 15) return (int32_t)cudaErrorNotSupported;
  if (q_stride < (int64_t)num_heads * 128 || num_blocks <= 0) return (int32_t)cudaErrorNotSupported;
  const int64_t cache_rows = (int64_t)num_blocks * num_kv_heads * page_size;
  if (cache_rows > INT32_MAX) return (int32_t)cudaErrorNotSupported;
  CUtensorMap tq, tk, tv;
  if (!ft_make_map(&tq, q, total_q, (int64_t)num_heads * 128, q_stride, 128, dtype) ||
      !ft_make_map(&tk, key_cache, cache_rows, 128, 128, (uint32_t)page_size, dtype) ||
      !ft_make_map(&tv, value_cache, cache_rows, 128, 128, (uint32_t)page_size, dtype))
    return (int32_t)cudaErrorNotSupported;
  FtParams p = {};
  p.o = out; p.cu_seqlens = cu_seqlens_q; p.cu_seqlens_k = cu_seqlens_k; p.block_table = block_table;
  p.bt_stride = block_table_stride; p.page = page_size;
  p.T = total_q; p.H = num_heads; p.KVH = num_kv_heads; p.o_stride = o_stride;
  p.scale_log2 = softmax_scale * 1.4426950408889634f; p.causal = causal; p.bf16 = (dtype == 1);
  p.v_lbo = g_ft_lbo; p.v_sbo = g_ft_sbo;
  return launch_ft<true>(tq, tk, tv, p, dim3((max_seqlen_q + FT_BM - 1) / FT_BM, num_heads, batch), (cudaStream_t)stream);
}
