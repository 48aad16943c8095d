// tc_gemm.cuh — the warpgroup-MMA GEMM behind every 16-bit tensor-core linear of the library (mmq_tc.cu: ggml
// blocks, GPTQ / AWQ checkpoints, packed-affine weights; w4a16.cu: repacked int4 tiles, dense 16-bit weights).
//
// Y[M, N] = X[M, K] . W[N, K]^T, swap-AB: the WEIGHT rows are the wgmma M dimension, the tokens its N (32, 64, 128
// or 256), so a decode batch of 32 tokens still fills the instruction.  Per CTA: one 128-row weight tile x one
// NT-token tile x one K split, two warpgroups plus, for token tiles up to 128, a TMA producer warp:
//   each warpgroup owns 64 weight rows: thread = (row, 32-k half of the 64-k step); it dequantises its 32 weights
//   (the source policy `Src`, f32 formula of the reference, ONE rounding to the activation format) into the
//   128-byte-swizzled K-major A stage, then the warpgroup issues 4 x wgmma m64nNTk16 against the activation stage;
//   one group stays in flight while the next step is dequantised.  Accumulators in registers; the same threads are
//   the epilogue.
//   the TMA brings activation tiles X[NT x 64] (and, for dense weights, W[128 x 64]) into a 4-deep ring, mbarrier
//   complete_tx; a slot is refilled once both warpgroups' MMAs on it have retired.  The producer is warp 8, which
//   waits for the upstream grid (PDL) and refills the ring off the compute warps' path; a 256-token tile needs 128
//   accumulators per thread, which nine warps cannot hold (an SM sub-partition then carries three warps), so there
//   thread 0 of warpgroup 0 drives the TMA between its MMA steps instead.
// Split-K (small token tiles with few row tiles): the K splits of one tile form a thread-block cluster along y;
// partial accumulators go to the leader's shared memory through DSMEM and are added in rank order (deterministic).
// f32 accumulation in k order, 16 k per instruction: results do not depend on NT, the split of M or the source path.
#pragma once
#include "tc_common.cuh"

namespace mrs {

constexpr int HG_BM = 128;                 // weight rows per CTA (two warpgroups x 64)
constexpr int HG_BK = 64;                  // k per stage: one 128-byte swizzle row of 16-bit values
constexpr int HG_STAGES = 4;
constexpr int HG_THREADS_PW = 256 + 32;   // with the producer warp (NT <= 128)
constexpr bool hg_producer_warp(int nt) { return nt <= 128; }
constexpr int HG_A_BYTES = HG_BM * HG_BK * 2;   // 16 KB

struct HgShape {
  void *y;                 // [M, N] in the activation format
  int M, N, K;
  int ksteps_per_split;    // 64-k steps per split CTA
  int pdl;                 // link of a programmatic-dependent-launch chain: x comes from the upstream grid
};

__host__ __device__ constexpr size_t hg_smem_bytes(int nt, int ksplit) {
  return 1024 + (size_t)HG_STAGES * (HG_A_BYTES + nt * 128) + 256 + (size_t)(ksplit - 1) * nt * HG_BM * 4;
}

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t map_to_rank(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local_smem_addr), "r"(rank));
  return remote;
}
__device__ __forceinline__ void st_cluster_f32_at(uint32_t remote_addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote_addr), "f"(v) : "memory");
}
// arrive on another CTA's mbarrier; release at cluster scope orders this thread's earlier remote stores before it
__device__ __forceinline__ void mbar_arrive_remote(uint32_t remote_bar_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote_bar_addr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred P1;\n\tWAITC_LOOP:\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra.uni WAITC_DONE;\n\tbra.uni WAITC_LOOP;\n\tWAITC_DONE:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

__device__ __forceinline__ uint32_t pack_act2(float lo, float hi, bool bf) {
  if (bf) { const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi); return *(const uint32_t *)&h; }
  const __half2 h = __floats2half2_rn(lo, hi);
  return *(const uint32_t *)&h;
}

// Epilogue of a source: 0 (default) writes y[M, N]; a source with `static constexpr int kEpi` 1 owns its row map:
// `live(row)` says whether weight row `row` exists and `out(row, tok)` is where its output goes (several matrices
// with their own outputs in one launch); kEpi 2 (GLU) additionally pairs the two warpgroups: warpgroup 1's rows are
// the up rows of warpgroup 0's gate rows, and only warpgroup 0 writes, act(T(gate)) * T(up) in T.
template <class S> __host__ __device__ constexpr auto hg_epi_kind(int) -> decltype(S::kEpi, int()) { return S::kEpi; }
template <class S> __host__ __device__ constexpr int hg_epi_kind(long) { return 0; }
template <class Src> __device__ __forceinline__ bool hg_row_live(const Src &src, int row, int N) {
  if constexpr (hg_epi_kind<Src>(0) != 0) return src.live(row);
  else return row < N;
}

// Src: struct with `static constexpr bool kTmaA` (A tiles come from the TMA map `tmap_w`, no dequantisation),
// `static constexpr int kAhead` (how many 64-k steps of raw weights a thread keeps in flight in registers), a
// per-thread `Raw` state, `load(Raw &, row, k)` (issues the loads of weights k .. k+31 of `row`) and
// `expand(const Raw &, row, k, uint32_t o[16])` (16 packed pairs of the activation format, k order).
template <class Src, int NT, bool BF>
__global__ void __launch_bounds__(hg_producer_warp(NT) ? HG_THREADS_PW : 256, 1)
hg_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w, const Src src, const HgShape p) {
  constexpr int X_BYTES = NT * 128;
  constexpr int NACC = NT / 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t *smem = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t *a_ring = smem, *x_ring = smem + HG_STAGES * HG_A_BYTES;
  uint64_t *bars = (uint64_t *)(x_ring + HG_STAGES * X_BYTES);
  uint64_t *x_full = bars, *x_empty = bars + HG_STAGES, *red_bar = bars + 2 * HG_STAGES;
  float *red = (float *)((uint8_t *)bars + 256);      // split-K partials [ksplit - 1][NT][128] (leader only)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.z * HG_BM, m0 = blockIdx.x * NT;
  const int ksplit = gridDim.y;
  const uint32_t rank = (ksplit > 1) ? cluster_ctarank() : 0u;
  const int nk_total = p.K / HG_BK;
  const int kb0 = (int)rank * p.ksteps_per_split;
  const int nk = max(0, min(p.ksteps_per_split, nk_total - kb0));

  if (p.pdl && tid == 0) pdl_launch_dependents();
  if (tid == 0) {
    for (int s = 0; s < HG_STAGES; s++) { mbar_init(&x_full[s], 1); mbar_init(&x_empty[s], 2); }
    mbar_init(red_bar, ksplit > 1 ? (uint32_t)(ksplit - 1) * 256u : 1u);
    fence_mbar_init();
  }
  __syncthreads();
  if (ksplit > 1) cluster_arrive_release();   // start-up cluster barrier (every barrier exists); waited on before DSMEM traffic

  // the TMA loads of step i into ring stage i % 4 (issued by one thread: the producer warp's lane 0, or thread 0)
  auto load_step = [&](int i) {
    const int s = i % HG_STAGES;
    mbar_arrive_expect_tx(&x_full[s], X_BYTES + (Src::kTmaA ? HG_A_BYTES : 0));
    tma_load_2d(x_ring + (size_t)s * X_BYTES, &tmap_x, (kb0 + i) * HG_BK, m0, &x_full[s]);
    if constexpr (Src::kTmaA) tma_load_2d(a_ring + (size_t)s * HG_A_BYTES, &tmap_w, (kb0 + i) * HG_BK, n0, &x_full[s]);
  };
  constexpr bool PW = hg_producer_warp(NT);
  if (PW && warp == 8) {
    // ===================== TMA producer warp =====================
    if (lane == 0) {
      if (p.pdl) pdl_wait();
      for (int i = 0; i < nk; i++) {
        if (i >= HG_STAGES) mbar_wait(&x_empty[i % HG_STAGES], ((i / HG_STAGES) & 1) ^ 1);
        load_step(i);
      }
    }
    if (ksplit > 1) cluster_wait_acquire();
    return;
  }
  if (!PW && tid == 0) {
    if (p.pdl) pdl_wait();   // the activations are the upstream grid's output (the other threads start on the weights)
    for (int i = 0; i < min(nk, HG_STAGES); i++) load_step(i);
  }

  // ===================== warpgroups 0, 1: dequantise, MMA, epilogue =====================
  const int g = warp >> 2, t = tid & 127;
  const int r = 64 * g + (t >> 1), hf = t & 1;   // weight row in the tile, which 32-k half of the step
  const int row = n0 + r;
  const bool live = hg_row_live(src, row, p.N);
  float acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; i++) acc[i] = 0.f;
  constexpr int AH = Src::kAhead;
  typename Src::Raw raw[AH];   // raw[d]: the weights of step i + d (register ring, shifted once per step)
  if constexpr (!Src::kTmaA) {
#pragma unroll
    for (int d = 0; d < AH; d++)
      if (live && d < nk) src.load(raw[d], row, (kb0 + d) * HG_BK + 32 * hf);
  }
  const uint32_t a_base = smem_u32(a_ring) + (uint32_t)(64 * g) * 128u, x_base = smem_u32(x_ring);
  for (int i = 0; i < nk; i++) {
    const int s = i % HG_STAGES, ph = (i / HG_STAGES) & 1;
    if constexpr (!Src::kTmaA) {
      const int k = (kb0 + i) * HG_BK + 32 * hf;
      uint32_t o[16];
      if (live) {
        const typename Src::Raw cur = raw[0];
#pragma unroll
        for (int d = 0; d + 1 < AH; d++) raw[d] = raw[d + 1];
        if (i + AH < nk) src.load(raw[AH - 1], row, k + AH * HG_BK);   // later steps' bytes in flight while this one is expanded
        src.expand(cur, row, k, o);
      } else {
#pragma unroll
        for (int j = 0; j < 16; j++) o[j] = 0u;
      }
      // (the MMAs that last read this stage belong to step i - 4, retired by the wait of step i - 1)
      const uint32_t dst = smem_u32(a_ring) + (uint32_t)s * HG_A_BYTES + (uint32_t)(r >> 3) * 1024u + (uint32_t)(r & 7) * 128u;
#pragma unroll
      for (int cc = 0; cc < 4; cc++) {   // 16-byte chunk c of the row lands at chunk c ^ (r % 8)
        const int c = 4 * hf + cc;
        sts128(dst + (uint32_t)((c ^ (r & 7)) << 4), make_uint4(o[4 * cc], o[4 * cc + 1], o[4 * cc + 2], o[4 * cc + 3]));
      }
      fence_proxy_async();               // generic-proxy writes -> visible to the tensor core
      wg_bar(1 + g);
    }
    mbar_wait(&x_full[s], ph);
    wgmma_fence();
    const uint64_t ad = wgmma_desc_sw128(a_base + (uint32_t)s * HG_A_BYTES), xd = wgmma_desc_sw128(x_base + (uint32_t)s * X_BYTES);
#pragma unroll
    for (int k16 = 0; k16 < HG_BK / 16; k16++) wgmma_ss<NT, BF>(acc, ad + (uint64_t)(2 * k16), xd + (uint64_t)(2 * k16), 1u);
    wgmma_commit();
    wgmma_wait<1>();
    if (i > 0) {
      const int sp = (i - 1) % HG_STAGES;
      if (t == 0) mbar_arrive(&x_empty[sp]);
      if (!PW && tid == 0 && i - 1 + HG_STAGES < nk) {   // both warpgroups' MMAs of step i - 1 have retired: refill its stage
        mbar_wait(&x_empty[sp], ((i - 1) / HG_STAGES) & 1);
        load_step(i - 1 + HG_STAGES);
      }
    }
  }
  wgmma_wait<0>();
  wgmma_hold<NACC>(acc);

  // ===================== epilogue =====================
  // acc[4 j + e]: weight row 16 w + lane / 4 (+ 8 for e >= 2) of the warpgroup's 64, token 8 j + 2 (lane % 4) (+ 1 for odd e)
  const int wr = 64 * g + 16 * (warp & 3) + (lane >> 2), tc = 2 * (lane & 3);
  if (ksplit > 1) {
    cluster_wait_acquire();
    if (rank != 0) {
      const uint32_t rbase = map_to_rank(smem_u32(red + (size_t)(rank - 1) * NT * HG_BM), 0u);
#pragma unroll
      for (int j = 0; j < NT / 8; j++)
#pragma unroll
        for (int e = 0; e < 4; e++)
          st_cluster_f32_at(rbase + (uint32_t)(((8 * j + tc + (e & 1)) * HG_BM + wr + 8 * (e >> 1)) * 4), acc[4 * j + e]);
      mbar_arrive_remote(map_to_rank(smem_u32(red_bar), 0u));
      return;
    }
    mbar_wait_cluster(red_bar, 0);
    for (int sp = 1; sp < ksplit; sp++) {
      const float *rp = red + (size_t)(sp - 1) * NT * HG_BM;
#pragma unroll
      for (int j = 0; j < NT / 8; j++)
#pragma unroll
        for (int e = 0; e < 4; e++) acc[4 * j + e] += rp[(8 * j + tc + (e & 1)) * HG_BM + wr + 8 * (e >> 1)];
    }
  }
  constexpr int EPI = hg_epi_kind<Src>(0);
  if constexpr (EPI == 2) {
    // GLU: thread t of warpgroup 1 holds, register for register, the up values of thread t of warpgroup 0's gate
    // values.  They pass rounded to T through the A ring, free once both warpgroups' MMAs have retired.
    uint16_t *xch = (uint16_t *)a_ring;   // [NACC][128]
    asm volatile("bar.sync 3, 256;" ::: "memory");
    if (g == 1) {
#pragma unroll
      for (int i = 0; i < NACC; i++) {
        if constexpr (BF) xch[i * 128 + t] = __bfloat16_as_ushort(__float2bfloat16_rn(acc[i]));
        else xch[i * 128 + t] = __half_as_ushort(__float2half_rn(acc[i]));
      }
    }
    asm volatile("bar.sync 3, 256;" ::: "memory");
    if (g == 1) return;
  }
  // PDL: y may only be overwritten once the upstream grid has completed
  if (p.pdl) pdl_wait();
  if constexpr (EPI == 0) {
#pragma unroll
    for (int j = 0; j < NT / 8; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int tok = m0 + 8 * j + tc + (e & 1), n = n0 + wr + 8 * (e >> 1);
        if (tok < p.M && n < p.N) {
          if constexpr (BF) ((__nv_bfloat16 *)p.y)[(size_t)tok * p.N + n] = __float2bfloat16_rn(acc[4 * j + e]);
          else ((__half *)p.y)[(size_t)tok * p.N + n] = __float2half_rn(acc[4 * j + e]);
        }
      }
  } else {
#pragma unroll
    for (int j = 0; j < NT / 8; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int tok = m0 + 8 * j + tc + (e & 1), n = n0 + wr + 8 * (e >> 1);
        if (tok < p.M && src.live(n)) {
          float v = acc[4 * j + e];
          if constexpr (EPI == 2) {   // as fused_glu: T(act(f32(T(gate)))), then the product in T
            const uint16_t u = ((const uint16_t *)a_ring)[(4 * j + e) * 128 + t];
            const float up = BF ? __bfloat162float(__ushort_as_bfloat16(u)) : __half2float(__ushort_as_half(u));
            const float gt = BF ? __bfloat162float(__float2bfloat16_rn(v)) : __half2float(__float2half_rn(v));
            const float a = glu_activation(gt, 0);
            v = (BF ? __bfloat162float(__float2bfloat16_rn(a)) : __half2float(__float2half_rn(a))) * up;
          }
          if constexpr (BF) *(__nv_bfloat16 *)src.out(n, tok) = __float2bfloat16_rn(v);
          else *(__half *)src.out(n, tok) = __float2half_rn(v);
        }
      }
  }
}

// split K over a cluster when the row tiles alone leave SMs idle.  Splits are whole 64-k steps; the partials take
// their own shared memory.
static inline int hg_pick_ksplit(int N, int K, int M, int NT) {
  if (NT > 64) return 1;
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int tiles = ((N + HG_BM - 1) / HG_BM) * ((M + NT - 1) / NT), nk = K / HG_BK;
  int ks = 1;
  for (int c = 2; c <= 4; c *= 2) {
    const int per = (nk + c - 1) / c;
    if (tiles * c <= sms && per >= 4 && per * (c - 1) < nk && hg_smem_bytes(NT, c) <= 227 * 1024) ks = c;
  }
  return ks;
}

// one launch over all token tiles: grid (token tiles, K splits, row tiles), clusters along the K splits.  Token tiles
// run fastest, so the CTAs that read the same weight rows are resident together and share them through L2.
// split_k false: one CTA per tile over all of K, so a row's result does not depend on M (the K split does)
template <class Src, int NT, bool BF>
static cudaError_t hg_launch_nt(const CUtensorMap &tx, const CUtensorMap &tw, const Src &src, HgShape p, cudaStream_t st,
                                bool split_k) {
  const int ks = split_k ? hg_pick_ksplit(p.N, p.K, p.M, NT) : 1;
  const int nk = p.K / HG_BK;
  p.ksteps_per_split = (nk + ks - 1) / ks;
  const size_t smem = hg_smem_bytes(NT, ks);
  auto kern = hg_kernel<Src, NT, BF>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   // per device: set on every launch
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((p.M + NT - 1) / NT, ks, (p.N + HG_BM - 1) / HG_BM);
  cfg.blockDim = dim3(hg_producer_warp(NT) ? HG_THREADS_PW : 256);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (ks > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = 1; attr[na].val.clusterDim.y = ks; attr[na].val.clusterDim.z = 1;
    na++;
  }
  if (p.pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    na++;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, tx, tw, src, p);
}

// x: [M, K] 16-bit row-major (dtype 0 f16, 1 bf16); w_dense: [N, K] when Src::kTmaA.  K % 64 == 0.
template <class Src>
static cudaError_t hg_run(const Src &src, const void *x, const void *w_dense, void *y, int M, int N, int K, int dtype, int pdl, cudaStream_t st,
                          bool split_k = true) {
  if (M <= 0 || N <= 0) return cudaSuccess;
  if (K % HG_BK != 0 || (dtype != MRS_F16 && dtype != MRS_BF16)) return cudaErrorInvalidValue;
  const int NT = M <= 32 ? 32 : M <= 64 ? 64 : M <= 128 ? 128 : 256;
  CUtensorMap tx, tw;
  if (!tc_make_map_2d(&tx, x, (uint64_t)M, (uint64_t)K, HG_BK, (uint32_t)NT, dtype)) return cudaErrorInvalidValue;
  if (Src::kTmaA) {
    if (!tc_make_map_2d(&tw, w_dense, (uint64_t)N, (uint64_t)K, HG_BK, HG_BM, dtype)) return cudaErrorInvalidValue;
  } else {
    tw = tx;   // unused
  }
  HgShape p = {y, M, N, K, 0, pdl};
  const bool bf = dtype == MRS_BF16;
#define MRS_HG(NTV) return bf ? hg_launch_nt<Src, NTV, true>(tx, tw, src, p, st, split_k) : hg_launch_nt<Src, NTV, false>(tx, tw, src, p, st, split_k)
  if (NT == 32) MRS_HG(32);
  if (NT == 64) MRS_HG(64);
  if (NT == 128) MRS_HG(128);
  MRS_HG(256);
#undef MRS_HG
}

}  // namespace mrs
