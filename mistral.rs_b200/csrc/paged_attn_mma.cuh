// paged_attn_mma.cuh — tensor-core decode attention over the HND paged cache (included by paged_attn.cu).
//
// The GQA group of one KV head is an MMA tile: the group's query heads (<= 16) are the M = 16 rows of
// mma.m16n8k16, the tokens of the work tile are N.  Per 64-token step the whole CTA (4 warps) gathers
// the K and V rows of the tile from their pages into XOR-swizzled shared memory with cp.async
// (16-byte copies, page ids staged once), then warp w owns tokens 16w..16w+15 of the step:
// S = Q K^T (16 MMAs for D = 128), online softmax in f32 (base 2), O += P V (16 MMAs, V^T fragments
// through ldmatrix.trans).  ~4 warp-instructions per token where the SIMT kernel needs ~85.
//
// FUSED (mrs_paged_decode_fused): the new token's q/k get RoPE (bit-identical to
// rotary_embedding_positions).  The new token never makes a round trip through the cache: the tile
// that owns the last position rotates k_new into a 16-row shared "new-token tile" (row 0 live),
// attends over it with one extra MMA step, and stores the K/V row to the cache on the side — so
// every tile can gather its first cached step BEFORE griddepcontrol.wait (the cache rows it reads
// were written by earlier tokens), and no fence sits on the critical path.
// MULTI (mrs_paged_decode_fused_multi, speculative verify): every sequence brings q_len query rows at positions
// kv_len - q_len .. kv_len - 1.  The MMA rows are (query i, head g) pairs of the KV head's group, query-major
// (row = i * group + g), split over blockIdx.z in slices of <= 16.  The q_len new K/V rows fill the new-token tile
// (row j live for j < q_len) and query i sees new row j only for j <= i; every tile's cached range stops at
// kv_len - q_len, and the tile whose chunk holds kv_len - 1 owns all new rows.
// CLUSTER: the tiles of one sequence form a thread-block cluster; their partial softmax states go to
// the leader's shared memory through DSMEM and the leader writes the output — no global partials,
// no fence + counter.  Otherwise split-KV partials are merged by the last tile (counter protocol).
//
// Numerics: q (rotated) and P are held in the activation dtype for the MMAs (the reference's decode
// kernels keep P in f32); accumulation is f32.  Tests bound the difference (<= 2.5 ulp of the output).
#pragma once
#include "mma_common.cuh"

namespace mrs {

constexpr int PM_WARPS = 4, PM_THREADS = PM_WARPS * 32, PM_BN = 64;
constexpr int PM_CL_MAX = 8;    // tiles of one sequence per cluster
constexpr int PM_CL_G = 8;      // heads per CTA supported by the cluster merge buffer
constexpr int PM_CL_GM = 16;    // MULTI: rows per CTA in the cluster merge buffer (a whole m16 tile)

template <int D> constexpr size_t pm_smem_bytes(bool fused, bool cluster, int cl_rows = PM_CL_G) {
  return (size_t)4 * PM_BN * D * 2 + (size_t)16 * D * 2 + (fused ? (size_t)2 * 16 * D * 2 : 0) +
         (cluster ? (size_t)PM_CL_MAX * cl_rows * (D + 2) * 4 : 0);
}

__device__ __forceinline__ uint32_t pm_cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void pm_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void pm_st_cluster_f32(const float *local_ptr, uint32_t rank, float v) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_ptr)), "r"(rank));
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote), "f"(v) : "memory");
}

template <typename T, int D, bool FUSED, bool CLUSTER, bool MULTI>
__device__ __forceinline__ void paged_decode_mma_body(const PagedParams &p) {
  static_assert(!MULTI || FUSED, "the multi-query form is the fused one");
  constexpr int KSTEPS = D / 16, DT = D / 8, CPR = D / 8, LPT = D / 8;
  constexpr int CLG = MULTI ? PM_CL_GM : PM_CL_G;
  constexpr int TILE_BYTES = PM_BN * D * 2;
  extern __shared__ __align__(128) uint8_t pm_smem[];
  uint8_t *sk[2] = {pm_smem, pm_smem + 2 * TILE_BYTES};
  uint8_t *sv[2] = {pm_smem + TILE_BYTES, pm_smem + 3 * TILE_BYTES};
  uint8_t *sq = pm_smem + 4 * TILE_BYTES;                  // [16][D] query tile
  uint8_t *snk = sq + 16 * D * 2, *snv = snk + 16 * D * 2;  // FUSED: new-token K / V tiles (row 0 live)
  float *dsm = (float *)(sq + 16 * D * 2 + (FUSED ? 2 * 16 * D * 2 : 0));   // CLUSTER: [PM_CL_MAX][CLG][D + 2]
  __shared__ int st_pages[2048 / 8 + 2];
  __shared__ int sm_last;

  const int tile = blockIdx.x, kvh = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (p.pdl && tid == 0) pdl_launch_dependents();
  const bool valid = p.block_valid_mask == nullptr || p.block_valid_mask[tile] != 0;
  if (!CLUSTER && !valid) return;
  int seq = tile, chunk_idx = 0;
  if (p.request_indices != nullptr) { seq = p.request_indices[tile]; chunk_idx = p.kv_tile_indices[tile]; }
  const int p0 = p.kv_indptr[seq], p1 = p.kv_indptr[seq + 1];
  const int32_t *pages = p.kv_indices + p0;
  const int kv_len = (p1 > p0) ? (p1 - p0 - 1) * p.page_size + p.kv_last_page_len[seq] : 0;
  int chunk = p.kv_chunk_size_ptr ? *p.kv_chunk_size_ptr : p.kv_chunk_size;
  if (chunk <= 0) chunk = kv_len > 0 ? kv_len : 1;
  const int t_begin = chunk_idx * chunk;
  const int t_end = valid ? min(kv_len, t_begin + chunk) : t_begin;
  const bool partial = p.tmp_o != nullptr;
  const int group = p.num_heads / p.num_kv_heads;
  const int Q = MULTI ? p.q_len : 1;                       // query rows per sequence
  const int h0 = kvh * group + blockIdx.z * p.heads_per_cta;
  const int gsize = min(p.heads_per_cta, group * Q - (int)blockIdx.z * p.heads_per_cta);   // MMA rows of this CTA, <= 16
  // MMA row r -> (query row qi of the sequence, query head h); MULTI clamps padding rows onto the last live one
  auto row_head = [&](int r, int &qi, int &h) {
    if constexpr (MULTI) {
      const int rr = min((int)blockIdx.z * p.heads_per_cta + r, group * Q - 1);
      qi = rr / group; h = kvh * group + rr % group;
    } else {
      qi = 0; h = h0 + r;
    }
  };
  // row of (tile or sequence t, query row qi, head h = MMA row g) in a [*, Q * heads] array: tmp_o / tmp_lse by
  // tile, out by sequence
  auto qh_row = [&](int t, int qi, int h, int g) -> int64_t {
    if constexpr (MULTI) return (int64_t)(t * Q + qi) * p.num_heads + h;
    else return (int64_t)t * p.num_heads + h0 + g;
  };
  const int win_lo = (p.window_left >= 0) ? max(0, kv_len - 1 - p.window_left) : 0;
  bool owns_new = false;
  if constexpr (FUSED) owns_new = valid && kv_len > 0 && (kv_len - 1) >= t_begin && (kv_len - 1) < t_end;
  // the new rows are attended from shared memory; MULTI: no tile reads a cached row at or past kv_len - q_len
  const int t_cache_end = MULTI ? max(t_begin, min(t_end, kv_len - Q)) : (owns_new ? kv_len - 1 : t_end);

  // page ids of the chunk -> shared memory (the page table predates the upstream kernel)
  const int pg0 = t_begin / p.page_size;
  const int npg = (t_cache_end > t_begin) ? (t_cache_end - 1) / p.page_size - pg0 + 1 : 0;
  for (int i = tid; i < npg && i < (int)(sizeof(st_pages) / sizeof(int)); i += PM_THREADS) st_pages[i] = pages[pg0 + i];
  const bool pages_in_smem = npg <= (int)(sizeof(st_pages) / sizeof(int));
  if constexpr (FUSED) {
    if (owns_new)
      for (int i = tid; i < 2 * 16 * D * 2 / 16; i += PM_THREADS) ((uint4 *)snk)[i] = make_uint4(0u, 0u, 0u, 0u);
  }
  __syncthreads();

  const T *kc = (const T *)p.kc, *vc = (const T *)p.vc;
  auto load_tile = [&](int it, int buf) {       // cached tokens t_begin + 64 it .. +63 of the chunk
    const int t0 = t_begin + it * PM_BN;
    for (int c = tid; c < PM_BN * CPR; c += PM_THREADS) {
      const int row = c / CPR, ch = c % CPR;
      const int t = t0 + row;
      const bool ok = t < t_cache_end;
      int64_t goff = 0;
      if (ok) {
        const int pgi = t / p.page_size;
        const int64_t pg = pages_in_smem ? st_pages[pgi - pg0] : pages[pgi];
        goff = pg * p.kv_block_stride + (int64_t)kvh * p.kv_head_stride + (int64_t)(t % p.page_size) * D + ch * 8;
      }
      cp_async16(sk[buf] + tile_off<D>(row, ch), kc + goff, ok);
      cp_async16(sv[buf] + tile_off<D>(row, ch), vc + goff, ok);
    }
    cp_async_commit();
  };
  const int ntiles = (t_cache_end > t_begin) ? (t_cache_end - t_begin + PM_BN - 1) / PM_BN : 0;
  if (ntiles > 0) load_tile(0, 0);     // cache rows of earlier tokens: safe before the upstream kernel is done
  else cp_async_commit();
  if (p.pdl) pdl_wait();

  // ---- query tile: rows = heads of the group (zero beyond gsize), RoPE in the fused form
  if (valid) {
    for (int idx = tid; idx < 16 * LPT; idx += PM_THREADS) {    // whole warps stay together (shuffles in rope)
      const int g = idx / LPT, gl = idx % LPT;
      int qi, h;
      row_head(g, qi, h);
      float x[8];
      if (g < gsize) Vec8<T>::load((const T *)p.q + (int64_t)(seq * Q + qi) * p.q_stride_n + (int64_t)h * p.q_stride_h + gl * 8, x);
      else {
#pragma unroll
        for (int i = 0; i < 8; i++) x[i] = 0.f;
      }
      if constexpr (FUSED) {
        const int64_t pos = p.positions[seq * Q + qi];
        rope_any<T, D>(x, (const T *)p.rope_cos + pos * (D / 2), (const T *)p.rope_sin + pos * (D / 2), gl, p.rope_interleaved != 0);
      }
      Vec8<T>::store((T *)(sq + tile_off<D>(g, gl)), x);
    }
    if constexpr (MULTI) {
      if (owns_new) {
        // new row j per LPT-lane group (32 / LPT per warp); a warp's trip count is uniform for the RoPE shuffles
        constexpr int GPW = 32 / LPT;
        const int gl = lane % LPT;
        for (int j0 = warp * GPW; j0 < Q; j0 += PM_WARPS * GPW) {
          const bool live = j0 + lane / LPT < Q;
          const int j = min(j0 + lane / LPT, Q - 1);
          const int64_t row = (int64_t)seq * Q + j;
          float kn[8], vn[8];
          Vec8<T>::load((const T *)p.k_new + row * p.kv_new_stride + (int64_t)kvh * D + gl * 8, kn);
          Vec8<T>::load((const T *)p.v_new + row * p.kv_new_stride + (int64_t)kvh * D + gl * 8, vn);
          const int64_t pos = p.positions[row];
          rope_any<T, D>(kn, (const T *)p.rope_cos + pos * (D / 2), (const T *)p.rope_sin + pos * (D / 2), gl, p.rope_interleaved != 0);
          if (live) {
            Vec8<T>::store((T *)(snk + tile_off<D>(j, gl)), kn);
            Vec8<T>::store((T *)(snv + tile_off<D>(j, gl)), vn);
            const int64_t slot = p.slot_mapping[row];
            if (slot >= 0 && blockIdx.z == 0) {
              const int64_t base = (slot / p.page_size) * p.kv_block_stride + (int64_t)kvh * p.kv_head_stride + (slot % p.page_size) * D;
              Vec8<T>::store((T *)p.kc + base + gl * 8, kn);
              Vec8<T>::store((T *)p.vc + base + gl * 8, vn);
            }
          }
        }
      }
    } else if constexpr (FUSED) {
      if (owns_new && warp == 0) {
        // every LPT-lane group computes the same row so the RoPE shuffles stay warp-wide
        const int gl = lane % LPT;
        float kn[8], vn[8];
        Vec8<T>::load((const T *)p.k_new + (int64_t)seq * p.kv_new_stride + (int64_t)kvh * D + gl * 8, kn);
        Vec8<T>::load((const T *)p.v_new + (int64_t)seq * p.kv_new_stride + (int64_t)kvh * D + gl * 8, vn);
        const int64_t pos = p.positions[seq];
        rope_any<T, D>(kn, (const T *)p.rope_cos + pos * (D / 2), (const T *)p.rope_sin + pos * (D / 2), gl, p.rope_interleaved != 0);
        if (lane < LPT) {
          Vec8<T>::store((T *)(snk + tile_off<D>(0, gl)), kn);
          Vec8<T>::store((T *)(snv + tile_off<D>(0, gl)), vn);
          const int64_t slot = p.slot_mapping[seq];
          if (slot >= 0 && blockIdx.z == 0) {     // the cache write is off the critical path: nobody reads it this step
            const int64_t base = (slot / p.page_size) * p.kv_block_stride + (int64_t)kvh * p.kv_head_stride + (slot % p.page_size) * D;
            Vec8<T>::store((T *)p.kc + base + gl * 8, kn);
            Vec8<T>::store((T *)p.vc + base + gl * 8, vn);
          }
        }
      }
    }
  }
  __syncthreads();

  uint32_t qa[KSTEPS][4];
#pragma unroll
  for (int ks = 0; ks < KSTEPS; ks++)
    ldsm_x4(smem_u32(sq + tile_off<D>(lane & 15, 2 * ks + (lane >> 4))), qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3]);

  float oacc[DT][4];
#pragma unroll
  for (int i = 0; i < DT; i++) { oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float scale_log2 = p.sm_scale * 1.4426950408889634f;

  // one warp step over 16 tokens held in rows row0..row0+15 of (kt, vt); token of row j is t_first + j,
  // live when win_lo <= t < t_hi, with t_hi0 for MMA rows 0..7 and t_hi1 for rows 8..15
  auto step16 = [&](const uint8_t *kt, const uint8_t *vt, int row0, int t_first, int t_hi0, int t_hi1) {
    float sacc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ks++) {
      const int row = row0 + (lane & 7) + ((lane >> 4) << 3);
      const int ch = 2 * ks + ((lane >> 3) & 1);
      uint32_t b0, b1, b2, b3;
      ldsm_x4(smem_u32(kt + tile_off<D>(row, ch)), b0, b1, b2, b3);
      mma16816<T>(sacc[0], qa[ks], b0, b1);
      mma16816<T>(sacc[1], qa[ks], b2, b3);
    }
    float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
    for (int j = 0; j < 2; j++) {
#pragma unroll
      for (int e = 0; e < 4; e++) {
        float s = sacc[j][e];
        if (p.softcap > 0.f) s = p.softcap * tanhf(s * p.sm_scale / p.softcap) * 1.4426950408889634f;
        else s *= scale_log2;
        const int t = t_first + 8 * j + 2 * (lane & 3) + (e & 1);
        if (t >= ((e >> 1) ? t_hi1 : t_hi0) || t < win_lo) s = -INFINITY;
        sacc[j][e] = s;
        mx[e >> 1] = fmaxf(mx[e >> 1], s);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; r++) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; r++) {
      corr[r] = (mx[r] == -INFINITY) ? 1.f : exp2f(m_run[r] - mx[r]);
      m_run[r] = mx[r];
    }
    uint32_t pa[4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const float p0 = (mx[0] == -INFINITY) ? 0.f : exp2f(sacc[j][0] - mx[0]);
      const float p1 = (mx[0] == -INFINITY) ? 0.f : exp2f(sacc[j][1] - mx[0]);
      const float p2 = (mx[1] == -INFINITY) ? 0.f : exp2f(sacc[j][2] - mx[1]);
      const float p3 = (mx[1] == -INFINITY) ? 0.f : exp2f(sacc[j][3] - mx[1]);
      rs[0] += p0 + p1; rs[1] += p2 + p3;
      pa[2 * j] = pack2<T>(p0, p1);
      pa[2 * j + 1] = pack2<T>(p2, p3);
    }
#pragma unroll
    for (int r = 0; r < 2; r++) l_run[r] = l_run[r] * corr[r] + rs[r];
#pragma unroll
    for (int i = 0; i < DT; i++) { oacc[i][0] *= corr[0]; oacc[i][1] *= corr[0]; oacc[i][2] *= corr[1]; oacc[i][3] *= corr[1]; }
#pragma unroll
    for (int dp = 0; dp < DT / 2; dp++) {
      const int row = row0 + (lane & 7) + (((lane >> 3) & 1) << 3);
      const int ch = 2 * dp + (lane >> 4);
      uint32_t b0, b1, b2, b3;
      ldsm_x4_t(smem_u32(vt + tile_off<D>(row, ch)), b0, b1, b2, b3);
      mma16816<T>(oacc[2 * dp], pa, b0, b1);
      mma16816<T>(oacc[2 * dp + 1], pa, b2, b3);
    }
  };

  for (int it = 0; it < ntiles; it++) {
    const int buf = it & 1;
    if (it + 1 < ntiles) load_tile(it + 1, buf ^ 1);
    else cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const int tw = t_begin + it * PM_BN + 16 * warp;     // first token of this warp's 16
    if (tw < t_cache_end) step16(sk[buf], sv[buf], 16 * warp, tw, t_cache_end, t_cache_end);   // warp-uniform
    __syncthreads();
  }
  cp_async_wait<0>();
  if constexpr (MULTI) {
    if (owns_new && warp == 0) {          // the new rows, from shared memory: query row qi sees new rows 0..qi
      int qa, qb, h;
      row_head(lane >> 2, qa, h);
      row_head((lane >> 2) + 8, qb, h);
      step16(snk, snv, 0, kv_len - Q, kv_len - Q + qa + 1, kv_len - Q + qb + 1);
    }
  } else if constexpr (FUSED) {
    if (owns_new && warp == 0) step16(snk, snv, 0, kv_len - 1, kv_len, kv_len);    // the new token, from shared memory
  }
#pragma unroll
  for (int r = 0; r < 2; r++) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }

  // ---- merge the four warp states: rows 0..7 of the m16 tile live in (c0, c1), rows 8..15 in (c2, c3)
  float *mo = (float *)pm_smem;                    // [PM_WARPS][16][D] f32 (the K/V buffers are free now)
  float *mm = mo + PM_WARPS * 16 * D, *ml = mm + PM_WARPS * 16;
  {
    const int r0 = lane >> 2;
#pragma unroll
    for (int i = 0; i < DT; i++) {
      const int col = 8 * i + 2 * (lane & 3);
      *(float2 *)(mo + ((size_t)warp * 16 + r0) * D + col) = make_float2(oacc[i][0], oacc[i][1]);
      *(float2 *)(mo + ((size_t)warp * 16 + r0 + 8) * D + col) = make_float2(oacc[i][2], oacc[i][3]);
    }
    if ((lane & 3) == 0) {
      mm[warp * 16 + r0] = m_run[0]; mm[warp * 16 + r0 + 8] = m_run[1];
      ml[warp * 16 + r0] = l_run[0]; ml[warp * 16 + r0 + 8] = l_run[1];
    }
  }
  __syncthreads();
  uint32_t crank = 0;
  if constexpr (CLUSTER) crank = pm_cluster_rank();
  for (int idx = tid; idx < gsize * D; idx += PM_THREADS) {
    const int g = idx / D, d = idx % D;
    int qi, h;
    row_head(g, qi, h);
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < PM_WARPS; w++) M = fmaxf(M, mm[w * 16 + g]);
    float L = 0.f, acc = 0.f;
    if (M > -INFINITY) {
#pragma unroll
      for (int w = 0; w < PM_WARPS; w++) {
        const float c = exp2f(mm[w * 16 + g] - M);
        L += ml[w * 16 + g] * c;
        acc += mo[((size_t)w * 16 + g) * D + d] * c;
      }
    }
    if constexpr (CLUSTER) {
      // unnormalised state of this tile -> slot `crank` of the leader's merge buffer
      float *slot = dsm + ((size_t)crank * CLG + g) * (D + 2);
      pm_st_cluster_f32(slot + d, 0u, acc);
      if (d == 0) { pm_st_cluster_f32(slot + D, 0u, M); pm_st_cluster_f32(slot + D + 1, 0u, L); }
    } else {
      const float val = (L > 0.f) ? acc / L : 0.f;
      if (partial) {
        // partials [tiles, Q * heads]
        ((T *)p.tmp_o)[qh_row(tile, qi, h, g) * D + d] = (T)val;
        // natural-log lse, as the SIMT kernel and merge_partials_kernel expect (M is a base-2 exponent)
        if (d == 0) p.tmp_lse[qh_row(tile, qi, h, g)] = (L > 0.f) ? (M + log2f(L)) * 0.6931471805599453f : -INFINITY;
      } else {
        ((T *)p.out)[qh_row(seq, qi, h, g) * D + d] = (T)val;
      }
    }
  }

  if constexpr (CLUSTER) {
    pm_cluster_sync();
    if (crank == 0 && valid) {
      const int nt = p.o_indptr[seq + 1] - p.o_indptr[seq];     // live tiles of this sequence (ranks 0..nt-1)
      for (int idx = tid; idx < gsize * D; idx += PM_THREADS) {
        const int g = idx / D, d = idx % D;
        int qi, h;
        row_head(g, qi, h);
        float M = -INFINITY;
        for (int r = 0; r < nt; r++) M = fmaxf(M, dsm[((size_t)r * CLG + g) * (D + 2) + D]);
        float L = 0.f, acc = 0.f;
        if (M > -INFINITY) {
          for (int r = 0; r < nt; r++) {
            const float *slot = dsm + ((size_t)r * CLG + g) * (D + 2);
            const float c = exp2f(slot[D] - M);
            L += slot[D + 1] * c;
            acc += slot[d] * c;
          }
        }
        ((T *)p.out)[qh_row(seq, qi, h, g) * D + d] = (T)((L > 0.f) ? acc / L : 0.f);
      }
    }
  } else if constexpr (FUSED) {
    if (partial) {
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
        for (int idx = tid; idx < gsize * D; idx += PM_THREADS) {
          const int g = idx / D, d = idx % D;
          int qi, h;
          row_head(g, qi, h);
          float M = -INFINITY;
          for (int t = t0; t < t1; t++) M = fmaxf(M, __ldcg(p.tmp_lse + (int64_t)(t * Q + qi) * p.num_heads + h));
          float W = 0.f, acc = 0.f;
          if (M > -INFINITY) {
            for (int t = t0; t < t1; t++) {
              const float w = __expf(__ldcg(p.tmp_lse + (int64_t)(t * Q + qi) * p.num_heads + h) - M);
              const unsigned short raw = __ldcg((const unsigned short *)p.tmp_o + ((int64_t)(t * Q + qi) * p.num_heads + h) * D + d);
              T tv;
              memcpy(&tv, &raw, 2);
              W += w;
              acc += w * (float)tv;
            }
          }
          ((T *)p.out)[((int64_t)(seq * Q + qi) * p.num_heads + h) * D + d] = (T)((W > 0.f) ? acc / W : 0.f);
        }
      }
    }
  }
}

template <typename T, int D, bool FUSED, bool CLUSTER>
__global__ void __launch_bounds__(PM_THREADS, 2) paged_decode_mma_kernel(const PagedParams p) {
  paged_decode_mma_body<T, D, FUSED, CLUSTER, false>(p);
}
template <typename T, int D, bool CLUSTER>
__global__ void __launch_bounds__(PM_THREADS, 2) paged_decode_mma_multi_kernel(const PagedParams p) {
  paged_decode_mma_body<T, D, true, CLUSTER, true>(p);
}

}  // namespace mrs
