// mmvq.cu — streaming decode GEMV (batch 1..8) over ggml quant blocks for sm_90a.
//
// Drop-in for the reference's `launch_mmvq_gguf_*` C ABI
// (REF: mistralrs-quant/kernels/mmvq_gguf/mmvq_gguf.cu:1322-1641, declared in
// mistralrs-quant/src/gguf/ffi.rs and called from src/gguf/fast_mmvq.rs:299,472,682).
//
// Design (written for this GPU, not a port of the dp4a kernel):
//  * The weight matrix is a flat byte stream.  Each CTA owns a contiguous range of rows and a
//    dedicated producer warp streams it HBM -> shared memory with cp.async.bulk (TMA engine)
//    into a multi-stage mbarrier ring: one 16-byte-aligned bulk copy per (row, 1024-element K
//    segment).  The byte phase (address mod 16) is preserved in shared memory, so ggml types
//    whose blocks are not 16-byte multiples (Q6_K 210 B, Q8_0 34 B, ...) need no re-tiling.
//  * 8 consumer warps; warp w owns two rows of the pass, lane l owns the l-th 32-weight unit
//    of the current K segment.  Activations are Q8_1-quantised (the reference's decode
//    numerics) and pre-permuted into unit order in shared memory once per CTA.
//  * Partial sums stay in registers across K segments; one butterfly reduction per row.
//  * Optional fused prologue (RMSNorm + Q8_1 quantisation of raw activations) and epilogue
//    (GLU, residual add) — the `mrs_*` entry points; the reference-shaped launchers use the
//    plain prologue (pre-quantised Q8_1 input).
//  * PDL: the producer starts streaming weights before griddepcontrol.wait, so under
//    programmatic stream serialisation the next GEMV's weights are already in flight while the
//    previous kernel drains.
#include "mmvq_types.cuh"

#include <stdio.h>

namespace mrs {

// CTA shape: NCW = 8 consumer warps + 1 producer warp, two CTAs per SM; a stage holds 2
// row-segments per consumer warp.
constexpr int SSW = 8;  // warps that take part in the RMSNorm sum of squares (fixes its summation order)

constexpr int MAX_STAGES = 12;

enum { MODE_PLAIN = 0, MODE_GLU = 1, MODE_QKV = 2 };

__device__ __forceinline__ uint4 sel_u4(bool first, const uint4 &a, const uint4 &b) {
  return make_uint4(first ? a.x : b.x, first ? a.y : b.y, first ? a.z : b.z, first ? a.w : b.w);
}

#ifdef MRS_TIMELINE
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define MRS_STAMP(i) do { if (p.dbg != nullptr) p.dbg[(size_t)blockIdx.x * 16 + (i)] = gtimer(); } while (0)
#else
#define MRS_STAMP(i) do { } while (0)
#endif
enum { X_Q8_1 = 0, X_RAW = 1 };

struct MmvqParams {
  const uint8_t *w[3];
  void *dst[3];
  int nrows[3];
  const void *x;         // X_Q8_1: block_q8_1[ncols][stride_col_y]; X_RAW: act[ncols][K]
  const void *norm_w;    // optional RMSNorm weight (X_RAW only)
  const void *residual;  // optional residual added in the epilogue (MODE_PLAIN only)
  float eps;
  int xkind, xdtype;
  int K, stride_col_y, stride_col_dst, ncols;
  int mode, activation, dst_dtype;
  int nstages, vrows, pdl, flags;
  int dst_q8;            // MODE_GLU: dst[0] is block_q8_1[ncols][stride_col_dst], the Q8_1 form of the output
#ifdef MRS_TIMELINE
  unsigned long long *dbg;  // dev build: [gridDim.x][16] globaltimer stamps of this launch
#endif
};

template <int T, int NCW, int UPLX = QT<T>::UPL> struct Geo {
  using Q = QT<T>;
  static constexpr int SLOTS = 2 * NCW;
  static constexpr int UPL = UPLX;                           // units per lane per K segment (per-launch: long streams take 2x)
  static constexpr int SEG_UNITS = 32 * UPL;                 // 32-weight units per K segment
  static constexpr int SEG_BLOCKS = SEG_UNITS / Q::UPB;      // weight blocks per segment (NB)
  static constexpr int SEG_BYTES = SEG_BLOCKS * Q::BYTES;    // bytes per row-segment (~2-3.5 KB)
  static constexpr int SLOT_BYTES = (SEG_BYTES + 30 + 15) & ~15;
  static constexpr int STAGE_BYTES = SLOTS * SLOT_BYTES;
  static constexpr int XU_BYTES = 32 + 4 * Q::AUX;           // smem bytes per unit per column
  // lane -> (block within segment, chunk): blk = lane % NBL, c = ui * CPS + lane / NBL
  static constexpr int NBL = (Q::UPB == 1) ? 32 : (SEG_BLOCKS < 32 ? SEG_BLOCKS : 32);
  static constexpr int CPS = (Q::UPB == 1) ? 1 : 32 / NBL;
  static_assert(Q::UPB == 1 || (NBL * CPS == 32 && CPS * UPL == Q::UPB), "segment geometry");
};

// position p in the consumption-ordered activation array <-> (weight block, chunk)
template <int T, int UPL> __device__ __forceinline__ int unit_to_pos(int blk, int c) {
  using G = Geo<T, 8, UPL>;
  if constexpr (QT<T>::UPB == 1) {
    return blk;
  } else {
    const int s = blk / G::SEG_BLOCKS, bl = blk - s * G::SEG_BLOCKS;
    return s * G::SEG_UNITS + (c / G::CPS) * 32 + bl + G::NBL * (c % G::CPS);
  }
}
template <int T, int UPL> __device__ __forceinline__ void pos_to_unit(int pos, int &blk, int &c) {
  using G = Geo<T, 8, UPL>;  // segment geometry does not depend on the CTA shape
  if constexpr (QT<T>::UPB == 1) {
    blk = pos; c = 0;
  } else {
    const int s = pos / G::SEG_UNITS, r = pos - s * G::SEG_UNITS;
    const int ui = r >> 5, lane = r & 31;
    blk = s * G::SEG_BLOCKS + (lane % G::NBL);
    c = ui * G::CPS + lane / G::NBL;
  }
}

__device__ __forceinline__ void resolve_row(const MmvqParams &p, int vrow, int which, int &m, int &row) {
  if (p.mode == MODE_QKV) {
    if (vrow < p.nrows[0]) { m = 0; row = vrow; }
    else if (vrow < p.nrows[0] + p.nrows[1]) { m = 1; row = vrow - p.nrows[0]; }
    else { m = 2; row = vrow - p.nrows[0] - p.nrows[1]; }
  } else if (p.mode == MODE_GLU) {
    m = which; row = vrow;
  } else {
    m = 0; row = vrow;
  }
}

// accessor handed to QT::aux — d8/s8 of q8_1 block j relative to the weight block
struct YGlobal {
  const block_q8_1 *y;
  __device__ __forceinline__ float d(int j) const { return __low2float(y[j].ds); }
  __device__ __forceinline__ float s(int j) const { return __high2float(y[j].ds); }
};
struct YSmem {
  const float2 *ds;  // (d, s) per q8 block, already widened
  __device__ __forceinline__ float d(int j) const { return ds[j].x; }
  __device__ __forceinline__ float s(int j) const { return ds[j].y; }
};

// Q8_1 quantisation of one 32-element block held by one thread (values already f32).
// Same arithmetic as REF mmvq_gguf.cu:1235-1251 incl. the butterfly summation order and the
// approximate divisions the reference gets from --use_fast_math.
__device__ __forceinline__ void quantize_block_q8_1(const float *v, int8_t *q, float &d_out, float &s_out) {
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 32; i++) amax = fmaxf(amax, fabsf(v[i]));
  float s[16];
#pragma unroll
  for (int i = 0; i < 16; i++) s[i] = v[i] + v[i + 16];
#pragma unroll
  for (int m = 8; m > 0; m >>= 1) {
#pragma unroll
    for (int i = 0; i < m; i++) s[i] = s[i] + s[i + m];
  }
  const float d = __fdividef(amax, 127.0f);
#pragma unroll
  for (int i = 0; i < 32; i++) q[i] = (amax == 0.0f) ? (int8_t)0 : (int8_t)roundf(__fdividef(v[i], d));
  d_out = __half2float(__float2half_rn(d));
  s_out = __half2float(__float2half_rn(s[0]));
}

// The whole CTA program; `cta` of `ncta` CTAs share the virtual rows of `p` (the wrappers below pass
// blockIdx/gridDim, or the position inside one half of a two-type launch).
template <int T, int NCOLS, bool FAST, int NCW, int UPL = QT<T>::UPL>
__device__ __forceinline__ void mmvq_body(const MmvqParams &p, const int cta, const int ncta) {
  using Q = QT<T>;
  using G = Geo<T, NCW, UPL>;
  constexpr int SLOTS = 2 * NCW;
  extern __shared__ __align__(128) uint8_t smem[];

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int nblocks = p.K / Q::QK;
  const int nseg = (nblocks + G::SEG_BLOCKS - 1) / G::SEG_BLOCKS;
  const int npos = nseg * G::SEG_UNITS;  // padded unit count (consumption order)
  const int row_bytes = nblocks * Q::BYTES;
  const int nst = p.nstages;

  // smem carve-up (plain offsets so every access stays in the shared window):
  // [barriers 256 B][xq0 | xq1 | xa][ring][(d,s) scratch for the fused prologue]
  uint64_t *full = (uint64_t *)smem;
  uint64_t *empty = full + MAX_STAGES;
  const uint32_t off_xq0 = 256;
  const uint32_t off_xq1 = off_xq0 + (uint32_t)NCOLS * npos * 16;
  const uint32_t off_xa = off_xq1 + (uint32_t)NCOLS * npos * 16;
  const uint32_t off_qb = off_xa + (uint32_t)NCOLS * npos * Q::AUX * 4;
  const uint32_t off_ring = (off_qb + (p.dst_q8 ? 2u * NCOLS * 32 * 4 : 0u) + 127u) & ~127u;
  int4 *xq0 = (int4 *)(smem + off_xq0);   // [NCOLS][npos]
  int4 *xq1 = (int4 *)(smem + off_xq1);   // [NCOLS][npos]
  float *xa = (float *)(smem + off_xa);   // [NCOLS][npos][AUX]
  float *qb = (float *)(smem + off_qb);   // dst_q8: [2][NCOLS][32] GLU outputs of a 32-row group, double-buffered
  uint8_t *ring = smem + off_ring;

  if (tid == 0) {
    MRS_STAMP(0);
    for (int i = 0; i < nst; i++) { mbar_init(&full[i], 32); mbar_init(&empty[i], NCW); }
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) MRS_STAMP(1);

  // contiguous virtual-row range of this CTA; a launch that writes Q8_1 hands out whole 32-row groups (one block each)
  const int gran = p.dst_q8 ? 32 : 1;
  const int vr0 = gran * (int)((long long)(p.vrows / gran) * cta / ncta);
  const int vr1 = gran * (int)((long long)(p.vrows / gran) * (cta + 1) / ncta);
  const int P = (p.mode == MODE_GLU) ? NCW : SLOTS;  // virtual rows per pass

  if (warp == NCW) {
    // =========================== producer warp: lane == slot ===========================
    // Weights are immutable, so streaming may start before the upstream kernel finished.  Let the
    // downstream kernel launch as early as possible too: it only prefetches ITS weights until its
    // own griddepcontrol.wait, which orders it after this whole grid.
    if (p.pdl) pdl_launch_dependents();
    int stage = 0, phase = 0;
    const int slot = lane;
    for (int base = vr0; base < vr1; base += P) {
      const uint8_t *rowp = nullptr;
      if (slot < SLOTS) {
        const int vrow = (p.mode == MODE_GLU) ? base + (slot >> 1) : base + slot;
        if (vrow < vr1) {
          int m, row;
          resolve_row(p, vrow, slot & 1, m, row);
          rowp = p.w[m] + (size_t)row * row_bytes;
        }
      }
      for (int s = 0; s < nseg; s++) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (rowp != nullptr) {
          const int off = s * G::SEG_BYTES;
          const int len = min(G::SEG_BYTES, row_bytes - off);
          const uintptr_t a = (uintptr_t)(rowp + off);
          const uintptr_t a0 = a & ~(uintptr_t)15;
          const uint32_t bytes = (uint32_t)(((a + len + 15) & ~(uintptr_t)15) - a0);
          mbar_arrive_expect_tx(&full[stage], bytes);
          bulk_g2s(ring + (uint32_t)stage * G::STAGE_BYTES + (uint32_t)slot * G::SLOT_BYTES, (const void *)a0, bytes, &full[stage]);
        } else {
          mbar_arrive(&full[stage]);
        }
        if (lane == 0 && base == vr0 && s == 0) MRS_STAMP(2);
        if (++stage == nst) { stage = 0; phase ^= 1; }
      }
    }
    if (lane == 0) MRS_STAMP(10);
    return;
  }

  // ============================= consumer warps =============================
  const int ctid = tid;  // 0 .. NCW*32-1
  constexpr int NCT = NCW * 32;
  constexpr int SST = SSW * 32;  // threads in the sum-of-squares pass (canonical order for both CTA shapes)
  // The RMSNorm weight is immutable: fetch it before the PDL wait — the first two chunks of every
  // thread (all of K <= 4096) into registers, anything longer only towards the cache.
  const bool reg16 = p.xkind == X_RAW && p.xdtype != MRS_F32;
  uint4 nwr0 = make_uint4(0u, 0u, 0u, 0u), nwr1 = nwr0;
  if (p.xkind == X_RAW && p.norm_w != nullptr) {
    if (reg16) {
      if (ctid < (p.K >> 3)) nwr0 = __ldg((const uint4 *)p.norm_w + ctid);
      if (NCW == SSW && ctid + NCT < (p.K >> 3)) nwr1 = __ldg((const uint4 *)p.norm_w + ctid + NCT);
    }
    if (!reg16 || (p.K >> 3) > 2 * NCT) {
      const int nbytes = p.K * ((p.xdtype == MRS_F32) ? 4 : 2);
      for (int off = ctid * 128; off < nbytes; off += NCT * 128)
        asm volatile("prefetch.global.L1 [%0];" ::"l"((const char *)p.norm_w + off));
    }
  }
  if (p.pdl) pdl_wait();  // activations come from the upstream kernel
  if (tid == 0) MRS_STAMP(3);
  if (p.xkind == X_Q8_1) {
    // gather pre-quantised Q8_1 blocks straight into consumption order.  QT::aux over the blocks yields the same floats
    // as QT::chunk_aux in the raw prologue below (same half-rounded d / sum, same integer sums), so a launch fed Q8_1
    // computes bit for bit what it computes from the raw activations (tests/test_mmvq_q8_io_gpu.py)
    const block_q8_1 *y = (const block_q8_1 *)p.x;
    for (int idx = ctid; idx < NCOLS * npos; idx += NCT) {
      const int col = idx / npos, pos = idx - col * npos;
      int blk, c;
      pos_to_unit<T, UPL>(pos, blk, c);
      int q[8];
      float a[Q::AUX];
      if (col < p.ncols && blk < nblocks) {
        const block_q8_1 *yb = y + (size_t)col * p.stride_col_y + (size_t)blk * (Q::QK / 32);
#pragma unroll
        for (int w = 0; w < 8; w++) {
          const int e = Q::x_elem(c, w);
          q[w] = *(const int *)(yb[e >> 5].qs + (e & 31));
        }
        Q::aux(q, c, YGlobal{yb}, a);
      } else {
#pragma unroll
        for (int w = 0; w < 8; w++) q[w] = 0;
#pragma unroll
        for (int i = 0; i < Q::AUX; i++) a[i] = 0.f;
      }
      xq0[idx] = make_int4(q[0], q[1], q[2], q[3]);
      xq1[idx] = make_int4(q[4], q[5], q[6], q[7]);
#pragma unroll
      for (int i = 0; i < Q::AUX; i++) xa[(size_t)idx * Q::AUX + i] = a[i];
    }
  } else {
    // fused prologue: (optional RMSNorm) -> round to activation dtype -> Q8_1 -> consumption
    // order, in ONE pass: every thread owns 8-element chunks (one 16-byte load), four
    // neighbouring lanes form a Q8_1 block, and each thread stores its 8 quantised bytes and the
    // unit's aux terms straight at their consumption-order position (QT::chunk_dest/chunk_aux) —
    // no natural-order staging, no permute pass.
    float *red = (float *)(smem + 192);  // 8 floats of scratch inside the header page
    const int nchunks = p.K >> 3;                  // 8-element chunks; 4 neighbouring lanes = one Q8_1 block
    const int nchunks_w = (nchunks + 31) & ~31;    // whole warps iterate together (shuffles below)
    for (int col = 0; col < NCOLS; col++) {
      const bool live = col < p.ncols;
      float inv_rms = 1.0f;
      // the first two chunks of each thread stay in registers between the passes (16-bit dtypes)
      uint4 xr0 = make_uint4(0u, 0u, 0u, 0u), xr1 = xr0;
      if (reg16 && live) {
        const uint4 *xc = (const uint4 *)((const uint16_t *)p.x + (int64_t)col * p.K);
        if (ctid < nchunks) xr0 = xc[ctid];
        if (ctid < SST && ctid + SST < nchunks) xr1 = xc[ctid + SST];
      }
      if (p.norm_w != nullptr && live) {
        // pass 0: sum of squares by the first SST threads, 8 elements (16 B for 16-bit dtypes)
        // per thread per trip, in chunk order ctid, ctid+SST, ... (zero chunks add exactly nothing)
        float ss = 0.f;
        int i0 = ctid * 8;
        if (ctid >= SST) {
          i0 = p.K;
        } else if (reg16) {
          float v[8];
          unpack_act8(xr0, p.xdtype, v);
#pragma unroll
          for (int e = 0; e < 8; e++) ss = fmaf(v[e], v[e], ss);
          unpack_act8(xr1, p.xdtype, v);
#pragma unroll
          for (int e = 0; e < 8; e++) ss = fmaf(v[e], v[e], ss);
          i0 += 2 * SST * 8;
        }
        for (int i = i0; i < p.K; i += SST * 8) {
          float v[8];
          load_act8(p.x, (int64_t)col * p.K + i, p.xdtype, v);
#pragma unroll
          for (int k = 0; k < 8; k++) ss = fmaf(v[k], v[k], ss);
        }
        ss = warp_sum(ss);
        asm volatile("bar.sync 1, %0;" ::"n"(NCT));
        if (lane == 0 && warp < SSW) red[warp] = ss;
        asm volatile("bar.sync 1, %0;" ::"n"(NCT));
        float tot = 0.f;
#pragma unroll
        for (int i = 0; i < SSW; i++) tot += red[i];
        inv_rms = rsqrtf(tot / (float)p.K + p.eps);
      }
      if (tid == 0) MRS_STAMP(4);
      int4 *c0 = xq0 + (size_t)col * npos, *c1 = xq1 + (size_t)col * npos;
      float *ca = xa + (size_t)col * npos * Q::AUX;
      int it = 0;
#pragma unroll 1
      for (int ch = ctid; ch < nchunks_w; ch += NCT, it++) {
        const bool ok = ch < nchunks;
        const bool inreg = reg16 && (it == 0 || (it == 1 && NCW == SSW));
        float v[8];
        if (ok && live) {
          if (inreg) unpack_act8(sel_u4(it == 0, xr0, xr1), p.xdtype, v);
          else load_act8(p.x, (int64_t)col * p.K + ch * 8, p.xdtype, v);
          if (p.norm_w != nullptr) {
            float wv[8];
            if (inreg) unpack_act8(sel_u4(it == 0, nwr0, nwr1), p.xdtype, wv);
            else load_act8(p.norm_w, ch * 8, p.xdtype, wv);
#pragma unroll
            for (int i = 0; i < 8; i++) v[i] = round_act(v[i] * inv_rms * wv[i], p.xdtype);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 8; i++) v[i] = 0.f;
        }
        float am = 0.f;
#pragma unroll
        for (int i = 0; i < 8; i++) am = fmaxf(am, fabsf(v[i]));
        am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 1));
        am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, 2));
        float bsum = 0.f;
        if constexpr (Q::NEEDS_SUM) {
          // the reference's butterfly sum of the 32 block elements (i+16, i+8, then 4/2/1)
          float t[8];
#pragma unroll
          for (int i = 0; i < 8; i++) t[i] = v[i] + __shfl_xor_sync(0xffffffffu, v[i], 2);
#pragma unroll
          for (int i = 0; i < 8; i++) t[i] = t[i] + __shfl_xor_sync(0xffffffffu, t[i], 1);
#pragma unroll
          for (int m = 4; m > 0; m >>= 1) {
#pragma unroll
            for (int i = 0; i < m; i++) t[i] = t[i] + t[i + m];
          }
          bsum = __half2float(__float2half_rn(t[0]));
        }
        const float d = __fdividef(am, 127.0f);
        uint32_t wq[2] = {0u, 0u};
#pragma unroll
        for (int i = 0; i < 8; i++) {
          const int qi = (am == 0.0f) ? 0 : (int)(int8_t)roundf(__fdividef(v[i], d));
          wq[i >> 2] |= (uint32_t)(qi & 0xff) << (8 * (i & 3));
        }
        const int isum8 = __dp4a((int)wq[0], 0x01010101, __dp4a((int)wq[1], 0x01010101, 0));
        const int isum16 = isum8 + __shfl_xor_sync(0xffffffffu, isum8, 1);
        if (ok) {
          const int e0 = ch * 8;
          const int blk = e0 / Q::QK, e = e0 - blk * Q::QK;
          int c, hi, w8;
          Q::chunk_dest(e, c, hi, w8);
          const int pos = unit_to_pos<T, UPL>(blk, c);
          *((int2 *)((hi ? c1 : c0) + pos) + w8) = make_int2((int)wq[0], (int)wq[1]);
          Q::chunk_aux(e, __half2float(__float2half_rn(d)), bsum, isum8, isum16, ca + (size_t)pos * Q::AUX);
        }
      }
    }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(NCT));

  if (tid == 0) MRS_STAMP(6);
  // ----------------------------- main streaming loop -----------------------------
  int stage = 0, phase = 0;
  const int lblk = lane % G::NBL;   // block within the segment owned by this lane
  const int lsub = lane / G::NBL;   // chunk offset within the step
  for (int base = vr0; base < vr1; base += P) {
    // the two slots of this warp; invalid slots are clamped to the last valid row (their
    // results are computed on whatever the slot holds and discarded)
    bool valid[2];
    int mm[2], rr[2];
    uint32_t ph[2];  // byte phase (address mod 16) of the row start, per slot
#pragma unroll
    for (int r = 0; r < 2; r++) {
      int vrow = (p.mode == MODE_GLU) ? base + warp : base + 2 * warp + r;
      valid[r] = vrow < vr1;
      if (!valid[r]) vrow = vr1 - 1;
      resolve_row(p, vrow, r, mm[r], rr[r]);
      ph[r] = (uint32_t)((uintptr_t)(p.w[mm[r]] + (size_t)rr[r] * row_bytes) & 15);
    }
    float acc[2][NCOLS];
#pragma unroll
    for (int r = 0; r < 2; r++)
#pragma unroll
      for (int j = 0; j < NCOLS; j++) acc[r][j] = 0.f;

    for (int s = 0; s < nseg; s++) {
      mbar_wait(&full[stage], phase);
      if (tid == 0 && base == vr0 && s == 0) MRS_STAMP(7);
      const uint8_t *st = ring + (uint32_t)stage * G::STAGE_BYTES + (uint32_t)(2 * warp) * G::SLOT_BYTES;
      // phase of this segment's start: (row phase + s * SEG_BYTES) mod 16
      const uint32_t sp = (uint32_t)(s * G::SEG_BYTES) & 15u;
      const uint8_t *wp0 = st + ((ph[0] + sp) & 15u) + lblk * Q::BYTES;
      const uint8_t *wp1 = st + G::SLOT_BYTES + ((ph[1] + sp) & 15u) + lblk * Q::BYTES;
      const bool live = (s * G::SEG_BLOCKS + lblk) < nblocks;  // ragged last segment
#pragma unroll
      for (int ui = 0; ui < G::UPL; ui++) {
        const int c = (Q::UPB == 1) ? 0 : ui * G::CPS + lsub;
        const uint32_t boff = (Q::UPB == 1) ? (uint32_t)(ui * 32 * Q::BYTES) : 0u;
        const bool ulive = (Q::UPB == 1) ? (s * G::SEG_BLOCKS + ui * 32 + lblk) < nblocks : live;
        if (ulive && (valid[0] || valid[1])) {  // a warp whose two slots are both padding skips the math
          typename Q::W w0, w1;
          Q::template load<FAST>(wp0 + boff, c, w0);
          Q::template load<FAST>(wp1 + boff, c, w1);
          const int pos = s * G::SEG_UNITS + ui * 32 + lane;
#pragma unroll
          for (int j = 0; j < NCOLS; j++) {
            const int idx = j * npos + pos;
            const int4 q0 = xq0[idx], q1 = xq1[idx];
            const int xq[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
            float a[Q::AUX];
            if constexpr (Q::AUX == 4) {
              const float4 t = *(const float4 *)(xa + (size_t)idx * 4);
              a[0] = t.x; a[1] = t.y; a[2] = t.z; a[3] = t.w;
            } else if constexpr (Q::AUX == 2) {
              const float2 t = *(const float2 *)(xa + (size_t)idx * 2);
              a[0] = t.x; a[1] = t.y;
            } else if constexpr (Q::AUX == 8) {
              const float4 t0 = *(const float4 *)(xa + (size_t)idx * 8), t1 = *(const float4 *)(xa + (size_t)idx * 8 + 4);
              a[0] = t0.x; a[1] = t0.y; a[2] = t0.z; a[3] = t0.w; a[4] = t1.x; a[5] = t1.y; a[6] = t1.z; a[7] = t1.w;
            } else {
#pragma unroll
              for (int i = 0; i < Q::AUX; i++) a[i] = xa[(size_t)idx * Q::AUX + i];
            }
            acc[0][j] += Q::dot(w0, xq, a, c);
            acc[1][j] += Q::dot(w1, xq, a, c);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == nst) { stage = 0; phase ^= 1; }
    }

    if (tid == 0 && base + P >= vr1) MRS_STAMP(8);
    // ----------------------------- reduce + epilogue -----------------------------
#pragma unroll
    for (int r = 0; r < 2; r++)
#pragma unroll
      for (int j = 0; j < NCOLS; j++) acc[r][j] = warp_sum(acc[r][j]);

    if (lane == 0) {
      if (p.mode == MODE_GLU) {
        if (valid[0]) {
#pragma unroll
          for (int j = 0; j < NCOLS; j++) {
            if (j < p.ncols) {
              // cast gate and up to the output dtype first, activation in f32, product in
              // dtype — REF mmvq_gguf.cu:866-870
              const float g = round_act(acc[0][j], p.dst_dtype);
              const float up = round_act(acc[1][j], p.dst_dtype);
              const float act = round_act(glu_activation(g, p.activation), p.dst_dtype);
              if (p.dst_q8) qb[(((base - vr0) >> 5) & 1) * NCOLS * 32 + j * 32 + ((base - vr0) & 31) + warp] = round_act(act * up, p.dst_dtype);
              else store_act(p.dst[0], (int64_t)j * p.stride_col_dst + rr[0], act * up, p.dst_dtype);
            }
          }
        }
      } else {
#pragma unroll
        for (int r = 0; r < 2; r++) {
          if (!valid[r]) continue;
          const int nr = p.nrows[mm[r]];
          const int64_t cs = (p.mode == MODE_QKV) ? nr : p.stride_col_dst;
#pragma unroll
          for (int j = 0; j < NCOLS; j++) {
            if (j < p.ncols) {
              float v = acc[r][j];
              if (p.residual != nullptr) {
                // y materialised in dtype, then residual add rounded again (candle `+`)
                v = round_act(v, p.dst_dtype) + load_act(p.residual, (int64_t)j * cs + rr[r], p.dst_dtype);
              }
              store_act(p.dst[mm[r]], (int64_t)j * cs + rr[r], v, p.dst_dtype);
            }
          }
        }
      }
    }
    if (p.dst_q8 && ((base + P - vr0) & 31) == 0) {
      // the 32 rows of this group are in qb: warp 0 writes their block_q8_1 with the arithmetic of the standalone
      // quantiser (quantize_q8_1_kernel: lane = element, warp_max / warp_sum, fast divisions, half d and sum)
      asm volatile("bar.sync 1, %0;" ::"n"(NCT));
      if (warp == 0) {
        const float *src = qb + (((base - vr0) >> 5) & 1) * NCOLS * 32;
        const int blk = (base + P - 32) >> 5;
#pragma unroll
        for (int j = 0; j < NCOLS; j++) {
          if (j < p.ncols) {
            const float v = src[j * 32 + lane];
            const float amax = warp_max(fabsf(v));
            const float sum = warp_sum(v);
            const float d = __fdividef(amax, 127.0f);
            block_q8_1 *yb = (block_q8_1 *)p.dst[0] + (size_t)j * p.stride_col_dst + blk;
            yb->qs[lane] = (amax == 0.0f) ? (int8_t)0 : (int8_t)roundf(__fdividef(v, d));
            if (lane == 0) yb->ds = __halves2half2(__float2half_rn(d), __float2half_rn(sum));
          }
        }
      }
    }
  }
  if (tid == 0) {
    MRS_STAMP(9);
#ifdef MRS_TIMELINE
    if (p.dbg != nullptr) { p.dbg[(size_t)blockIdx.x * 16 + 15] = gridDim.x; p.dbg[(size_t)blockIdx.x * 16 + 14] = (unsigned long long)p.vrows << 32 | (unsigned)p.K; }
#endif
  }
}

template <int T, int NCOLS, bool FAST, int NCW, int UPL>
__global__ void __launch_bounds__((NCW + 1) * 32, NCOLS == 1 ? 3 : 2) mmvq_stream_kernel(const MmvqParams p) {
  mmvq_body<T, NCOLS, FAST, NCW, UPL>(p, (int)blockIdx.x, (int)gridDim.x);
}

// Two launches that read the same activations but hold different ggml types (Q4_K_M keeps attn_v in
// Q6_K on half the layers) as ONE grid: CTAs [0, g1) run the first program, the rest the second.
// Batch 1, aligned rows.
template <int T1, int T2>
__global__ void __launch_bounds__(9 * 32, 2) mmvq_dual_kernel(const MmvqParams pa, const MmvqParams pb, const int g1) {
  if ((int)blockIdx.x < g1) mmvq_body<T1, 1, true, 8>(pa, (int)blockIdx.x, g1);
  else mmvq_body<T2, 1, true, 8>(pb, (int)blockIdx.x - g1, (int)gridDim.x - g1);
}

// ---------------------------------------------------------------- host side
#ifdef MRS_TIMELINE
static unsigned long long *g_dbg = nullptr;
static int g_dbg_launch = 0, g_dbg_max = 0;
// dev build only: stamps of launch i land at buf[i * 320 * 16 ...]; returns launches recorded so far
extern "C" int mrs_mmvq_timeline(unsigned long long *buf, int max_launches) {
  const int n = g_dbg_launch;
  g_dbg = buf; g_dbg_max = max_launches; g_dbg_launch = 0;
  return n;
}
#endif
// per-device properties (a process may drive several GPUs: device-mapped layers, threaded TP)
constexpr int MAX_DEVICES = 64;
struct DevInfo { int num_sms, max_smem; };
static DevInfo g_dev[MAX_DEVICES] = {};
static int g_flags = 0;
static long long g_long_min_bytes = 128ll << 20;  // streams at least this long take 2x K segments
static int g_ctas_per_sm = 2;  // CTAs of ONE launch per SM; 1 leaves half an SM for the next launch (PDL overlap)

static const DevInfo &query_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= MAX_DEVICES) dev = 0;
  DevInfo &d = g_dev[dev];
  if (d.num_sms == 0) {
    int sms = 0, smem = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    d.max_smem = smem > 0 ? smem : 227 * 1024;
    d.num_sms = sms > 0 ? sms : 132;
  }
  return d;
}

// shared-memory plan of a launch: ring depth and bytes; two CTAs per SM by design, one CTA per SM
// with a deeper ring (and a one-wave grid) when two do not fit (long K x wide blocks)
template <int T, int UPL>
static bool plan8(const MmvqParams &p, int ncols, const DevInfo &d, int &nst, size_t &smem, int &ctas_per_sm) {
  using G = Geo<T, 8, UPL>;
  const int nblocks = p.K / QT<T>::QK;
  const int nseg = (nblocks + G::SEG_BLOCKS - 1) / G::SEG_BLOCKS;
  const int npos = nseg * G::SEG_UNITS;
  const size_t xbytes = 256 + (size_t)ncols * npos * G::XU_BYTES + (p.dst_q8 ? 2 * (size_t)ncols * 32 * 4 : 0) + 128;
  // batch 1 may run three CTAs per SM (72-register kernels): 24 consumer warps hide the shared-memory
  // and dp4a latencies better than 16
  ctas_per_sm = (ncols == 1) ? g_ctas_per_sm : (g_ctas_per_sm > 2 ? 2 : g_ctas_per_sm);
  size_t budget = (size_t)d.max_smem / (ctas_per_sm < 2 ? 2 : ctas_per_sm) - 1024;
  const size_t full = (size_t)d.max_smem - 1024;
  nst = MAX_STAGES;
  while (nst > 2 && xbytes + (size_t)nst * G::STAGE_BYTES > budget) nst--;
  smem = xbytes + (size_t)nst * G::STAGE_BYTES;
  if (smem > budget && ctas_per_sm == 3) {   // does not fit three times: two CTAs per SM
    ctas_per_sm = 2;
    budget = (size_t)d.max_smem / 2 - 1024;
    nst = MAX_STAGES;
    while (nst > 2 && xbytes + (size_t)nst * G::STAGE_BYTES > budget) nst--;
    smem = xbytes + (size_t)nst * G::STAGE_BYTES;
  }
  if (smem > budget) {
    ctas_per_sm = 1;
    while (nst < 4 && xbytes + (size_t)(nst + 1) * G::STAGE_BYTES <= full) nst++;
    smem = xbytes + (size_t)nst * G::STAGE_BYTES;
  }
  return smem <= (size_t)d.max_smem;
}

template <int T, int NCOLS, bool FAST, int UPL>
static cudaError_t launch_one(MmvqParams p, cudaStream_t stream) {
  constexpr int NCW = 8, SLOTS = 2 * NCW;
  const DevInfo &d = query_device();
  int nst, ctas_per_sm;
  size_t smem;
  if (!plan8<T, UPL>(p, NCOLS, d, nst, smem, ctas_per_sm)) return cudaErrorInvalidConfiguration;
  p.nstages = nst;
  p.flags = g_flags;
#ifdef MRS_TIMELINE
  p.dbg = (g_dbg != nullptr && g_dbg_launch < g_dbg_max) ? g_dbg + (size_t)(g_dbg_launch++) * 320 * 16 : nullptr;
#endif
  const int P = (p.mode == MODE_GLU) ? NCW : SLOTS;
  int grid = (p.vrows + P - 1) / P;
  if (p.dst_q8) grid = p.vrows / 32;  // whole 32-row groups per CTA
  const int max_grid = ctas_per_sm * d.num_sms;
  if (grid > max_grid) grid = max_grid;
  if (grid < 1) grid = 1;
  auto kern = mmvq_stream_kernel<T, NCOLS, FAST, NCW, UPL>;
  // the attribute is per device (context): set it on every launch — it is cheap, and a process-wide
  // "already set" flag would leave the second GPU of a multi-device process at the 48 KB default
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, d.max_smem);
  return launch_pdl(kern, dim3(grid), dim3((NCW + 1) * 32), smem, stream, p.pdl, p);
}

template <int T> static bool rows_aligned(const MmvqParams &p) {
  using Q = QT<T>;
  const int row_bytes = (p.K / Q::QK) * Q::BYTES;
  bool fast = (row_bytes % Q::WALIGN) == 0;
  for (int m = 0; m < 3; m++)
    if (p.w[m] != nullptr && ((uintptr_t)p.w[m] % Q::WALIGN) != 0) fast = false;
  return fast;
}

template <int T1, int T2>
static cudaError_t launch_dual(MmvqParams pa, MmvqParams pb, cudaStream_t stream) {
  const DevInfo &d = query_device();
  int nsa, nsb, ca, cb;
  size_t sma, smb;
  if (pa.ncols != 1 || pb.ncols != 1 || !rows_aligned<T1>(pa) || !rows_aligned<T2>(pb) ||
      !plan8<T1, QT<T1>::UPL>(pa, 1, d, nsa, sma, ca) || !plan8<T2, QT<T2>::UPL>(pb, 1, d, nsb, smb, cb) || ca < 2 || cb < 2)
    return cudaErrorNotSupported;
  if (ca != 2 || cb != 2) {   // the dual grid is planned for two CTAs per SM
    const int keep = g_ctas_per_sm; g_ctas_per_sm = 2;
    const bool ok = plan8<T1, QT<T1>::UPL>(pa, 1, d, nsa, sma, ca) && plan8<T2, QT<T2>::UPL>(pb, 1, d, nsb, smb, cb) && ca == 2 && cb == 2;
    g_ctas_per_sm = keep;
    if (!ok) return cudaErrorNotSupported;
  }
  pa.nstages = nsa; pb.nstages = nsb; pa.flags = pb.flags = g_flags;
#ifdef MRS_TIMELINE
  pa.dbg = (g_dbg != nullptr && g_dbg_launch < g_dbg_max) ? g_dbg + (size_t)(g_dbg_launch++) * 320 * 16 : nullptr;
  pb.dbg = pa.dbg;
#endif
  // one wave: 2 CTAs per SM in total, the second (smaller) program gets what it asks for first
  const int slots = 2 * d.num_sms;
  const int Pa = (pa.mode == MODE_GLU) ? 8 : 16, Pb = (pb.mode == MODE_GLU) ? 8 : 16;
  int ga = (pa.vrows + Pa - 1) / Pa, gb = (pb.vrows + Pb - 1) / Pb;
  if (ga < 1 || gb < 1) return cudaErrorNotSupported;
  if (ga + gb > slots) {
    if (gb > slots / 2) gb = slots / 2;
    if (ga > slots - gb) ga = slots - gb;
  }
  auto kern = mmvq_dual_kernel<T1, T2>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, d.max_smem);
  return launch_pdl(kern, dim3(ga + gb), dim3(9 * 32), sma > smb ? sma : smb, stream, pa.pdl, pa, pb, ga);
}

// supported type pairs of the two-type launch (the k-quant "M" recipes: attn_v one step up)
static cudaError_t mmvq_dispatch_dual(int t1, const MmvqParams &pa, int t2, const MmvqParams &pb, cudaStream_t stream) {
  if (t1 == MRS_Q4_K && t2 == MRS_Q6_K) return launch_dual<MRS_Q4_K, MRS_Q6_K>(pa, pb, stream);
  if (t1 == MRS_Q5_K && t2 == MRS_Q6_K) return launch_dual<MRS_Q5_K, MRS_Q6_K>(pa, pb, stream);
  if (t1 == MRS_Q4_K && t2 == MRS_Q5_K) return launch_dual<MRS_Q4_K, MRS_Q5_K>(pa, pb, stream);
  return cudaErrorNotSupported;
}

// long streams (lm_head-sized) take K segments twice as long: longer copies keep more bytes in flight per
// TMA issue; layer-sized matrices keep the short segments, whose pipeline bubbles are smaller.  Only the k-quants the "M" recipes put on `output`.
template <int T> struct HasLong { static constexpr bool value = (T == MRS_Q4_K || T == MRS_Q6_K); };

template <int T>
static cudaError_t launch_type(MmvqParams p, cudaStream_t stream) {
  using Q = QT<T>;
  // FAST: every block start is aligned to the type's natural alignment
  const bool fast = rows_aligned<T>(p);
  const int row_bytes = (p.K / Q::QK) * Q::BYTES;
  size_t wbytes = 0;  // weight bytes this launch streams
  for (int m = 0; m < 3; m++)
    if (p.w[m] != nullptr) wbytes += (size_t)p.nrows[m] * row_bytes;
  const int b = p.ncols;
#define MRS_DISPATCH(NC)                                                                          \
  do {                                                                                            \
    if constexpr (HasLong<T>::value) {                                                            \
      if (fast && NC == 1 && !(g_flags & 8) && wbytes >= (size_t)g_long_min_bytes)                \
        return launch_one<T, NC, true, 2 * Q::UPL>(p, stream);                                    \
    }                                                                                             \
    return fast ? launch_one<T, NC, true, Q::UPL>(p, stream) : launch_one<T, NC, false, Q::UPL>(p, stream); \
  } while (0)
  if (b == 1) { MRS_DISPATCH(1); }
  if (b == 2) { MRS_DISPATCH(2); }
  if (b <= 4) { MRS_DISPATCH(4); }
  MRS_DISPATCH(8);
#undef MRS_DISPATCH
}

cudaError_t mmvq_dispatch(int type, const MmvqParams &p, cudaStream_t stream) {
  if (p.ncols < 1 || p.ncols > 8) return cudaErrorInvalidValue;
  switch (type) {
  case MRS_Q4_0: return launch_type<MRS_Q4_0>(p, stream);
  case MRS_Q4_1: return launch_type<MRS_Q4_1>(p, stream);
  case MRS_Q5_0: return launch_type<MRS_Q5_0>(p, stream);
  case MRS_Q5_1: return launch_type<MRS_Q5_1>(p, stream);
  case MRS_Q8_0: return launch_type<MRS_Q8_0>(p, stream);
  case MRS_Q2_K: return launch_type<MRS_Q2_K>(p, stream);
  case MRS_Q3_K: return launch_type<MRS_Q3_K>(p, stream);
  case MRS_Q4_K: return launch_type<MRS_Q4_K>(p, stream);
  case MRS_Q5_K: return launch_type<MRS_Q5_K>(p, stream);
  case MRS_Q6_K: return launch_type<MRS_Q6_K>(p, stream);
  default: return cudaErrorInvalidValue;
  }
}

// ---------------------------------------------------------------- standalone Q8_1 quantiser
// REF: mmvq_gguf.cu:1220-1318 (kernel) and :1606-1641 (launchers): grid (ceil(kx_padded/256),
// rows), one warp per 32-element block, zero padding to kx_padded.
template <typename T>
__global__ void quantize_q8_1_kernel(const T *__restrict__ x, block_q8_1 *__restrict__ y, int kx, int kx_padded) {
  const int ix = blockDim.x * blockIdx.x + threadIdx.x;
  if (ix >= kx_padded) return;
  const int iy = blockIdx.y;
  const int64_t ip = (int64_t)iy * kx_padded + ix;
  const int ib = (int)(ip >> 5), iqs = (int)(ip & 31);
  const float xi = (ix < kx) ? (float)x[(int64_t)iy * kx + ix] : 0.0f;
  const float amax = warp_max(fabsf(xi));
  const float sum = warp_sum(xi);
  const float d = __fdividef(amax, 127.0f);
  const int8_t q = (amax == 0.0f) ? (int8_t)0 : (int8_t)roundf(__fdividef(xi, d));
  y[ib].qs[iqs] = q;
  if (iqs == 0) y[ib].ds = __halves2half2(__float2half_rn(d), __float2half_rn(sum));
}

}  // namespace mrs

using namespace mrs;

static int g_mrs_pdl = 0;  // PDL on reference-shaped launchers is opt-in (mrs_set_pdl)

extern "C" void mrs_set_pdl(int enabled) { g_mrs_pdl = enabled; }
// flags: bit 3 = never use the long-segment variant; bits 8.. = long-segment threshold in MiB
extern "C" void mrs_set_mmvq_flags(int f) { g_flags = f & 0xff; if (f >> 8) g_long_min_bytes = (long long)(f >> 8) << 20; }
extern "C" int mrs_mmvq_has_wide(void) { return 0; }
extern "C" void mrs_set_mmvq_ctas_per_sm(int n) { g_ctas_per_sm = n < 1 ? 1 : (n > 3 ? 3 : n); }

static inline void report(cudaError_t e, const char *what) {
  if (e != cudaSuccess) fprintf(stderr, "mrs_b200: %s failed: %s\n", what, cudaGetErrorString(e));
}

// ---- reference-shaped launchers ------------------------------------------------------------
#define MRS_Q8_1_LAUNCHER(tag, ctype)                                                          \
  extern "C" void launch_mmvq_gguf_quantize_q8_1_##tag(const void *x, void *vy, int kx,        \
                                                       int kx_padded, int num_rows,            \
                                                       void *stream) {                         \
    dim3 grid((kx_padded + 255) / 256, num_rows, 1);                                           \
    quantize_q8_1_kernel<ctype><<<grid, 256, 0, (cudaStream_t)stream>>>(                       \
        (const ctype *)x, (block_q8_1 *)vy, kx, kx_padded);                                    \
  }
MRS_Q8_1_LAUNCHER(bf16, __nv_bfloat16)
MRS_Q8_1_LAUNCHER(f16, __half)
MRS_Q8_1_LAUNCHER(f32, float)

static void run_plain(int type, int dt, const void *vx, const void *vy, void *dst, int ncols_x, int nrows_x,
                      int stride_col_y, int stride_col_dst, int b_size, void *stream) {
  if (b_size < 1 || b_size > 8) return;  // REF launcher: `default: break`
  MmvqParams p = {};
  p.w[0] = (const uint8_t *)vx; p.dst[0] = dst; p.nrows[0] = nrows_x;
  p.x = vy; p.xkind = X_Q8_1; p.K = ncols_x; p.stride_col_y = stride_col_y;
  p.stride_col_dst = stride_col_dst; p.ncols = b_size; p.mode = MODE_PLAIN; p.dst_dtype = dt;
  p.vrows = nrows_x; p.pdl = g_mrs_pdl;
  report(mmvq_dispatch(type, p, (cudaStream_t)stream), "mmvq plain");
}

static void run_glu(int type, int dt, const void *vg, const void *vu, const void *vy, void *dst, int ncols_x,
                    int nrows_x, int stride_col_y, int stride_col_dst, int b_size, int activation, void *stream) {
  if (b_size < 1 || b_size > 8) return;
  MmvqParams p = {};
  p.w[0] = (const uint8_t *)vg; p.w[1] = (const uint8_t *)vu; p.dst[0] = dst; p.nrows[0] = nrows_x; p.nrows[1] = nrows_x;
  p.x = vy; p.xkind = X_Q8_1; p.K = ncols_x; p.stride_col_y = stride_col_y;
  p.stride_col_dst = stride_col_dst; p.ncols = b_size; p.mode = MODE_GLU; p.activation = activation;
  p.dst_dtype = dt; p.vrows = nrows_x; p.pdl = g_mrs_pdl;
  report(mmvq_dispatch(type, p, (cudaStream_t)stream), "mmvq fused_glu");
}

static void run_qkv(int type, int dt, const void *vq, const void *vk, const void *vv, const void *vy, void *qd,
                    void *kd, void *vd, int ncols_x, int nq, int nk, int nv, int stride_col_y, int b_size,
                    void *stream) {
  if (b_size < 1 || b_size > 8) return;
  MmvqParams p = {};
  p.w[0] = (const uint8_t *)vq; p.w[1] = (const uint8_t *)vk; p.w[2] = (const uint8_t *)vv;
  p.dst[0] = qd; p.dst[1] = kd; p.dst[2] = vd; p.nrows[0] = nq; p.nrows[1] = nk; p.nrows[2] = nv;
  p.x = vy; p.xkind = X_Q8_1; p.K = ncols_x; p.stride_col_y = stride_col_y; p.ncols = b_size;
  p.mode = MODE_QKV; p.dst_dtype = dt; p.vrows = nq + nk + nv; p.pdl = g_mrs_pdl;
  report(mmvq_dispatch(type, p, (cudaStream_t)stream), "mmvq fused_qkv");
}

#define MRS_MMVQ_SET(tag, TYPE, dtag, DT)                                                              \
  extern "C" void launch_mmvq_gguf_##tag##_##dtag##_plain(const void *vx, const void *vy, void *dst,   \
      int ncols_x, int nrows_x, int stride_col_y, int stride_col_dst, int b_size, void *stream) {      \
    run_plain(TYPE, DT, vx, vy, dst, ncols_x, nrows_x, stride_col_y, stride_col_dst, b_size, stream);  \
  }                                                                                                    \
  extern "C" void launch_mmvq_gguf_##tag##_##dtag##_fused_glu(const void *vx_gate, const void *vx_up,  \
      const void *vy, void *dst, int ncols_x, int nrows_x, int stride_col_y, int stride_col_dst,       \
      int b_size, int activation, void *stream) {                                                      \
    run_glu(TYPE, DT, vx_gate, vx_up, vy, dst, ncols_x, nrows_x, stride_col_y, stride_col_dst, b_size, \
            activation, stream);                                                                       \
  }                                                                                                    \
  extern "C" void launch_mmvq_gguf_##tag##_##dtag##_fused_qkv(const void *vx_q, const void *vx_k,      \
      const void *vx_v, const void *vy, void *q_dst, void *k_dst, void *v_dst, int ncols_x,            \
      int nrows_q, int nrows_k, int nrows_v, int stride_col_y, int b_size, void *stream) {             \
    run_qkv(TYPE, DT, vx_q, vx_k, vx_v, vy, q_dst, k_dst, v_dst, ncols_x, nrows_q, nrows_k, nrows_v,   \
            stride_col_y, b_size, stream);                                                             \
  }
#define MRS_MMVQ_TYPE(tag, TYPE)            \
  MRS_MMVQ_SET(tag, TYPE, bf16, MRS_BF16)   \
  MRS_MMVQ_SET(tag, TYPE, f16, MRS_F16)     \
  MRS_MMVQ_SET(tag, TYPE, f32, MRS_F32)
MRS_MMVQ_TYPE(q4_0, MRS_Q4_0)
MRS_MMVQ_TYPE(q4_1, MRS_Q4_1)
MRS_MMVQ_TYPE(q5_0, MRS_Q5_0)
MRS_MMVQ_TYPE(q5_1, MRS_Q5_1)
MRS_MMVQ_TYPE(q8_0, MRS_Q8_0)
MRS_MMVQ_TYPE(q2_k, MRS_Q2_K)
MRS_MMVQ_TYPE(q3_k, MRS_Q3_K)
MRS_MMVQ_TYPE(q4_k, MRS_Q4_K)
MRS_MMVQ_TYPE(q5_k, MRS_Q5_K)
MRS_MMVQ_TYPE(q6_k, MRS_Q6_K)

// forward declaration (defined below in this file)
static cudaError_t mmvq_dispatch_dual_entry(int t1, const MmvqParams &pa, int t2, const MmvqParams &pb, cudaStream_t stream);

// ---- native fused entry points (same arithmetic, fewer launches) ------------------------
// y = W . q8_1( [rmsnorm_w *] x ) [+ residual]; mode bits 0-1: 0 plain, 1 fused GLU, 2 fused QKV.
// x is raw activations [b_size, K] of dtype `dt`; norm_w may be NULL; residual may be NULL.
// mode bit 2 (4): x is already block_q8_1 [b_size][K / 32] (norm_w must be NULL).
// mode bit 3 (8, fused GLU only, n0 % 32 == 0): dst0 receives the block_q8_1 [b_size][n0 / 32] form of the
// output instead of the output, bit for bit what launch_mmvq_gguf_quantize_q8_1_* makes of it.
extern "C" int mrs_mmvq_fused(int ggml_type, int mode, int dt, const void *w0, const void *w1, const void *w2,
                              const void *x, const void *norm_w, float eps, const void *residual,
                              void *dst0, void *dst1, void *dst2, int K, int n0, int n1, int n2,
                              int b_size, int activation, int pdl, void *stream) {
  const bool xq8 = (mode & 4) != 0, yq8 = (mode & 8) != 0;
  if (mode & ~15) return (int)cudaErrorInvalidValue;
  mode &= 3;
  if (mode == 3 || (xq8 && norm_w != nullptr) || (yq8 && (mode != MODE_GLU || n0 % 32 != 0))) return (int)cudaErrorInvalidValue;
  MmvqParams p = {};
  p.w[0] = (const uint8_t *)w0; p.w[1] = (const uint8_t *)w1; p.w[2] = (const uint8_t *)w2;
  p.dst[0] = dst0; p.dst[1] = dst1; p.dst[2] = dst2;
  p.nrows[0] = n0; p.nrows[1] = n1; p.nrows[2] = n2;
  p.x = x; p.xkind = xq8 ? X_Q8_1 : X_RAW; p.stride_col_y = K / 32; p.xdtype = dt; p.norm_w = norm_w; p.eps = eps;
  p.residual = residual; p.dst_q8 = yq8;
  p.K = K; p.stride_col_dst = yq8 ? n0 / 32 : n0; p.ncols = b_size; p.mode = mode; p.activation = activation;
  p.dst_dtype = dt; p.pdl = pdl;
  p.vrows = (mode == MODE_QKV) ? n0 + n1 + n2 : n0;
  return (int)mmvq_dispatch(ggml_type, p, (cudaStream_t)stream);
}

static cudaError_t mmvq_dispatch_dual_entry(int t1, const MmvqParams &pa, int t2, const MmvqParams &pb, cudaStream_t stream) {
  return mrs::mmvq_dispatch_dual(t1, pa, t2, pb, stream);
}

// QKV of one token block where attn_v has its own ggml type (k-quant "M" files): q∥k rows of type
// type_qk and the v rows of type type_v read the same [RMSNorm'd] activations; one grid when the
// pair is supported (batch 1, aligned rows), otherwise the two launches it replaces.  Arithmetic
// identical to mrs_mmvq_fused(mode 2, w2 = NULL) + mrs_mmvq_fused(mode 0) on wv.
extern "C" int mrs_mmvq_fused_qkv_mixed(int type_qk, int type_v, int dt, const void *wq, const void *wk, const void *wv,
                                        const void *x, const void *norm_w, float eps, void *q, void *k, void *v,
                                        int K, int nq, int nk, int nv, int b_size, int pdl, void *stream) {
  MmvqParams pa = {}, pb = {};
  pa.w[0] = (const uint8_t *)wq; pa.w[1] = (const uint8_t *)wk; pa.dst[0] = q; pa.dst[1] = k;
  pa.nrows[0] = nq; pa.nrows[1] = nk; pa.nrows[2] = 0;
  pa.x = x; pa.xkind = X_RAW; pa.xdtype = dt; pa.norm_w = norm_w; pa.eps = eps;
  pa.K = K; pa.stride_col_dst = nq; pa.ncols = b_size; pa.mode = MODE_QKV; pa.dst_dtype = dt; pa.pdl = pdl;
  pa.vrows = nq + nk;
  pb.w[0] = (const uint8_t *)wv; pb.dst[0] = v; pb.nrows[0] = nv;
  pb.x = x; pb.xkind = X_RAW; pb.xdtype = dt; pb.norm_w = norm_w; pb.eps = eps;
  pb.K = K; pb.stride_col_dst = nv; pb.ncols = b_size; pb.mode = MODE_PLAIN; pb.dst_dtype = dt; pb.pdl = pdl;
  pb.vrows = nv;
  cudaError_t e = (b_size == 1) ? mmvq_dispatch_dual_entry(type_qk, pa, type_v, pb, (cudaStream_t)stream) : cudaErrorNotSupported;
  if (e != cudaErrorNotSupported) return (int)e;
  e = mmvq_dispatch(type_qk, pa, (cudaStream_t)stream);
  if (e != cudaSuccess) return (int)e;
  return (int)mmvq_dispatch(type_v, pb, (cudaStream_t)stream);
}
