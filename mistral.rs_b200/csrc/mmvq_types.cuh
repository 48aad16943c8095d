// mmvq_types.cuh — per-quant-type "unit" arithmetic for the streaming decode GEMV.
//
// A *unit* is 32 weights of one ggml block chosen so that the weight bytes of the unit are
// one contiguous chunk of the block (Q4_K: one 16-byte chunk of qs = 16 low-nibble + 16
// high-nibble weights).  The activation side is pre-permuted into unit order in shared memory
// (x_elem), so every type reads its 32 int8 activations with two conflict-free LDS.128.
//
// Arithmetic is the reference's Q8_1 integer-dot scheme, type by type
// (REF: mistralrs-quant/kernels/mmvq_gguf/mmvq_gguf.cu:244-450 vec_dot_*_impl and
// :458-684 wrappers): integer dp4a dots per scale group, then f32 scale products.  The
// per-thread decomposition differs from the reference (one lane owns a whole 32-weight unit
// instead of 8/16 weights), so results agree up to f32 summation order.
#pragma once
#include "common.cuh"

namespace mrs {

// aligned or unaligned word fetch from the staged weight bytes in shared memory
template <int ALIGN, int N>
__device__ __forceinline__ void ld_words(const uint8_t *p, uint32_t (&out)[N]) {
  if constexpr (ALIGN >= 16 && N == 4) {
    const uint4 v = *(const uint4 *)p;
    out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
  } else if constexpr (ALIGN >= 8 && N == 2) {
    const uint2 v = *(const uint2 *)p;
    out[0] = v.x; out[1] = v.y;
  } else if constexpr (ALIGN >= 4) {
#pragma unroll
    for (int i = 0; i < N; i++) out[i] = ((const uint32_t *)p)[i];
  } else {
    lds_words_unaligned<N>(p, out);
  }
}

// unsigned-bytes x signed-bytes dot product (IDP.4A.U8.S8)
__device__ __forceinline__ int dp4a_us(uint32_t a, int b, int c) {
  int d;
  asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

template <int TYPE> struct QT;

// ------------------------------------------------------------------ Q4_K (144 B / 256)
// layout: half2 dm | scales[12] | qs[128]   REF mmvq_gguf.cu:171-177; dot :386-407,:586-618
template <> struct QT<MRS_Q4_K> {
  static constexpr int BYTES = 144, QK = 256, UPB = 8, AUX = 4, WALIGN = 16, UPL = 2;
  // unit c: chunk c of qs; j = c>>1 (64-wide group), h = c&1 (16-byte half)
  static constexpr bool NEEDS_SUM = false;
  // fused prologue: where the 8 activations at element e (multiple of 8) of a weight block go —
  // unit c, image half hi (0: xq0, 1: xq1), 8-byte half w8 — and what they add to the unit's aux
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) {
    const int r = e & 63;
    c = 2 * (e >> 6) + ((r >> 4) & 1); hi = r >> 5; w8 = (r >> 3) & 1;
  }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float, int, int isum16, float *a) {
    const int r = e & 63, hi = r >> 5;
    if (((r >> 3) & 1) == 0) { a[hi] = hi ? d * 0.0625f : d; a[2 + hi] = d * (float)isum16; }
  }
  __device__ static __forceinline__ int x_elem(int c, int w) {
    const int j = c >> 1, h = c & 1;
    return 64 * j + 16 * h + (w < 4 ? 4 * w : 32 + 4 * (w - 4));
  }
  // aux: d8 of the two q8 blocks and d8 * (sum of the 16 activations) for the min term
  template <typename Y> __device__ static __forceinline__ void aux(const int *q, int c, Y y, float *a) {
    const int j = c >> 1;
    a[0] = y.d(2 * j); a[1] = y.d(2 * j + 1);
    const int s0 = __dp4a(q[0], 0x01010101, __dp4a(q[1], 0x01010101, __dp4a(q[2], 0x01010101, __dp4a(q[3], 0x01010101, 0))));
    const int s1 = __dp4a(q[4], 0x01010101, __dp4a(q[5], 0x01010101, __dp4a(q[6], 0x01010101, __dp4a(q[7], 0x01010101, 0))));
    a[2] = a[0] * (float)s0; a[3] = a[1] * (float)s1;
    a[1] *= 0.0625f;  // the dot leaves the high nibbles in place (x16), exact power of two
  }
  struct W { uint32_t q[4]; uint32_t h[4]; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int c, W &w) {
    ld_words<(AL ? 16 : 1), 4>(blk, w.h);
    ld_words<(AL ? 16 : 1), 4>(blk + 16 + 16 * c, w.q);
  }
  // 6-bit scale/min of sub-blocks 2j (->lo) and 2j+1 (->hi): REF :598-609
  __device__ static __forceinline__ void scales(const uint32_t *h, int j, int &sc_lo, int &sc_hi, int &m_lo, int &m_hi) {
    // scales as six uint16: s16[k] = (h[1 + k/2] >> 16*(k&1)) & 0xffff
    auto s16 = [&](int k) -> uint32_t {
      const uint32_t wsel = (k < 2) ? h[1] : ((k < 4) ? h[2] : h[3]);
      return (wsel >> (16 * (k & 1))) & 0xffffu;
    };
    uint32_t a0, a1;
    if (j < 2) {
      a0 = s16(j) & 0x3f3f; a1 = s16(j + 2) & 0x3f3f;
    } else {
      a0 = (s16(j + 2) & 0x0f0f) | ((s16(j - 2) & 0xc0c0) >> 2);
      a1 = ((s16(j + 2) >> 4) & 0x0f0f) | ((s16(j) & 0xc0c0) >> 2);
    }
    sc_lo = a0 & 0xff; sc_hi = a0 >> 8; m_lo = a1 & 0xff; m_hi = a1 >> 8;
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int c) {
    int sc_lo, sc_hi, m_lo, m_hi;
    scales(w.h, c >> 1, sc_lo, sc_hi, m_lo, m_hi);
    int dlo = 0, dhi = 0;  // dhi accumulates 16x the high-nibble dot (nibbles left in place)
#pragma unroll
    for (int i = 0; i < 4; i++) {
      dlo = __dp4a((int)(w.q[i] & 0x0F0F0F0Fu), xq[i], dlo);
      dhi = dp4a_us(w.q[i] & 0xF0F0F0F0u, xq[4 + i], dhi);
    }
    const float2 dm = __half22float2(*(const __half2 *)&w.h[0]);
    const float sd = xa[0] * (float)(dlo * sc_lo) + xa[1] * (float)(dhi * sc_hi);
    const float sm = xa[2] * (float)m_lo + xa[3] * (float)m_hi;
    return dm.x * sd - dm.y * sm;
  }
};

// ------------------------------------------------------------------ Q5_K (176 B / 256)
// layout: half2 dm | scales[12] | qh[32] | qs[128]  REF :179-186; dot :409-432,:620-660
template <> struct QT<MRS_Q5_K> {
  static constexpr int BYTES = 176, QK = 256, UPB = 8, AUX = 4, WALIGN = 16, UPL = 4;
  static constexpr bool NEEDS_SUM = false;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) { QT<MRS_Q4_K>::chunk_dest(e, c, hi, w8); }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float, int, int isum16, float *a) {
    const int r = e & 63, hi = r >> 5;
    if (((r >> 3) & 1) == 0) { a[hi] = d; a[2 + hi] = d * (float)isum16; }
  }
  __device__ static __forceinline__ int x_elem(int c, int w) { return QT<MRS_Q4_K>::x_elem(c, w); }
  template <typename Y> __device__ static __forceinline__ void aux(const int *q, int c, Y y, float *a) {
    QT<MRS_Q4_K>::aux(q, c, y, a);
    a[1] *= 16.0f;  // undo Q4_K's in-place-nibble folding
  }
  struct W { uint32_t q[4]; uint32_t qh[4]; uint32_t h[4]; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int c, W &w) {
    ld_words<(AL ? 16 : 1), 4>(blk, w.h);
    ld_words<(AL ? 16 : 1), 4>(blk + 16 + 16 * (c & 1), w.qh);  // qh[l], l in 16h..16h+15
    ld_words<(AL ? 16 : 1), 4>(blk + 48 + 16 * c, w.q);
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int c) {
    int sc_lo, sc_hi, m_lo, m_hi;
    const int j = c >> 1;
    QT<MRS_Q4_K>::scales(w.h, j, sc_lo, sc_hi, m_lo, m_hi);
    int dlo = 0, dhi = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint32_t vh = w.qh[i] >> (2 * j);
      const uint32_t lo = (w.q[i] & 0x0F0F0F0Fu) | ((vh << 4) & 0x10101010u);
      const uint32_t hi = ((w.q[i] >> 4) & 0x0F0F0F0Fu) | ((vh << 3) & 0x10101010u);
      dlo = __dp4a((int)lo, xq[i], dlo);
      dhi = __dp4a((int)hi, xq[4 + i], dhi);
    }
    const float2 dm = __half22float2(*(const __half2 *)&w.h[0]);
    const float sd = xa[0] * (float)(dlo * sc_lo) + xa[1] * (float)(dhi * sc_hi);
    const float sm = xa[2] * (float)m_lo + xa[3] * (float)m_hi;
    return dm.x * sd - dm.y * sm;
  }
};

// ------------------------------------------------------------------ Q6_K (210 B / 256)
// layout: ql[128] | qh[64] | int8 scales[16] | half d   REF :188-195; dot :434-450,:662-684
// unit c = 4n + t: ql chunk c; low nibbles -> elements 128n + 32(t>>1) + 16(t&1) + i,
// high nibbles -> +64; qh[32n + 16(t&1) + i] bits 2(t>>1) (+4 for the high group).
template <> struct QT<MRS_Q6_K> {
  static constexpr int BYTES = 210, QK = 256, UPB = 8, AUX = 2, WALIGN = 2, UPL = 2;
  static constexpr bool NEEDS_SUM = false;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) {
    const int r = e & 127, r2 = r & 63;
    c = 4 * (e >> 7) + 2 * (r2 >> 5) + ((r2 >> 4) & 1); hi = r >> 6; w8 = (r2 >> 3) & 1;
  }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float, int, int, float *a) {
    const int r = e & 127;
    if (((r >> 3) & 1) == 0) a[r >> 6] = d;
  }
  __device__ static __forceinline__ int x_elem(int c, int w) {
    const int n = c >> 2, t = c & 3;
    const int lo = 128 * n + 32 * (t >> 1) + 16 * (t & 1);
    return w < 4 ? lo + 4 * w : lo + 64 + 4 * (w - 4);
  }
  template <typename Y> __device__ static __forceinline__ void aux(const int *, int c, Y y, float *a) {
    const int n = c >> 2, t = c & 3;
    a[0] = y.d(4 * n + (t >> 1));
    a[1] = y.d(4 * n + (t >> 1) + 2);
  }
  struct W { uint32_t ql[4]; uint32_t qh[4]; int sc_a, sc_b; float d; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int c, W &w) {
    const int n = c >> 2, t = c & 3;
    lds_words_unaligned<4>(blk + 16 * c, w.ql);
    lds_words_unaligned<4>(blk + 128 + 32 * n + 16 * (t & 1), w.qh);
    const int8_t *sc = (const int8_t *)(blk + 192);
    const int is = 8 * n + 2 * (t >> 1) + (t & 1);
    w.sc_a = sc[is]; w.sc_b = sc[is + 4];
    w.d = half_bits_to_float(lds_u16<AL>(blk + 208));
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int c) {
    const int sh = 2 * ((c & 3) >> 1);
    int da = 0, db = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint32_t vh = w.qh[i] >> sh;
      const uint32_t a = (w.ql[i] & 0x0F0F0F0Fu) | ((vh << 4) & 0x30303030u);
      const uint32_t b = ((w.ql[i] >> 4) & 0x0F0F0F0Fu) | (vh & 0x30303030u);
      da = __dp4a((int)__vsub4(a, 0x20202020u), xq[i], da);
      db = __dp4a((int)__vsub4(b, 0x20202020u), xq[4 + i], db);
    }
    return w.d * (xa[0] * (float)(da * w.sc_a) + xa[1] * (float)(db * w.sc_b));
  }
};

// ------------------------------------------------------------------ Q2_K (84 B / 256)
// layout: scales[16] | qs[64] | half2 dm   REF :154-160; dot :348-366,:534-552
// unit c = 4n + g: qs[32n + 8g .. +8); byte l holds elements 128n + 32j + 8g + l, j=0..3
template <> struct QT<MRS_Q2_K> {
  static constexpr int BYTES = 84, QK = 256, UPB = 8, AUX = 8, WALIGN = 4, UPL = 8;
  static constexpr bool NEEDS_SUM = false;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) {
    const int r = e & 127, jj = r >> 5;
    c = 4 * (e >> 7) + ((r & 31) >> 3); hi = jj >> 1; w8 = jj & 1;
  }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float, int isum8, int, float *a) {
    const int jj = (e & 127) >> 5;
    a[jj] = d; a[4 + jj] = d * (float)isum8;
  }
  __device__ static __forceinline__ int x_elem(int c, int w) {
    const int n = c >> 2, g = c & 3;
    return 128 * n + 32 * (w >> 1) + 8 * g + 4 * (w & 1);
  }
  template <typename Y> __device__ static __forceinline__ void aux(const int *q, int c, Y y, float *a) {
    const int n = c >> 2;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      a[j] = y.d(4 * n + j);
      a[4 + j] = a[j] * (float)__dp4a(q[2 * j], 0x01010101, __dp4a(q[2 * j + 1], 0x01010101, 0));
    }
  }
  struct W { uint32_t q[2]; uint32_t sc; uint32_t dm; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int c, W &w) {
    const int n = c >> 2, g = c & 3;
    ld_words<(AL ? 4 : 1), 2>(blk + 16 + 32 * n + 8 * g, w.q);
    // scale bytes 8n + 2j + (g>>1), j = 0..3 -> packed into one word
    const uint8_t *s = blk + 8 * n + (g >> 1);
    w.sc = (uint32_t)s[0] | ((uint32_t)s[2] << 8) | ((uint32_t)s[4] << 16) | ((uint32_t)s[6] << 24);
    uint32_t t[1];
    ld_words<(AL ? 4 : 1), 1>(blk + 80, t);
    w.dm = t[0];
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int) {
    float sd = 0.f, sm = 0.f;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int sc = (w.sc >> (8 * j)) & 0xff;
      const int v0 = (int)((w.q[0] >> (2 * j)) & 0x03030303u);
      const int v1 = (int)((w.q[1] >> (2 * j)) & 0x03030303u);
      const int idot = __dp4a(v0, xq[2 * j], __dp4a(v1, xq[2 * j + 1], 0));
      sd += xa[j] * (float)(idot * (sc & 0xF));
      sm += xa[4 + j] * (float)(sc >> 4);
    }
    const float2 dm = __half22float2(*(const __half2 *)&w.dm);
    return dm.x * sd - dm.y * sm;
  }
};

// ------------------------------------------------------------------ Q3_K (110 B / 256)
// layout: hmask[32] | qs[64] | scales[12] | half d   REF :162-169; dot :368-384,:554-584
template <> struct QT<MRS_Q3_K> {
  static constexpr int BYTES = 110, QK = 256, UPB = 8, AUX = 4, WALIGN = 2, UPL = 8;
  static constexpr bool NEEDS_SUM = false;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) { QT<MRS_Q2_K>::chunk_dest(e, c, hi, w8); }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float, int, int, float *a) { a[(e & 127) >> 5] = d; }
  __device__ static __forceinline__ int x_elem(int c, int w) { return QT<MRS_Q2_K>::x_elem(c, w); }
  template <typename Y> __device__ static __forceinline__ void aux(const int *, int c, Y y, float *a) {
    const int n = c >> 2;
#pragma unroll
    for (int j = 0; j < 4; j++) a[j] = y.d(4 * n + j);
  }
  struct W { uint32_t q[2]; uint32_t hm[2]; int sc[4]; float d; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int c, W &w) {
    const int n = c >> 2, g = c & 3;
    lds_words_unaligned<2>(blk + 32 + 32 * n + 8 * g, w.q);
    lds_words_unaligned<2>(blk + 8 * g, w.hm);
    const uint8_t *s = blk + 96;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int is = 8 * n + 2 * j + (g >> 1);
      const int low = (s[is & 7] >> (4 * (is >> 3))) & 0xF;
      const int high = (s[8 + (is & 3)] >> (2 * (is >> 2))) & 3;
      w.sc[j] = (low | (high << 4)) - 32;
    }
    w.d = half_bits_to_float(lds_u16<AL>(blk + 108));
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int c) {
    const int n = c >> 2;
    float sd = 0.f;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      // hmask bit (4n + j) set => no -4 offset   (REF :374-376: vih from ~hmask)
      const uint32_t h0 = (~w.hm[0] >> (4 * n + j)) & 0x01010101u;
      const uint32_t h1 = (~w.hm[1] >> (4 * n + j)) & 0x01010101u;
      const uint32_t v0 = __vsubss4((w.q[0] >> (2 * j)) & 0x03030303u, h0 << 2);
      const uint32_t v1 = __vsubss4((w.q[1] >> (2 * j)) & 0x03030303u, h1 << 2);
      const int idot = __dp4a((int)v0, xq[2 * j], __dp4a((int)v1, xq[2 * j + 1], 0));
      sd += xa[j] * (float)(idot * w.sc[j]);
    }
    return w.d * sd;
  }
};

// ------------------------------------------------------------------ 32-wide types: unit == block
template <int AUXN> struct X32 {
  __device__ static __forceinline__ int x_elem(int, int w) { return 4 * w; }
};

// Q8_0 (34 B): half d | int8 qs[32]   REF :136-141; dot :336-346
template <> struct QT<MRS_Q8_0> {
  static constexpr int BYTES = 34, QK = 32, UPB = 1, AUX = 1, WALIGN = 2, UPL = 2;
  static constexpr bool NEEDS_SUM = false;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) { c = 0; hi = e >> 4; w8 = (e >> 3) & 1; }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float sm, int, int, float *a) {
    if (e == 0) { a[0] = d; }
  }
  __device__ static __forceinline__ int x_elem(int, int w) { return 4 * w; }
  template <typename Y> __device__ static __forceinline__ void aux(const int *, int, Y y, float *a) { a[0] = y.d(0); }
  struct W { uint32_t q[8]; float d; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int, W &w) {
    w.d = half_bits_to_float(lds_u16<AL>(blk));
    lds_words_unaligned<8>(blk + 2, w.q);
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int) {
    int s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) s = __dp4a((int)w.q[i], xq[i], s);
    return (float)s * w.d * xa[0];
  }
};

// Q4_0 (18 B): half d | qs[16]   REF :197-202; dot :244-258
template <> struct QT<MRS_Q4_0> {
  static constexpr int BYTES = 18, QK = 32, UPB = 1, AUX = 2, WALIGN = 2, UPL = 4;
  static constexpr bool NEEDS_SUM = true;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) { c = 0; hi = e >> 4; w8 = (e >> 3) & 1; }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float sm, int, int, float *a) {
    if (e == 0) { a[0] = d; a[1] = sm; }
  }
  __device__ static __forceinline__ int x_elem(int, int w) { return 4 * w; }
  template <typename Y> __device__ static __forceinline__ void aux(const int *, int, Y y, float *a) { a[0] = y.d(0); a[1] = y.s(0); }
  struct W { uint32_t q[4]; float d; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int, W &w) {
    w.d = half_bits_to_float(lds_u16<AL>(blk));
    lds_words_unaligned<4>(blk + 2, w.q);
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int) {
    int s = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      s = __dp4a((int)(w.q[i] & 0x0F0F0F0Fu), xq[i], s);
      s = __dp4a((int)((w.q[i] >> 4) & 0x0F0F0F0Fu), xq[4 + i], s);
    }
    return w.d * ((float)s * xa[0] - 8.0f * xa[1]);
  }
};

// Q4_1 (20 B): half2 dm | qs[16]   REF :204-209; dot :260-277
template <> struct QT<MRS_Q4_1> {
  static constexpr int BYTES = 20, QK = 32, UPB = 1, AUX = 2, WALIGN = 4, UPL = 4;
  static constexpr bool NEEDS_SUM = true;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) { c = 0; hi = e >> 4; w8 = (e >> 3) & 1; }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float sm, int, int, float *a) {
    if (e == 0) { a[0] = d; a[1] = sm; }
  }
  __device__ static __forceinline__ int x_elem(int, int w) { return 4 * w; }
  template <typename Y> __device__ static __forceinline__ void aux(const int *, int, Y y, float *a) { a[0] = y.d(0); a[1] = y.s(0); }
  struct W { uint32_t q[4]; uint32_t dm; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int, W &w) {
    uint32_t t[5];
    ld_words<(AL ? 4 : 1), 5>(blk, t);
    w.dm = t[0];
#pragma unroll
    for (int i = 0; i < 4; i++) w.q[i] = t[1 + i];
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int) {
    int s = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      s = __dp4a((int)(w.q[i] & 0x0F0F0F0Fu), xq[i], s);
      s = __dp4a((int)((w.q[i] >> 4) & 0x0F0F0F0Fu), xq[4 + i], s);
    }
    const float2 dm = __half22float2(*(const __half2 *)&w.dm);
    return (float)s * (dm.x * xa[0]) + dm.y * xa[1];
  }
};

// spread 4 consecutive high bits onto bit 4 of each byte — REF :286-300
__device__ __forceinline__ uint32_t q5_hi_lo(uint32_t vh) {
  return ((vh << 4) & 0x00000010u) | ((vh << 11) & 0x00001000u) | ((vh << 18) & 0x00100000u) |
         ((vh << 25) & 0x10000000u);
}
__device__ __forceinline__ uint32_t q5_hi_hi(uint32_t vh) {
  return ((vh >> 12) & 0x00000010u) | ((vh >> 5) & 0x00001000u) | ((vh << 2) & 0x00100000u) |
         ((vh << 9) & 0x10000000u);
}

// Q5_0 (22 B): half d | qh[4] | qs[16]   REF :211-217; dot :279-306
template <> struct QT<MRS_Q5_0> {
  static constexpr int BYTES = 22, QK = 32, UPB = 1, AUX = 2, WALIGN = 2, UPL = 4;
  static constexpr bool NEEDS_SUM = true;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) { c = 0; hi = e >> 4; w8 = (e >> 3) & 1; }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float sm, int, int, float *a) {
    if (e == 0) { a[0] = d; a[1] = sm; }
  }
  __device__ static __forceinline__ int x_elem(int, int w) { return 4 * w; }
  template <typename Y> __device__ static __forceinline__ void aux(const int *, int, Y y, float *a) { a[0] = y.d(0); a[1] = y.s(0); }
  struct W { uint32_t q[4]; uint32_t qh; float d; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int, W &w) {
    w.d = half_bits_to_float(lds_u16<AL>(blk));
    uint32_t t[5];
    lds_words_unaligned<5>(blk + 2, t);
    w.qh = t[0];
#pragma unroll
    for (int i = 0; i < 4; i++) w.q[i] = t[1 + i];
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int) {
    int s = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint32_t vh = w.qh >> (4 * i);
      s = __dp4a((int)((w.q[i] & 0x0F0F0F0Fu) | q5_hi_lo(vh)), xq[i], s);
      s = __dp4a((int)(((w.q[i] >> 4) & 0x0F0F0F0Fu) | q5_hi_hi(vh)), xq[4 + i], s);
    }
    return w.d * ((float)s * xa[0] - 16.0f * xa[1]);
  }
};

// Q5_1 (24 B): half2 dm | qh[4] | qs[16]   REF :219-225; dot :308-334
template <> struct QT<MRS_Q5_1> {
  static constexpr int BYTES = 24, QK = 32, UPB = 1, AUX = 2, WALIGN = 8, UPL = 4;
  static constexpr bool NEEDS_SUM = true;
  __device__ static __forceinline__ void chunk_dest(int e, int &c, int &hi, int &w8) { c = 0; hi = e >> 4; w8 = (e >> 3) & 1; }
  __device__ static __forceinline__ void chunk_aux(int e, float d, float sm, int, int, float *a) {
    if (e == 0) { a[0] = d; a[1] = sm; }
  }
  __device__ static __forceinline__ int x_elem(int, int w) { return 4 * w; }
  template <typename Y> __device__ static __forceinline__ void aux(const int *, int, Y y, float *a) { a[0] = y.d(0); a[1] = y.s(0); }
  struct W { uint32_t q[4]; uint32_t qh; uint32_t dm; };
  template <bool AL> __device__ static __forceinline__ void load(const uint8_t *blk, int, W &w) {
    uint32_t t[6];
    ld_words<(AL ? 4 : 1), 6>(blk, t);
    w.dm = t[0]; w.qh = t[1];
#pragma unroll
    for (int i = 0; i < 4; i++) w.q[i] = t[2 + i];
  }
  __device__ static __forceinline__ float dot(const W &w, const int *xq, const float *xa, int) {
    int s = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint32_t vh = w.qh >> (4 * i);
      s = __dp4a((int)((w.q[i] & 0x0F0F0F0Fu) | q5_hi_lo(vh)), xq[i], s);
      s = __dp4a((int)(((w.q[i] >> 4) & 0x0F0F0F0Fu) | q5_hi_hi(vh)), xq[4 + i], s);
    }
    const float2 dm = __half22float2(*(const __half2 *)&w.dm);
    return (float)s * (dm.x * xa[0]) + dm.y * xa[1];
  }
};

}  // namespace mrs
