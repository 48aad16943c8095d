/* mrs_b200_quant.h — C ABI of the quantized-linear hot path (libmrs_b200.so).
 *
 * Every `launch_mmvq_gguf_*` symbol below has exactly the name, argument order and meaning of
 * the reference launcher it replaces, so mistralrs-quant's `extern "C"` block
 * (mistralrs-quant/src/gguf/ffi.rs, consumed by src/gguf/fast_mmvq.rs:116-157) links against
 * this library unchanged.  Contract (SURVEY §8b): raw device pointers already offset by the
 * tensor's start_offset; the caller owns all memory incl. the Q8_1 scratch; every call is
 * asynchronous on `stream`, allocation-free and CUDA-graph capturable; launchers return void and
 * do not check cudaGetLastError (like the reference); batch b_size outside 1..8 is a no-op.
 */
#ifndef MRS_B200_QUANT_H
#define MRS_B200_QUANT_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* Q8_1 activation quantiser — REF kernels/mmvq_gguf/mmvq_gguf.cu:1606-1641.
 * x [num_rows, kx] -> vy block_q8_1[num_rows][kx_padded/32] (36 B blocks, zero padded). */
void launch_mmvq_gguf_quantize_q8_1_bf16(const void *x, void *vy, int kx, int kx_padded, int num_rows, void *stream);
void launch_mmvq_gguf_quantize_q8_1_f16(const void *x, void *vy, int kx, int kx_padded, int num_rows, void *stream);
void launch_mmvq_gguf_quantize_q8_1_f32(const void *x, void *vy, int kx, int kx_padded, int num_rows, void *stream);

/* Decode GEMV, batch 1..8 — REF mmvq_gguf.cu:1322-1604 (launchers), fast_mmvq.rs:116-157.
 *  plain:      dst[b, row] = sum_k deq(vx[row, k]) * q8_1(vy)[b, k]
 *  fused_glu:  dst = dst_t(act(dst_t(gate.x))) * dst_t(up.x), activation = GluActivationType 0..4
 *  fused_qkv:  three projections sharing vy; outputs are dense [b, nrows_*]
 * vx*: ggml blocks [nrows, ncols_x/qk]; vy: block_q8_1 [b][stride_col_y]; dst [b][stride_col_dst]. */
#define MRS_MMVQ_DECL(q, t)                                                                                    \
  void launch_mmvq_gguf_##q##_##t##_plain(const void *vx, const void *vy, void *dst, int ncols_x, int nrows_x, \
                                          int stride_col_y, int stride_col_dst, int b_size, void *stream);     \
  void launch_mmvq_gguf_##q##_##t##_fused_glu(const void *vx_gate, const void *vx_up, const void *vy,          \
                                              void *dst, int ncols_x, int nrows_x, int stride_col_y,           \
                                              int stride_col_dst, int b_size, int activation, void *stream);   \
  void launch_mmvq_gguf_##q##_##t##_fused_qkv(const void *vx_q, const void *vx_k, const void *vx_v,            \
                                              const void *vy, void *q_dst, void *k_dst, void *v_dst,           \
                                              int ncols_x, int nrows_q, int nrows_k, int nrows_v,              \
                                              int stride_col_y, int b_size, void *stream);
#define MRS_MMVQ_DECL_T(q) MRS_MMVQ_DECL(q, bf16) MRS_MMVQ_DECL(q, f16) MRS_MMVQ_DECL(q, f32)
MRS_MMVQ_DECL_T(q4_0) MRS_MMVQ_DECL_T(q4_1) MRS_MMVQ_DECL_T(q5_0) MRS_MMVQ_DECL_T(q5_1) MRS_MMVQ_DECL_T(q8_0)
MRS_MMVQ_DECL_T(q2_k) MRS_MMVQ_DECL_T(q3_k) MRS_MMVQ_DECL_T(q4_k) MRS_MMVQ_DECL_T(q5_k) MRS_MMVQ_DECL_T(q6_k)

/* ---- native additions (not in the reference; see INTEGRATION.md for the Rust-side use) ---- */

/* Programmatic dependent launch for the reference-shaped launchers (default off). */
void mrs_set_pdl(int enabled);

/* Tuning/diagnostic switches of the decode GEMV.  bit 3 (value 8): never use the long-K-segment
 * variant; bits 8.. : smallest stream (MiB of weights per launch) that takes it (default 128).
 * Both variants compute the same integer dots, but the long segments hand a block's chunks to other
 * lanes, so an f32 output may differ in its last bit.  mrs_set_mmvq_ctas_per_sm: resident CTAs of one
 * launch per SM (1..3, default 2; 3 applies to batch 1). */
void mrs_set_mmvq_flags(int flags);
void mrs_set_mmvq_ctas_per_sm(int n);
int mrs_mmvq_has_wide(void);

/* One launch for [RMSNorm ->] Q8_1 -> GEMV [-> GLU | + residual]: replaces rms_norm +
 * launch_mmvq_gguf_quantize_q8_1_* + launch_mmvq_gguf_*  (+ the residual add).
 * mode 0 plain (w0), 1 fused GLU (w0 = gate, w1 = up), 2 fused QKV (w0,w1[,w2]; n2 may be 0).
 * x [b_size, K] of dtype dt (0 f16 / 1 bf16 / 2 f32), 16-byte aligned; norm_w / residual may be NULL.
 * mode | 4: x is already block_q8_1 [b_size][K / 32] (norm_w must be NULL) — what a mode | 8 launch wrote.
 * mode | 8 (fused GLU, n0 % 32 == 0): dst0 receives the block_q8_1 [b_size][n0 / 32] form of the output, byte for
 * byte what launch_mmvq_gguf_quantize_q8_1_* makes of the dt output; each CTA owns whole 32-row groups.
 * Results with mode | 4 equal those with the same activations raw, bit for bit.
 * ggml_type: GgmlDType code (2 q4_0 .. 14 q6_k).  Returns a cudaError_t. */
int mrs_mmvq_fused(int ggml_type, int mode, int dt, const void *w0, const void *w1, const void *w2, const void *x,
                   const void *norm_w, float eps, const void *residual, void *dst0, void *dst1, void *dst2, int K,
                   int n0, int n1, int n2, int b_size, int activation, int pdl, void *stream);

/* QKV projection where attn_v carries its own ggml type (llama.cpp's k-quant "M" recipes, e.g.
 * Q4_K_M: attn_q/attn_k Q4_K, attn_v Q6_K on half the layers): q||k rows and v rows read the same
 * [RMSNorm'd] activations.  One grid for the supported pairs (Q4_K+Q6_K, Q5_K+Q6_K, Q4_K+Q5_K) at
 * batch 1, otherwise the two launches it stands for; results identical to
 * mrs_mmvq_fused(mode 2, w2 = NULL) followed by mrs_mmvq_fused(mode 0) on wv.  Replaces the
 * reference's fused_qkv fallback to three plain launches (REF fast_mmvq.rs fused_qkv dtype check). */
int mrs_mmvq_fused_qkv_mixed(int type_qk, int type_v, int dt, const void *wq, const void *wk, const void *wv,
                             const void *x, const void *norm_w, float eps, void *q, void *k, void *v, int K, int nq,
                             int nk, int nv, int b_size, int pdl, void *stream);

/* Prefill GEMM (batch > 8) on the warpgroup tensor cores (wgmma): Y[M,N] = X[M,K] . W[N,K]^T, W in ggml blocks,
 * X/Y dtype 0 f16 / 1 bf16, K % 64 == 0.  Replaces launch_mmq_quantize_q8_1_* +
 * launch_mmq_gguf_<q> (REF fast_mmq.rs:102-185): no activation quantisation pass. */
int32_t mrs_mmq_gguf(int32_t ggml_type, const void *w, const void *x, void *y, int32_t M, int32_t N, int32_t K,
                     int32_t dtype, void *stream);
/* The ggml-block dequant GEMM (mrs_mmq_gguf's kernel and numerics) over n_mats = 1..3 matrices of one ggml type that
 * share X [M, K] (q|k|v, gate|up), in one launch: Y_m [M, rows[m]] = X . W_m^T, every W_m [rows[m], K] in its own
 * buffer, every Y_m row-major in its own buffer (host arrays w, rows, y of n_mats entries).
 * glu != 0: n_mats == 2, W_0 = gate and W_1 = up with rows[0] == rows[1]; only y[0] is written (y[1] may be NULL),
 * y[0] = T(silu(T(X . W_0^T))) * T(X . W_1^T) with the product rounded in T, as fused_glu.
 * pdl != 0: a link of a programmatic-dependent-launch chain — the weights stream before the upstream grid completes,
 * X is read and Y written after; the launch before it on `stream` must be a link or a plain kernel.
 * dtype 0 f16, 1 bf16; K % 64 == 0 (% 256 for k-quants); w, x 16-byte aligned, y 2-byte aligned.  pdl bit 0: PDL
 * link; bit 1 (value 2): never split K over a cluster, so every output row is the same for any M (a split, chosen from
 * M, sums the K partials in another order).  0 or a cudaError (cudaErrorInvalidValue for a bad type, count or shape,
 * cudaErrorMisalignedAddress).  Kernel: csrc/mmq_tc.cu. */
int32_t mrs_mmq_gguf_grouped(int32_t ggml_type, int32_t n_mats, const void **w, const int32_t *rows, void **y,
                             const void *x, int32_t M, int32_t K, int32_t dtype, int32_t glu, int32_t pdl, void *stream);

/* GPTQ / AWQ int4 linear from the raw checkpoint tensors (no Marlin repack) on the same
 * wgmma kernel: Y[M,N] f16 = X[M,K] f16 . W; GPTQ qweight [K/8,N] (w = (q-8)*s, optional
 * act-order g_idx [K]), AWQ qweight [K,N/8] + qzeros [K/g,N/8] (w = (q-z)*s); scales f16 [K/g,N].
 * Stands in for marlin_{gptq,awq}_4bit_f16 + {gptq,awq}_marlin_repack (REF gptq/marlin_ffi.rs:6-81). */
int32_t mrs_gptq_gemm(const void *x, const int32_t *qweight, const void *scales, const int32_t *qzeros,
                      const int32_t *g_idx, void *y, int32_t M, int32_t K, int32_t N, int32_t group_size,
                      int32_t is_awq, void *stream);

/* ---- GPTQ / AWQ through the reference's Marlin symbols — REF mistralrs-quant/src/gptq/marlin_ffi.rs:6-81
 * (same names, argument order and return convention: 0 ok, cudaError or -1 otherwise).  `weight` of
 * the matmuls is the buffer our own *_marlin_repack filled (opaque to the Rust side, same byte
 * count as the reference's [k/16, n*16/8] i32 result); `scales` arrive permuted by
 * marlin_permute_scales (gptq_cuda.rs:542-565) in the activation dtype; `zeros`: raw AWQ qzeros
 * (ignored for GPTQ: symmetric, w = (q-8)*s); `workspace` is unused (no global locks: split-K is
 * reduced inside a thread-block cluster).  Kernel: csrc/w4a16.cu, any m >= 1. */
int marlin_gptq_4bit_f16(const void *inputs, const int32_t *weight, const void *scales, const void *zeros,
                         const void *out, int m, int k, int n, const void *workspace, int groupsize, int64_t stream);
int marlin_gptq_4bit_bf16(const void *inputs, const int32_t *weight, const void *scales, const void *zeros,
                          const void *out, int m, int k, int n, const void *workspace, int groupsize, int64_t stream);
int marlin_awq_4bit_f16(const void *inputs, const int32_t *weight, const void *scales, const void *zeros,
                        const void *out, int m, int k, int n, const void *workspace, int groupsize, int64_t stream);
int marlin_awq_4bit_bf16(const void *inputs, const int32_t *weight, const void *scales, const void *zeros,
                         const void *out, int m, int k, int n, const void *workspace, int groupsize, int64_t stream);
/* weight: GPTQ [k/8, n] i32 / AWQ [k, n] i32 with n = out_dim/8; perm: argsort(g_idx) [k] i32 (GPTQ;
 * NULL = identity); bits must be 4 — REF kernels/marlin/marlin_repack.cu:255,473 */
void gptq_marlin_repack(const void *weight, const void *perm, const void *result, int k, int n, int bits, int64_t stream);
void awq_marlin_repack(const void *weight, const void *perm, const void *result, int k, int n, int bits, int64_t stream);

/* Native forms of the same kernel: explicit dtype / scale-column convention, and the dense
 * 16-bit linear (lm_head of GPTQ/AWQ checkpoints at decode batch; REF kernels/gemv/gemv.cu). */
int32_t mrs_w4a16_gemm(const void *x, const void *w_tiles, const void *scales, const int32_t *qzeros, void *y, int32_t M,
                       int32_t K, int32_t N, int32_t group, int32_t dtype, int32_t scale_perm, void *stream);
int32_t mrs_dense_linear(const void *x, const void *w, void *y, int32_t M, int32_t K, int32_t N, int32_t dtype, void *stream);

/* ---- packed-affine GGUF (the reference's opt-in `PackedAffine` path for batched GGUF linears) — same names, argument
 * order and return convention as REF mistralrs-quant/src/gguf/packed_affine.rs:1436-1509 (0 ok, -1 shape / format
 * outside the plan, else a cudaError).
 * repack: `format` = ggml type code (2,3,6,7,8,9,10..15: Q4_0 Q4_1 Q5_0 Q5_1 Q8_0 Q8_1 Q2_K..Q6_K Q8_K, :44-69);
 * `source` = ggml blocks [n, k/block]; writes payload (padded_n*k*bits/8 bytes: 4-bit for Q4_0/Q4_1/Q2_K/Q3_K/Q4_K,
 * else 8-bit), scales and offsets (k/group*padded_n 16-bit values each, group 16 for Q2_K/Q3_K/Q6_K else 32) such that
 * w = scale * q - offset; rows n..padded_n-1 are zero.  The layout inside the three buffers is this library's
 * (csrc/affine.cuh) and only its own marlin_affine_* reads it.
 * matmul: output [m, n] with n the PADDED width the buffers were packed for; `workspace` unused.  Kernel: the
 * wgmma dequant GEMM of csrc/mmq_tc.cu with csrc/affine.cuh's dequantiser; any m >= 1, k % 64 == 0. */
int32_t mrs_gguf_affine_repack_f16(int32_t format, const void *source, void *payload, void *scales, void *offsets,
                                   int32_t k, int32_t n, int32_t padded_n, uintptr_t stream);
int32_t mrs_gguf_affine_repack_bf16(int32_t format, const void *source, void *payload, void *scales, void *offsets,
                                    int32_t k, int32_t n, int32_t padded_n, uintptr_t stream);
int32_t marlin_affine_u4_f16(const void *input, const void *weight, void *scales, void *offsets, void *output, int32_t m,
                             int32_t k, int32_t n, int32_t group_size, void *workspace, int64_t stream);
int32_t marlin_affine_u4_bf16(const void *input, const void *weight, void *scales, void *offsets, void *output, int32_t m,
                              int32_t k, int32_t n, int32_t group_size, void *workspace, int64_t stream);
int32_t marlin_affine_u8_f16(const void *input, const void *weight, void *scales, void *offsets, void *output, int32_t m,
                             int32_t k, int32_t n, int32_t group_size, void *workspace, int64_t stream);
int32_t marlin_affine_u8_bf16(const void *input, const void *weight, void *scales, void *offsets, void *output, int32_t m,
                              int32_t k, int32_t n, int32_t group_size, void *workspace, int64_t stream);

#ifdef __cplusplus
}
#endif
#endif
