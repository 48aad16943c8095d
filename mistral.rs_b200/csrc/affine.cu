// affine.cu — device repack of ggml block tensors into the packed-affine form (a5): unsigned 4- or 8-bit payload plus a
// 16-bit scale and offset per 16 / 32 weights, w = scale * q - offset.  Behind the reference's own symbols
// `mrs_gguf_affine_repack_{f16,bf16}` (REF mistralrs-quant/src/gguf/packed_affine.rs:1436-1457 declarations, :526-585
// call site: source blocks [n, k/block] -> payload padded_n*k*bits/8 bytes, scales / offsets k/group*padded_n values).
// The matching GEMM entry points `marlin_affine_{u4,u8}_{f16,bf16}` live in mmq_tc.cu (same wgmma kernel as the
// checkpoint-layout int4 GEMM, with affine.cuh's dequantiser).
//
// One thread per (row, 32-weight segment); the per-format arithmetic is affine.cuh, which the CPU suite runs on the
// host against the oracle.  HBM-bound, run once per weight at load time: bytes = source + payload + metadata.
// Layout of the three outputs: see affine.cuh (row-major per output channel; padding rows n..padded_n-1 are zero weights).
#include "affine.cuh"
#include "common.cuh"

namespace mrs {

__global__ void __launch_bounds__(256)
affine_repack_kernel(int format, affine::Spec sp, const uint8_t *__restrict__ src, uint8_t *__restrict__ payload, uint16_t *__restrict__ scales,
                     uint16_t *__restrict__ offsets, int k, int n, int padded_n, int bf16) {
  const int segs = k / 32;
  const size_t row_bytes = (size_t)(k / sp.block_elems) * sp.block_bytes, prow = (size_t)k * sp.bits / 8, gpr = (size_t)(k / sp.group);
  const long long total = (long long)padded_n * segs;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / segs), seg = (int)(i % segs);
    affine::repack_segment(format, sp, r < n ? src + (size_t)r * row_bytes : nullptr, seg, payload + (size_t)r * prow, scales + (size_t)r * gpr,
                           offsets + (size_t)r * gpr, bf16 != 0);
  }
}

static int32_t affine_repack(int format, const void *source, void *payload, void *scales, void *offsets, int k, int n, int padded_n, int bf16,
                             cudaStream_t st) {
  affine::Spec sp;
  if (!affine::spec_for(format, sp)) return -1;
  if (k <= 0 || n <= 0 || padded_n < n || k % sp.block_elems != 0 || k % 64 != 0) return -1;
  if (source == nullptr || payload == nullptr || scales == nullptr || offsets == nullptr) return -1;
  const long long total = (long long)padded_n * (k / 32);
  const int blocks = (int)((total + 255) / 256 < 132 * 8 ? (total + 255) / 256 : 132 * 8);   // grid-stride over at most 8 CTAs per SM (132 SMs)
  affine_repack_kernel<<<blocks, 256, 0, st>>>(format, sp, (const uint8_t *)source, (uint8_t *)payload, (uint16_t *)scales, (uint16_t *)offsets, k,
                                                n, padded_n, bf16);
  return (int32_t)cudaGetLastError();
}

}  // namespace mrs

// REF packed_affine.rs:1436-1457.  0 on success, -1 for a format / shape outside the plan, else the cudaError of the launch.
extern "C" int32_t mrs_gguf_affine_repack_f16(int32_t format, const void *source, void *payload, void *scales, void *offsets, int32_t k,
                                              int32_t n, int32_t padded_n, uintptr_t stream) {
  return mrs::affine_repack(format, source, payload, scales, offsets, k, n, padded_n, 0, (cudaStream_t)stream);
}
extern "C" int32_t mrs_gguf_affine_repack_bf16(int32_t format, const void *source, void *payload, void *scales, void *offsets, int32_t k,
                                               int32_t n, int32_t padded_n, uintptr_t stream) {
  return mrs::affine_repack(format, source, payload, scales, offsets, k, n, padded_n, 1, (cudaStream_t)stream);
}
