#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY — builds the UNMODIFIED reference CUDA kernels of the hot path
# straight from /root/reference (sources are never copied into this repo) into
# oracle/_ref/*.so.  These shared objects are the GPU-side oracle ("what does the
# reference itself compute on these inputs?") and the "beat this" timing baseline.
#
# Flags follow mistralrs-quant/build.rs:28-43 and mistralrs-paged-attn/build.rs:110-131
# (-O3 --use_fast_math, half/bf16 operators enabled, -DENABLE_FP8 for paged-attn); the
# arch is what the reference's build scripts would pick on an H100 (compute cap 90 ->
# sm_90, no "a" suffix: mistralrs-quant/build.rs:147).
#
# Usage: oracle/build_ref.sh [target ...]   (default: all fast targets; "flashinfer" is
# ~10 min and is only built when asked for or when ALL=1).
set -euo pipefail
REF=${MRS_REFERENCE_ROOT:-/root/reference}
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/_ref"
mkdir -p "$OUT"
if [ ! -d "$REF" ]; then
  echo "build_ref: $REF not present (GPU box?) - using prebuilt oracle/_ref/*.so if any"; exit 0
fi
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
COMMON=(-std=c++17 -O3 -U__CUDA_NO_HALF_OPERATORS__ -U__CUDA_NO_HALF_CONVERSIONS__
        -U__CUDA_NO_HALF2_OPERATORS__ -U__CUDA_NO_BFLOAT16_CONVERSIONS__
        --expt-relaxed-constexpr --expt-extended-lambda --use_fast_math
        -gencode arch=compute_90,code=sm_90 --compiler-options -fPIC -shared)
Q="$REF/mistralrs-quant/kernels"
P="$REF/mistralrs-paged-attn/src/cuda"
C="$REF/mistralrs-core/src/cuda"

build() { # name  sources...  [-- extra flags]
  local name=$1; shift
  local so="$OUT/libref_$name.so"
  local newest=0
  for a in "$@"; do [ -f "$a" ] && [ "$a" -nt "$so" ] && newest=1; done
  if [ -f "$so" ] && [ $newest -eq 0 ]; then echo "build_ref: $name up to date"; return; fi
  echo "build_ref: building $name"; local t0=$SECONDS
  "$NVCC" "${COMMON[@]}" "$@" -o "$so.tmp" && mv "$so.tmp" "$so"
  echo "build_ref: $name done in $((SECONDS-t0)) s"
}

targets=("$@")
if [ ${#targets[@]} -eq 0 ]; then targets=(mmvq rotary ops cache pagedattn rmsnorm mmq marlin); fi
if [ "${ALL:-0}" = "1" ]; then targets+=(flashinfer); fi

for t in "${targets[@]}"; do
  case $t in
    mmvq)      build mmvq "$Q/mmvq_gguf/mmvq_gguf.cu" & ;;
    rotary)    build rotary "$Q/rotary/rotary.cu" -I"$Q/rotary" & ;;
    ops)       build ops "$Q/ops/ops.cu" & ;;
    cache)     build cache "$P/reshape_and_cache_kernel.cu" "$P/gather_kv_cache_kernel.cu" "$P/copy_blocks_kernel.cu" -I"$P" -DENABLE_FP8 & ;;
    pagedattn) build pagedattn "$P/pagedattention_v1_bf16.cu" "$P/pagedattention_v2_bf16.cu" "$P/pagedattention_v1_f16.cu" "$P/pagedattention_v2_f16.cu" -I"$P" -DENABLE_FP8 & ;;
    rmsnorm)   build rmsnorm "$C/sort.cu" & ;;
    mmq)       build mmq "$Q/mmq_gguf/mmq_quantize.cu" "$Q/mmq_gguf/mmq_instance_q4_k.cu" "$Q/mmq_gguf/mmq_instance_q6_k.cu" "$Q/mmq_gguf/mmq_instance_q8_0.cu" -I"$Q/mmq_gguf" & ;;
    marlin)    build marlin "$Q/marlin/marlin_matmul_f16.cu" "$Q/marlin/marlin_matmul_bf16.cu" "$Q/marlin/marlin_repack.cu" -I"$Q/marlin" & ;;
    flashinfer) build flashinfer "$P/flashinfer_decode.cu" -I"$P" -DENABLE_FP8 & ;;
    *) echo "unknown target $t"; exit 2 ;;
  esac
done
wait
ls -la "$OUT"
