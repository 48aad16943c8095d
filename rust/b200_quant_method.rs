//! How mistralrs-quant binds the H100 library — SOURCE ONLY (no Rust toolchain exists in the build
//! image, so this file is checked mechanically against include/*.h by tests/test_abi.py, not compiled).
//!
//! 1. Nothing changes for the reference-named launchers: `gguf/ffi.rs`, `gptq/marlin_ffi.rs`,
//!    `rotary/ffi.rs`, `utils/ffi.rs`, `mistralrs-paged-attn/src/cuda/ffi.rs` keep their `extern "C"`
//!    blocks; `build.rs` links `libmrs_b200` instead of compiling `kernels/*.cu`
//!    (`println!("cargo:rustc-link-lib=dylib=mrs_b200")`), and `GgufMatMul::forward_raw`
//!    (gguf/mod.rs:440-479) dispatches exactly as before: batch 1..=8 -> `fast_mmvq::*`,
//!    larger -> `fast_mmq::*`, GPTQ/AWQ -> `marlin_matmul`.
//! 2. The native fast paths are opt-in wrappers over `mrs_b200_ffi.rs` (generated from the C
//!    headers).  The one below replaces `fast_mmvq::plain` + the preceding RMSNorm + the following
//!    residual add with a single launch; it keeps `QuantMethod`'s contract (same shapes, dtypes and
//!    error behaviour) because it is only a different implementation of `forward_raw`.
use std::ffi::c_void;

use candle_core::{cuda::cudarc::driver::DevicePtr, quantized::QTensor, DType, Result, Storage, Tensor};

use crate::mrs_b200_ffi as ffi;

/// GgmlDType -> the integer code both libraries use (candle's numbering: Q4_0 = 2 ... Q6K = 14).
fn ggml_code(dtype: candle_core::quantized::GgmlDType) -> Result<i32> {
    use candle_core::quantized::GgmlDType::*;
    Ok(match dtype {
        Q4_0 => 2, Q4_1 => 3, Q5_0 => 6, Q5_1 => 7, Q8_0 => 8,
        Q2K => 10, Q3K => 11, Q4K => 12, Q5K => 13, Q6K => 14,
        other => candle_core::bail!("mrs_b200: unsupported ggml dtype {other:?}"),
    })
}

fn act_code(dtype: DType) -> Result<i32> {
    Ok(match dtype {
        DType::F16 => 0,
        DType::BF16 => 1,
        DType::F32 => 2,
        other => candle_core::bail!("mrs_b200: activations must be f16/bf16/f32, got {other:?}"),
    })
}

/// `y = W . q8_1(rmsnorm(x)) + residual` in one launch (decode, batch 1..=8).
/// Mirrors `fast_mmvq::plain` (gguf/fast_mmvq.rs:299): same guards, same output allocation, same stream.
pub fn fused_norm_linear_residual(
    w: &QTensor,
    xs: &Tensor,
    norm_weight: Option<&Tensor>,
    eps: f32,
    residual: Option<&Tensor>,
) -> Result<Tensor> {
    let (nrows, ncols) = w.shape().dims2()?;
    let batch = xs.elem_count() / ncols;
    if !(1..=8).contains(&batch) {
        candle_core::bail!("mrs_b200 fused decode linear: batch {batch} outside 1..=8");
    }
    let dev = xs.device().as_cuda_device()?;
    let stream = dev.cuda_stream();
    let xs = xs.contiguous()?;
    let out = unsafe { dev.alloc::<half::bf16>(nrows * batch)? };
    let (w_ptr, _wg) = w.device_ptr_with_guard(&stream)?;
    let ptr_of = |t: &Tensor| -> Result<u64> {
        let (st, l) = t.storage_and_layout();
        match &*st {
            Storage::Cuda(c) => Ok(c.as_cuda_slice::<half::bf16>()?.device_ptr(&stream).0 + (l.start_offset() * 2) as u64),
            _ => candle_core::bail!("mrs_b200: tensor must live on CUDA"),
        }
    };
    let x_ptr = ptr_of(&xs)?;
    let n_ptr = norm_weight.map(ptr_of).transpose()?.unwrap_or(0);
    let r_ptr = residual.map(ptr_of).transpose()?.unwrap_or(0);
    let (o_ptr, _og) = out.device_ptr(&stream);
    let rc = unsafe {
        ffi::mrs_mmvq_fused(
            ggml_code(w.dtype())?, 0, act_code(xs.dtype())?, w_ptr as *const c_void, std::ptr::null(), std::ptr::null(),
            x_ptr as *const c_void, n_ptr as *const c_void, eps, r_ptr as *const c_void, o_ptr as *mut c_void,
            std::ptr::null_mut(), std::ptr::null_mut(), ncols as i32, nrows as i32, 0, 0, batch as i32, 0,
            /* pdl */ 1, stream.cu_stream() as *mut c_void,
        )
    };
    if rc != 0 {
        candle_core::bail!("mrs_mmvq_fused failed with cudaError {rc}");
    }
    crate::utils::wrap_cuda_output(out, dev, (batch, nrows))
}
