"""Prefill (batch > 8) quantized GEMM — mirror of `fast_mmq::plain`
(REF mistralrs-quant/src/gguf/fast_mmq.rs:762-826) on the wgmma dequant-GEMM kernel
(`mrs_mmq_gguf`, csrc/mmq_tc.cu).  Unlike the reference there is no activation quantisation
pass: activations stay bf16/f16 and weights are dequantised on the fly into shared memory."""
import ctypes

import torch

from . import GGML, lib

_DT_CODE = {torch.float16: 0, torch.bfloat16: 1}


def forward(w, xs: torch.Tensor) -> torch.Tensor:
    """w: quant.QTensor [N, K]; xs [..., K] bf16/f16 -> [..., N]."""
    if xs.dtype not in _DT_CODE:
        raise ValueError(f"fast_mmq: input dtype must be BF16 or F16, got {xs.dtype}")
    nrows, ncols = w.shape
    if xs.shape[-1] != ncols:
        raise ValueError(f"fast_mmq: shape mismatch: weight [{nrows}, {ncols}] vs input tail {xs.shape[-1]}")
    if xs.device != w.device:
        raise ValueError("fast_mmq: input and weight are on different devices")
    if ncols % 64:
        raise ValueError("fast_mmq: K must be a multiple of 64")
    xs = xs.contiguous()
    M = xs.numel() // ncols
    out = torch.empty(*xs.shape[:-1], nrows, dtype=xs.dtype, device=xs.device)
    rc = lib().mrs_mmq_gguf(ctypes.c_int(GGML[w.dtype]), ctypes.c_void_p(w.data.data_ptr()), ctypes.c_void_p(xs.data_ptr()),
                            ctypes.c_void_p(out.data_ptr()), ctypes.c_int(M), ctypes.c_int(nrows), ctypes.c_int(ncols),
                            ctypes.c_int(_DT_CODE[xs.dtype]), ctypes.c_void_p(torch.cuda.current_stream(xs.device).cuda_stream))
    if rc != 0:
        raise RuntimeError(f"mrs_mmq_gguf failed with cudaError {rc}")
    return out


def grouped(ws, xs: torch.Tensor, glu=False, pdl=False):
    """One launch of `mrs_mmq_gguf_grouped` over 1..3 QTensors of one ggml type that share K: returns
    [xs . W_m^T for each m], or with glu=True (ws = (gate, up)) silu(xs . gate^T) * (xs . up^T) in one tensor.
    xs [M, K] bf16/f16."""
    ws = list(ws)
    if not 1 <= len(ws) <= 3 or len({w.dtype for w in ws}) != 1 or len({w.shape[1] for w in ws}) != 1:
        raise ValueError("fast_mmq grouped: need 1..3 weights of one ggml type and one K")
    if glu and (len(ws) != 2 or tuple(ws[0].shape) != tuple(ws[1].shape)):
        raise ValueError("fast_mmq grouped: glu needs gate and up of one shape")
    if xs.dtype not in _DT_CODE or xs.dim() != 2 or xs.shape[1] != ws[0].shape[1]:
        raise ValueError(f"fast_mmq grouped: need a bf16/f16 input [M, {ws[0].shape[1]}], got {tuple(xs.shape)} {xs.dtype}")
    xs = xs.contiguous()
    M, K = xs.shape
    outs = [torch.empty(M, w.shape[0], dtype=xs.dtype, device=xs.device) for w in (ws[:1] if glu else ws)]
    n = len(ws)
    w_arr = (ctypes.c_void_p * n)(*[w.data.data_ptr() for w in ws])
    rows = (ctypes.c_int32 * n)(*[w.shape[0] for w in ws])
    y_arr = (ctypes.c_void_p * n)(*([o.data_ptr() for o in outs] + [None] * (n - len(outs))))
    rc = lib().mrs_mmq_gguf_grouped(ctypes.c_int32(GGML[ws[0].dtype]), ctypes.c_int32(n), w_arr, rows, y_arr,
                                    ctypes.c_void_p(xs.data_ptr()), ctypes.c_int32(M), ctypes.c_int32(K),
                                    ctypes.c_int32(_DT_CODE[xs.dtype]), ctypes.c_int32(int(glu)), ctypes.c_int32(int(pdl)),
                                    ctypes.c_void_p(torch.cuda.current_stream(xs.device).cuda_stream))
    if rc != 0:
        raise RuntimeError(f"mrs_mmq_gguf_grouped failed with cudaError {rc}")
    return outs[0] if glu else outs


# ---- the reference's entry points over this kernel (REF mistralrs-quant/src/gguf/fast_mmq.rs:760-826).  In the reference the
# point of the fused forms is ONE activation-quantisation pass shared by the projections; this design never quantises
# activations, so they are the same projections over the same bf16/f16 input — kept under the reference's names so a
# caller written against fast_mmq finds them. ----
def plain(w, xs: torch.Tensor) -> torch.Tensor:
    return forward(w, xs)


def fused_qkv(q_w, k_w, v_w, xs: torch.Tensor):
    return forward(q_w, xs), forward(k_w, xs), forward(v_w, xs)


def fused_glu(gate_w, up_w, xs: torch.Tensor, activation) -> torch.Tensor:
    if tuple(gate_w.shape) != tuple(up_w.shape):
        raise ValueError(f"fast_mmq fused_glu: gate/up shape mismatch {tuple(gate_w.shape)} vs {tuple(up_w.shape)}")
    from . import ops
    return ops.fused_glu(forward(gate_w, xs), forward(up_w, xs), activation)


def fused_ffn(gate_w, up_w, down_w, xs: torch.Tensor, activation) -> torch.Tensor:
    if tuple(gate_w.shape) != tuple(up_w.shape):
        raise ValueError(f"fast_mmq fused_ffn: gate/up shape mismatch {tuple(gate_w.shape)} vs {tuple(up_w.shape)}")
    return forward(down_w, fused_glu(gate_w, up_w, xs, activation))
