"""GPTQ / AWQ int4 linear — mirrors of `GptqLayer` (REF mistralrs-quant/src/gptq/gptq_cuda.rs:
forward_raw :357-398, gptq_linear :451-623).

`GptqMarlinLayer` follows the reference's load and forward flow call for call, through the
reference's own C symbols (which libmrs_b200.so exports): `{gptq,awq}_marlin_repack` at load,
`marlin_permute_scales`, then `marlin_{gptq,awq}_4bit_{f16,bf16}` per forward — on our kernel
behind them (csrc/w4a16.cu: swap-AB wgmma GEMM, HBM-bound at decode batch).
`GptqLayer` consumes the checkpoint tensors as stored (no repack) on the same wgmma
dequant-GEMM (`mrs_gptq_gemm`, prefill-sized batches, true act-order semantics).  Only bits == 4
is implemented.  Like the reference the activations are computed in F16 (`quantized_act_type`)
and tensor parallelism is rejected (`distributed/layers.rs:776-788`)."""
import ctypes

import torch

from . import lib


class GptqLayer:
    def __init__(self, qweight, scales, qzeros=None, g_idx=None, bits=4, group_size=128, is_awq=False, bias=None,
                 world_size=1):
        if world_size > 1:
            raise ValueError("GPTQ/AWQ layers do not support tensor parallelism")
        if bits != 4:
            raise ValueError("only 4-bit GPTQ/AWQ is implemented")
        if not qweight.is_cuda:
            raise ValueError("GPTQ is only supported on CUDA")   # gptq_cpu.rs bails the same way
        self.is_awq = is_awq
        if is_awq:
            self.k, self.n = qweight.shape[0], qweight.shape[1] * 8
            if qzeros is None:
                raise ValueError("AWQ needs qzeros")
        else:
            self.k, self.n = qweight.shape[0] * 8, qweight.shape[1]
        if scales.shape != (self.k // group_size, self.n) or scales.dtype != torch.float16:
            raise ValueError(f"scales must be f16 [{self.k // group_size}, {self.n}]")
        self.qweight, self.scales, self.qzeros, self.g_idx = qweight.contiguous(), scales.contiguous(), qzeros, g_idx
        self.group_size, self.bias = group_size, bias

    def quantized_act_type(self):
        return torch.float16

    def forward(self, a: torch.Tensor) -> torch.Tensor:
        """QuantMethod::forward: cast to quantized_act_type, forward_raw, cast back."""
        orig = a.dtype
        y = self.forward_raw(a.to(torch.float16))
        return y.to(orig)

    def forward_raw(self, a: torch.Tensor) -> torch.Tensor:
        if not a.is_cuda:
            raise ValueError("Expected CUDA input to GptqLayer")
        if a.shape[-1] != self.k or a.dtype != torch.float16:
            raise ValueError("GptqLayer: bad input shape/dtype")
        x = a.reshape(-1, self.k).contiguous()
        out = torch.empty(x.shape[0], self.n, dtype=torch.float16, device=a.device)
        P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
        rc = lib().mrs_gptq_gemm(P(x), P(self.qweight), P(self.scales), P(self.qzeros), P(self.g_idx), P(out),
                                 ctypes.c_int(x.shape[0]), ctypes.c_int(self.k), ctypes.c_int(self.n),
                                 ctypes.c_int(self.group_size), ctypes.c_int(int(self.is_awq)),
                                 ctypes.c_void_p(torch.cuda.current_stream(a.device).cuda_stream))
        if rc != 0:
            raise RuntimeError(f"mrs_gptq_gemm failed with cudaError {rc}")
        out = out.reshape(*a.shape[:-1], self.n)
        return out + self.bias if self.bias is not None else out


def marlin_permute_scales(s: torch.Tensor, size_k: int, size_n: int, group_size: int) -> torch.Tensor:
    """REF gptq_cuda.rs:542-565 (`size_k` is what the reference passes: in_dim / pack_factor)."""
    scale_perm = [i + 8 * j for i in range(8) for j in range(8)]
    scale_perm_single = [2 * i + j for i in range(4) for j in (0, 1, 8, 9, 16, 17, 24, 25)]
    if group_size < size_k and group_size != -1:
        s = s.reshape(-1, len(scale_perm))[:, torch.tensor(scale_perm, device=s.device)]
    else:
        s = s.reshape(-1, len(scale_perm_single))[:, torch.tensor(scale_perm_single, device=s.device)]
    return s.reshape(-1, size_n).contiguous()


class GptqMarlinLayer:
    """The reference's default GPTQ/AWQ path (bits 4): repack at load, Marlin matmul per forward."""

    def __init__(self, qweight, scales, qzeros=None, g_idx=None, bits=4, group_size=128, is_awq=False, bias=None,
                 world_size=1):
        if world_size > 1:
            raise ValueError("GPTQ/AWQ layers do not support tensor parallelism")
        if bits != 4:
            raise ValueError("only 4-bit GPTQ/AWQ is implemented")
        if not qweight.is_cuda:
            raise ValueError("GPTQ is only supported on CUDA")
        dev = qweight.device
        st = ctypes.c_int64(torch.cuda.current_stream(dev).cuda_stream)
        P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
        self.is_awq = is_awq
        if is_awq:
            self.k, self.n = qweight.shape[0], qweight.shape[1] * 8
            self.q_weight = torch.empty(self.k // 16, self.n * 16 // 8, dtype=torch.int32, device=dev)
            lib().awq_marlin_repack(P(qweight.contiguous()), ctypes.c_void_p(0), P(self.q_weight), ctypes.c_int(self.k),
                                    ctypes.c_int(qweight.shape[1]), ctypes.c_int(bits), st)
        else:
            self.k, self.n = qweight.shape[0] * 8, qweight.shape[1]
            if g_idx is None:
                g_idx = torch.arange(self.k, device=dev, dtype=torch.int32) // (group_size if group_size > 0 else self.k)
            perm = torch.argsort(g_idx.cpu(), stable=True).to(torch.int32).to(dev)   # REF gptq_cuda.rs:578-582
            self.q_weight = torch.empty(self.k // 16, self.n * 16 // 8, dtype=torch.int32, device=dev)
            lib().gptq_marlin_repack(P(qweight.contiguous()), P(perm), P(self.q_weight), ctypes.c_int(self.k),
                                     ctypes.c_int(self.n), ctypes.c_int(bits), st)
        self.scales = marlin_permute_scales(scales, self.k // 8, self.n, group_size)
        self.qzeros = qzeros.contiguous() if qzeros is not None else None
        self.workspace = torch.zeros(self.n // 8, dtype=torch.int32, device=dev)
        self.group_size, self.bias = group_size, bias

    def quantized_act_type(self):
        return torch.float16

    def forward(self, a: torch.Tensor) -> torch.Tensor:
        orig = a.dtype
        return self.forward_raw(a.to(torch.float16)).to(orig)

    def forward_raw(self, a: torch.Tensor) -> torch.Tensor:
        """marlin_matmul (REF marlin_backend.rs:20-140): f16 or bf16 input, output of the same dtype."""
        if not a.is_cuda:
            raise ValueError("Expected CUDA input to GptqLayer")
        if a.shape[-1] != self.k or a.dtype not in (torch.float16, torch.bfloat16):
            raise ValueError("GptqMarlinLayer: bad input shape/dtype")
        x = a.reshape(-1, self.k).contiguous()
        scales = self.scales if self.scales.dtype == a.dtype else self.scales.to(a.dtype)
        out = torch.empty(x.shape[0], self.n, dtype=a.dtype, device=a.device)
        P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
        name = f"marlin_{'awq' if self.is_awq else 'gptq'}_4bit_{'f16' if a.dtype == torch.float16 else 'bf16'}"
        fn = getattr(lib(), name)
        fn.restype = ctypes.c_int
        groupsize = -1 if self.scales.shape[0] == 1 else self.k // self.scales.shape[0]
        rc = fn(P(x), P(self.q_weight), P(scales), P(self.qzeros), P(out), ctypes.c_int(x.shape[0]), ctypes.c_int(self.k),
                ctypes.c_int(self.n), P(self.workspace), ctypes.c_int(groupsize),
                ctypes.c_int64(torch.cuda.current_stream(a.device).cuda_stream))
        if rc != 0:
            raise RuntimeError(f"{name} failed with status {rc}")
        out = out.reshape(*a.shape[:-1], self.n)
        return out + self.bias if self.bias is not None else out


def dense_linear(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """y = x . w^T with dense f16/bf16 w [N, K] on the swap-AB wgmma kernel (the lm_head of GPTQ/AWQ
    checkpoints at decode batch; REF kernels/gemv/gemv.cu + candle matmul)."""
    if x.dtype != w.dtype or x.dtype not in (torch.float16, torch.bfloat16):
        raise ValueError("dense_linear: x and w must both be f16 or bf16")
    K = w.shape[1]
    xs = x.reshape(-1, K).contiguous()
    out = torch.empty(xs.shape[0], w.shape[0], dtype=x.dtype, device=x.device)
    rc = lib().mrs_dense_linear(ctypes.c_void_p(xs.data_ptr()), ctypes.c_void_p(w.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                ctypes.c_int(xs.shape[0]), ctypes.c_int(K), ctypes.c_int(w.shape[0]),
                                ctypes.c_int(0 if x.dtype == torch.float16 else 1),
                                ctypes.c_void_p(torch.cuda.current_stream(x.device).cuda_stream))
    if rc != 0:
        raise RuntimeError(f"mrs_dense_linear failed with cudaError {rc}")
    return out.reshape(*x.shape[:-1], w.shape[0])
