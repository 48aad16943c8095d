"""Host-side mirror of the reference's GGUF quantized-linear wrappers.

Mirrors, name for name and argument for argument:
  * `QTensor`            — candle's quantized tensor as the reference uses it (raw ggml blocks).
  * `plain / fused_glu / fused_qkv` — mistralrs-quant/src/gguf/fast_mmvq.rs:299,472,682
    (quantise activations to Q8_1 into a per-(device, stream, capacity) workspace, then one
    MMVQ launch; batch 1..=8; output dtype == input dtype).
  * `GgufMatMul`         — mistralrs-quant/src/gguf/mod.rs:44,440-479 (`QuantMethod::forward`).
  * `GluActivationType`  — mistralrs-quant/src/utils/ops.rs:2601-2607.

Everything below the argument checks is a call through the C ABI of libmrs_b200.so with raw
device pointers and the current CUDA stream, exactly what the Rust FFI does.
"""
import ctypes
from dataclasses import dataclass
from enum import IntEnum

import torch

from . import BLOCK_BYTES, BLOCK_ELEMS, MMVQ_TYPES, lib

MMVQ_MAX_BATCH = 8          # fast_mmvq.rs: MMVQ_MAX_BATCH
MATRIX_ROW_PADDING = 512    # fast_mmvq.rs / mmvq_gguf.cu:24
Q8_1_BLOCK_SIZE = 32
Q8_1_TYPE_SIZE = 36


class GluActivationType(IntEnum):
    Silu = 0
    Gelu = 1
    Relu = 2
    GeluErf = 3
    Sigmoid = 4


_DT_TAG = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}
_DT_CODE = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}


@dataclass
class QTensor:
    """Raw ggml blocks on the device: `data` is uint8 [nrows * ncols / qk * block_bytes]."""
    data: torch.Tensor
    dtype: str          # "q4_k", ...
    shape: tuple        # (nrows, ncols)

    def __post_init__(self):
        nrows, ncols = self.shape
        if self.dtype not in BLOCK_BYTES:
            raise ValueError(f"unsupported ggml dtype {self.dtype}")
        if ncols % BLOCK_ELEMS[self.dtype]:
            raise ValueError(f"ncols {ncols} not a multiple of the {self.dtype} block size")
        want = nrows * (ncols // BLOCK_ELEMS[self.dtype]) * BLOCK_BYTES[self.dtype]
        if self.data.dtype != torch.uint8 or self.data.numel() != want:
            raise ValueError(f"QTensor data must be uint8[{want}], got {self.data.dtype}[{self.data.numel()}]")

    @property
    def device(self):
        return self.data.device

    def nbytes(self):
        return self.data.numel()

    QUANTIZABLE = ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0")

    @classmethod
    def quantize(cls, src: torch.Tensor, dtype: str, device=None):
        """f32 [rows, cols] -> ggml blocks of `dtype` (candle `QTensor::quantize`, REF gguf/mod.rs:601-604): on the host
        (C++ host/ggml_quantize.hpp), uploaded to `device` (default: src's).  The 32-wide block types only."""
        import ctypes as C
        import numpy as np
        from . import GGML
        from .kv_index import host_lib
        if dtype not in cls.QUANTIZABLE:
            raise NotImplementedError(f"no host quantiser for {dtype} (only {', '.join(cls.QUANTIZABLE)}); K-quant quantisation is not provided")
        if src.dim() != 2 or src.shape[1] % BLOCK_ELEMS[dtype]:
            raise ValueError(f"quantize: expected [rows, cols] with cols a multiple of {BLOCK_ELEMS[dtype]}, got {tuple(src.shape)}")
        x = np.ascontiguousarray(src.detach().to(torch.float32).cpu().numpy())
        out = np.empty(x.size // BLOCK_ELEMS[dtype] * BLOCK_BYTES[dtype], dtype=np.uint8)
        L = host_lib()
        n = L.mrs_ggml_quantize(C.c_int32(GGML[dtype]), C.c_void_p(x.ctypes.data), C.c_int64(x.size), C.c_void_p(out.ctypes.data))
        if n != out.size:
            raise RuntimeError(f"mrs_ggml_quantize({dtype}) returned {n}, expected {out.size}")
        return cls(torch.from_numpy(out).to(device if device is not None else src.device), dtype, tuple(src.shape))


def supports(dtype: str) -> bool:
    return dtype in MMVQ_TYPES


def _pad(k, m):
    return (k + m - 1) // m * m


_WORKSPACE = {}


def _workspace(device, nbytes):
    """Grow-never-free scratch keyed like fast_mmvq.rs:70-112 (stable addresses for graphs)."""
    cap = 1 << max(int(nbytes) - 1, 0).bit_length()
    key = (device.index, torch.cuda.current_stream(device).cuda_stream, cap)
    buf = _WORKSPACE.get(key)
    if buf is None:
        buf = torch.empty(cap, dtype=torch.uint8, device=device)
        _WORKSPACE[key] = buf
    return buf


def _stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _check_common(name, w: QTensor, xs: torch.Tensor):
    if not supports(w.dtype):
        raise ValueError(f"{name}: unsupported quant dtype {w.dtype}")
    if not w.data.is_cuda:
        raise ValueError(f"{name}: weight must live on CUDA")
    if xs.device != w.device:
        raise ValueError(f"{name}: input and weight are on different devices")
    nrows, ncols = w.shape
    if xs.dim() < 1:
        raise ValueError(f"{name}: input must have at least one dimension")
    k = xs.shape[-1]
    b_size = 1
    for d in xs.shape[:-1]:
        b_size *= d
    if k != ncols:
        raise ValueError(f"{name}: shape mismatch: weight [{nrows}, {ncols}] vs input tail {k}")
    if b_size == 0 or b_size > MMVQ_MAX_BATCH:
        raise ValueError(f"{name}: batch size {b_size} out of supported range 1..={MMVQ_MAX_BATCH}")
    if xs.dtype not in _DT_TAG:
        raise ValueError(f"{name}: input dtype must be BF16, F16, or F32, got {xs.dtype}")
    return nrows, ncols, k, b_size


def quantize_q8_1(xs: torch.Tensor, k_padded=None) -> torch.Tensor:
    """`launch_mmvq_gguf_quantize_q8_1_{bf16,f16,f32}` into a fresh uint8 buffer (tests)."""
    xs = xs.contiguous()
    k = xs.shape[-1]
    rows = xs.numel() // k
    k_padded = k_padded or _pad(k, MATRIX_ROW_PADDING)
    out = torch.empty(rows * (k_padded // 32) * 36, dtype=torch.uint8, device=xs.device)
    fn = getattr(lib(), f"launch_mmvq_gguf_quantize_q8_1_{_DT_TAG[xs.dtype]}")
    fn(_ptr(xs), _ptr(out), ctypes.c_int(k), ctypes.c_int(k_padded), ctypes.c_int(rows), _stream_ptr(xs.device))
    return out


def _quantize_into_workspace(xs, k, b_size):
    k_padded = _pad(k, MATRIX_ROW_PADDING)
    scratch = _workspace(xs.device, b_size * (k_padded // Q8_1_BLOCK_SIZE) * Q8_1_TYPE_SIZE)
    fn = getattr(lib(), f"launch_mmvq_gguf_quantize_q8_1_{_DT_TAG[xs.dtype]}")
    fn(_ptr(xs), _ptr(scratch), ctypes.c_int(k), ctypes.c_int(k_padded), ctypes.c_int(b_size), _stream_ptr(xs.device))
    return scratch, k_padded // Q8_1_BLOCK_SIZE


def plain(w: QTensor, xs: torch.Tensor) -> torch.Tensor:
    """w @ xs^T with Q8_1 activations — fast_mmvq.rs:299 `plain`."""
    nrows, ncols, k, b_size = _check_common("fast_mmvq", w, xs)
    xs = xs.contiguous()
    scratch, stride_col_y = _quantize_into_workspace(xs, k, b_size)
    out = torch.empty(*xs.shape[:-1], nrows, dtype=xs.dtype, device=xs.device)
    fn = getattr(lib(), f"launch_mmvq_gguf_{w.dtype}_{_DT_TAG[xs.dtype]}_plain")
    fn(_ptr(w.data), _ptr(scratch), _ptr(out), ctypes.c_int(k), ctypes.c_int(nrows), ctypes.c_int(stride_col_y),
       ctypes.c_int(nrows), ctypes.c_int(b_size), _stream_ptr(xs.device))
    return out


def fused_glu(gate_w: QTensor, up_w: QTensor, xs: torch.Tensor, activation: GluActivationType) -> torch.Tensor:
    """act(gate @ x) * (up @ x) in one launch — fast_mmvq.rs:472 `fused_glu`."""
    if gate_w.dtype != up_w.dtype:
        raise ValueError(f"fast_mmvq fused_glu: gate/up dtype mismatch {gate_w.dtype} vs {up_w.dtype}")
    if gate_w.shape != up_w.shape:
        raise ValueError(f"fast_mmvq fused_glu: gate/up shape mismatch {gate_w.shape} vs {up_w.shape}")
    nrows, ncols, k, b_size = _check_common("fast_mmvq fused_glu", gate_w, xs)
    xs = xs.contiguous()
    scratch, stride_col_y = _quantize_into_workspace(xs, k, b_size)
    out = torch.empty(*xs.shape[:-1], nrows, dtype=xs.dtype, device=xs.device)
    fn = getattr(lib(), f"launch_mmvq_gguf_{gate_w.dtype}_{_DT_TAG[xs.dtype]}_fused_glu")
    fn(_ptr(gate_w.data), _ptr(up_w.data), _ptr(scratch), _ptr(out), ctypes.c_int(k), ctypes.c_int(nrows),
       ctypes.c_int(stride_col_y), ctypes.c_int(nrows), ctypes.c_int(b_size), ctypes.c_int(int(activation)),
       _stream_ptr(xs.device))
    return out


def fused_qkv(q_w: QTensor, k_w: QTensor, v_w: QTensor, xs: torch.Tensor):
    """q/k/v projections sharing one Q8_1 activation — fast_mmvq.rs:682 `fused_qkv`."""
    if not (q_w.dtype == k_w.dtype == v_w.dtype):
        raise ValueError("fast_mmvq fused_qkv: q/k/v dtype mismatch")
    if not (q_w.shape[1] == k_w.shape[1] == v_w.shape[1]):
        raise ValueError("fast_mmvq fused_qkv: q/k/v input width mismatch")
    _, _, k, b_size = _check_common("fast_mmvq fused_qkv", q_w, xs)
    xs = xs.contiguous()
    scratch, stride_col_y = _quantize_into_workspace(xs, k, b_size)
    outs = [torch.empty(*xs.shape[:-1], w.shape[0], dtype=xs.dtype, device=xs.device) for w in (q_w, k_w, v_w)]
    fn = getattr(lib(), f"launch_mmvq_gguf_{q_w.dtype}_{_DT_TAG[xs.dtype]}_fused_qkv")
    fn(_ptr(q_w.data), _ptr(k_w.data), _ptr(v_w.data), _ptr(scratch), _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]),
       ctypes.c_int(k), ctypes.c_int(q_w.shape[0]), ctypes.c_int(k_w.shape[0]), ctypes.c_int(v_w.shape[0]),
       ctypes.c_int(stride_col_y), ctypes.c_int(b_size), _stream_ptr(xs.device))
    return tuple(outs)


def mmvq_fused(w0: QTensor, xs: torch.Tensor, *, mode=0, w1=None, w2=None, norm_w=None, eps=1e-5,
               residual=None, activation=GluActivationType.Silu, pdl=False):
    """Native fused entry (`mrs_mmvq_fused`): [RMSNorm] -> Q8_1 -> GEMV -> [GLU | +residual]
    in ONE launch.  mode 0 plain, 1 fused GLU (w0=gate, w1=up), 2 fused QKV."""
    _, _, k, b_size = _check_common("mrs_mmvq_fused", w0, xs)
    xs = xs.contiguous()
    ws = [w0, w1, w2]
    n = [w.shape[0] if w is not None else 0 for w in ws]
    outs = [torch.empty(*xs.shape[:-1], n[0], dtype=xs.dtype, device=xs.device)]
    if mode == 2:
        outs += [torch.empty(*xs.shape[:-1], n[i], dtype=xs.dtype, device=xs.device) for i in (1, 2)]
    null = ctypes.c_void_p(0)
    rc = lib().mrs_mmvq_fused(
        ctypes.c_int(_ggml_code(w0.dtype)), ctypes.c_int(mode), ctypes.c_int(_DT_CODE[xs.dtype]),
        _ptr(w0.data), _ptr(w1.data) if w1 is not None else null, _ptr(w2.data) if w2 is not None else null,
        _ptr(xs), _ptr(norm_w) if norm_w is not None else null, ctypes.c_float(eps),
        _ptr(residual) if residual is not None else null,
        _ptr(outs[0]), _ptr(outs[1]) if mode == 2 else null, _ptr(outs[2]) if mode == 2 else null,
        ctypes.c_int(k), ctypes.c_int(n[0]), ctypes.c_int(n[1]), ctypes.c_int(n[2]), ctypes.c_int(b_size),
        ctypes.c_int(int(activation)), ctypes.c_int(1 if pdl else 0), _stream_ptr(xs.device))
    if rc != 0:
        raise RuntimeError(f"mrs_mmvq_fused failed with cudaError {rc}")
    return outs[0] if mode != 2 else tuple(outs)


def fused_qkv_mixed(wq: QTensor, wk: QTensor, wv: QTensor, xs: torch.Tensor, *, norm_w=None, eps=1e-5, pdl=False):
    """`mrs_mmvq_fused_qkv_mixed`: QKV where attn_v has its own ggml type (Q4_K_M: Q4_K q/k, Q6_K v) —
    one grid for the supported pairs at batch 1, else the two launches it stands for."""
    _, _, k, b_size = _check_common("mrs_mmvq_fused_qkv_mixed", wq, xs)
    if wk.dtype != wq.dtype or wk.shape[1] != k or wv.shape[1] != k:
        raise ValueError("mrs_mmvq_fused_qkv_mixed: q/k must share a dtype and all three the input width")
    xs = xs.contiguous()
    outs = [torch.empty(*xs.shape[:-1], w.shape[0], dtype=xs.dtype, device=xs.device) for w in (wq, wk, wv)]
    null = ctypes.c_void_p(0)
    rc = lib().mrs_mmvq_fused_qkv_mixed(
        ctypes.c_int(_ggml_code(wq.dtype)), ctypes.c_int(_ggml_code(wv.dtype)), ctypes.c_int(_DT_CODE[xs.dtype]),
        _ptr(wq.data), _ptr(wk.data), _ptr(wv.data), _ptr(xs), _ptr(norm_w) if norm_w is not None else null,
        ctypes.c_float(eps), _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]), ctypes.c_int(k),
        ctypes.c_int(wq.shape[0]), ctypes.c_int(wk.shape[0]), ctypes.c_int(wv.shape[0]), ctypes.c_int(b_size),
        ctypes.c_int(1 if pdl else 0), _stream_ptr(xs.device))
    if rc != 0:
        raise RuntimeError(f"mrs_mmvq_fused_qkv_mixed failed with cudaError {rc}")
    return tuple(outs)


def _ggml_code(name):
    from . import GGML
    return GGML[name]


class GgufMatMul:
    """`QuantMethod` over ggml blocks — mistralrs-quant/src/gguf/mod.rs:44 (`GgufMatMul`).

    forward(x): x [..., K] -> [..., N] (+ bias).  Dispatch as gguf/mod.rs:440-479: flat batch
    1..=8 -> MMVQ; larger batches -> the wgmma dequant-GEMM prefill path (`mmq.forward`).
    """

    def __init__(self, w: QTensor, bias: torch.Tensor = None):
        self.w = w
        self.b = bias

    def quantized_act_type(self):
        return None  # gguf/mod.rs: GGUF keeps the caller's activation dtype

    def _packed_affine_for(self, flat_batch, x):
        """Opt-in packed path (REF gguf/mod.rs:326-366): the pack is built on first use and kept."""
        from . import packed_affine as PA
        if not PA.should_dispatch(self.w.dtype, self.w.shape, flat_batch, x.dtype, x.device.type) or x.device != self.w.device:
            return None
        if getattr(self, "_packed", None) is None or self._packed.dtype != x.dtype:
            self._packed = PA.PackedAffine(self.w.data, self.w.dtype, self.w.shape, x.dtype)
        return self._packed

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        b_size = x.numel() // x.shape[-1]
        packed = self._packed_affine_for(b_size, x)
        if packed is not None:
            y = packed.forward(x)
            return y if self.b is None else y + self.b
        if 1 <= b_size <= MMVQ_MAX_BATCH:
            y = plain(self.w, x)
        else:
            from . import mmq
            y = mmq.forward(self.w, x)
        if self.b is not None:
            y = y + self.b
        return y

    def dtype_and_device(self):
        return (self.w.dtype, self.w.device)

    def dequantize_w(self) -> torch.Tensor:
        """f32 [N, K] of the weight, on its device (REF gguf/mod.rs `dequantize_w`): every row through the block decoder
        of the embedding gather kernel.  CUDA only — there is no host dequantiser in the product."""
        from . import ops
        if self.w.device.type != "cuda":
            raise RuntimeError("dequantize_w runs on the CUDA block decoders; the weight is on " + str(self.w.device))
        ids = torch.arange(self.w.shape[0], dtype=torch.int32, device=self.w.device)
        return ops.embedding_gather(self.w, ids, dtype=torch.float32)

    def apply_isq(self, dtype, device=None):
        """In-situ re-quantisation (REF gguf/mod.rs:633-708): None or the layer's own type -> the same blocks moved to
        `device`; another type -> dequantise, quantise on the host, upload.  Bias follows."""
        device = torch.device(device) if device is not None else self.w.device
        bias = None if self.b is None else self.b.to(device)
        if dtype is None or dtype == self.w.dtype:
            return GgufMatMul(QTensor(self.w.data.to(device), self.w.dtype, self.w.shape), bias)
        return GgufMatMul(QTensor.quantize(self.dequantize_w(), dtype, device), bias)

    # ---- UQFF (REF gguf/mod.rs:755-806 `serialize_uqff` / `deserialize_uqff`; entry names docs uqff-format.md) ----
    QUANTIZED_SERDE_TYPE_GGUF = 0       # REF lib.rs `QuantizedSerdeType::Gguf`

    def serialize_uqff(self, prefix: str):
        """name -> array entries of this layer: `<prefix>.weight.format` (u8 scalar), `<prefix>.weight` (raw ggml blocks),
        `<prefix>.weight.dtype` (u32 scalar, ggml code), `<prefix>.weight.shape` (u32 vector), `<prefix>.bias` if any."""
        import numpy as np
        out = {f"{prefix}.weight.format": np.array(self.QUANTIZED_SERDE_TYPE_GGUF, dtype=np.uint8),
               f"{prefix}.weight": self.w.data.detach().cpu().numpy().reshape(-1),
               f"{prefix}.weight.dtype": np.array(_ggml_code(self.w.dtype), dtype=np.uint32),
               f"{prefix}.weight.shape": np.array(list(self.w.shape), dtype=np.uint32)}
        if self.b is not None:
            out[f"{prefix}.bias"] = self.b.detach().cpu()
        return out

    @classmethod
    def deserialize_uqff(cls, archive, prefix: str, device):
        """archive: uqff_file.UqffArchive.  Blocks are uploaded as stored."""
        bias = archive.load_tensor(f"{prefix}.bias", device) if archive.contains(f"{prefix}.bias") else None
        return cls(archive.load_qtensor(prefix, device), bias)
