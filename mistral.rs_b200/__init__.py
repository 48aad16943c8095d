"""mistral.rs_b200 — H100-native (sm_90a) quantized-linear + paged-attention hot path.

The product is `libmrs_b200.so`: hand-written CUDA kernels behind the reference's own
`extern "C"` symbols (include/*.h).  This Python package is only the thin host-side mirror of
the reference's Rust wrappers (`mistralrs-quant::gguf::fast_mmvq`, `mistralrs-paged-attn`
backend functions) used by the tests and the benchmark: PyTorch supplies device memory, streams
and torch.distributed — nothing else.  There is NO CPU fallback: importing the op modules
without the built extension raises.

The directory name contains a dot, so load it with `__graft_entry__.load_package()` (which
registers it as `mistralrs_b200`).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmrs_b200.so")

_lib = None


class ExtensionMissing(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """The CUDA extension.  Fails loudly when it has not been built (no fallback path)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ExtensionMissing(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU fallback."
            )
        _lib = ctypes.CDLL(LIB_PATH)
    return _lib


# ggml dtype codes (GgmlDType numbering of the reference / candle)
GGML = {
    "q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8, "q8_1": 9,
    "q2_k": 10, "q3_k": 11, "q4_k": 12, "q5_k": 13, "q6_k": 14,
}
BLOCK_ELEMS = {"q4_0": 32, "q4_1": 32, "q5_0": 32, "q5_1": 32, "q8_0": 32, "q8_1": 32,
               "q2_k": 256, "q3_k": 256, "q4_k": 256, "q5_k": 256, "q6_k": 256}
BLOCK_BYTES = {"q4_0": 18, "q4_1": 20, "q5_0": 22, "q5_1": 24, "q8_0": 34, "q8_1": 36,
               "q2_k": 84, "q3_k": 110, "q4_k": 144, "q5_k": 176, "q6_k": 210}
MMVQ_TYPES = ["q4_0", "q4_1", "q5_0", "q5_1", "q8_0", "q2_k", "q3_k", "q4_k", "q5_k", "q6_k"]
