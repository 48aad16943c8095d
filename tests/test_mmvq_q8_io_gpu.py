"""Q8_1 activations handed between decode GEMVs (mrs_mmvq_fused mode bits 4 and 8): the fused-GLU launch can write its
output in block_q8_1 form, and a launch can take block_q8_1 input instead of quantising raw activations itself.  The
decoder chains gate∥up -> down this way, so both ends must be bit for bit what the unchained launches compute."""
import ctypes

import numpy as np
import pytest
import torch

from mistralrs_b200 import lib, quant
from util import ALL_TYPES, make_acts, make_weight, to_dev

pytestmark = pytest.mark.gpu

X_Q8_1, Y_Q8_1 = 4, 8
Q8_1_BYTES = 36  # half2 ds + 32 int8 per 32 elements


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _fused(ggml, mode, w0, w1, x, residual, dst, K, n0, n1, b, norm=None):
    from mistralrs_b200.quant import _ggml_code
    return lib().mrs_mmvq_fused(ctypes.c_int(_ggml_code(ggml)), ctypes.c_int(mode), ctypes.c_int(1), _ptr(w0), _ptr(w1),
                                _ptr(None), _ptr(x), _ptr(norm), ctypes.c_float(1e-5), _ptr(residual), _ptr(dst),
                                _ptr(None), _ptr(None), ctypes.c_int(K), ctypes.c_int(n0), ctypes.c_int(n1),
                                ctypes.c_int(0), ctypes.c_int(b), ctypes.c_int(0), ctypes.c_int(0),
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def _quantize_q8_1(x):
    """launch_mmvq_gguf_quantize_q8_1_bf16 on [b, K] -> bytes [b, K / 32 * 36]"""
    b, K = x.shape
    y = torch.zeros(b, K // 32 * Q8_1_BYTES, dtype=torch.uint8, device=x.device)
    lib().launch_mmvq_gguf_quantize_q8_1_bf16(_ptr(x), _ptr(y), ctypes.c_int(K), ctypes.c_int(K), ctypes.c_int(b),
                                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return y


@pytest.mark.parametrize("dtype", ["q4_k", "q6_k", "q8_0"])
@pytest.mark.parametrize("batch", [1, 2, 4, 8])
def test_glu_q8_1_output_is_the_quantised_glu_output(cuda, dtype, batch):
    # n = 14336 (Llama-3-8B) and 1056 (33 groups: fewer groups than CTAs in a full wave)
    K = 4096
    for n in (14336, 1056):
        wg, wu = (quant.QTensor(to_dev(make_weight(dtype, n, K, 60 + i).reshape(-1), cuda), dtype, (n, K)) for i in range(2))
        x = to_dev(make_acts(batch, K, 62, "bf16"), cuda, "bf16")
        nw = to_dev(1.0 + 0.1 * make_acts(1, K, 63, "bf16")[0], cuda, "bf16")
        act = quant.mmvq_fused(wg, x, mode=1, w1=wu, norm_w=nw, eps=1e-5)
        q8 = torch.full((batch, n // 32 * Q8_1_BYTES), 0x5A, dtype=torch.uint8, device=cuda)
        assert _fused(dtype, 1 | Y_Q8_1, wg.data, wu.data, x, None, q8, K, n, n, batch, norm=nw) == 0
        torch.cuda.synchronize()
        assert torch.equal(q8, _quantize_q8_1(act)), (dtype, batch, n)


@pytest.mark.parametrize("dtype", ALL_TYPES)
@pytest.mark.parametrize("batch", [1, 2, 4, 8])
def test_q8_1_input_equals_raw_input(cuda, dtype, batch):
    # the X_Q8_1 gather (QT::aux over the q8_1 blocks) and the fused prologue (QT::chunk_aux on the fly) build the same
    # activation image, so the outputs agree bit for bit, residual epilogue included
    for K in (4096, 14336):
        N = 96
        w = quant.QTensor(to_dev(make_weight(dtype, N, K, 70).reshape(-1), cuda), dtype, (N, K))
        x = to_dev(make_acts(batch, K, 71, "bf16"), cuda, "bf16")
        res = to_dev(make_acts(batch, N, 72, "bf16"), cuda, "bf16")
        raw = torch.empty(batch, N, dtype=torch.bfloat16, device=cuda)
        viaq8 = torch.empty_like(raw)
        rc = _fused(dtype, 0, w.data, None, x, res, raw, K, N, 0, batch)
        # 8 columns of a 14336-wide image of the small-block types do not fit in shared memory: both forms refuse it
        assert _fused(dtype, X_Q8_1, w.data, None, _quantize_q8_1(x), res, viaq8, K, N, 0, batch) == rc
        if rc != 0:
            assert batch == 8 and K == 14336 and dtype not in ("q4_k", "q6_k"), (dtype, batch, K, rc)
            continue
        torch.cuda.synchronize()
        assert torch.equal(raw, viaq8), (dtype, batch, K)


def test_q8_1_modes_reject_what_they_cannot_do(cuda):
    K, n = 256, 48                                  # 48 rows: not whole 32-row groups
    w = torch.zeros(n * 144, dtype=torch.uint8, device=cuda)
    x = torch.zeros(1, K, dtype=torch.bfloat16, device=cuda)
    out = torch.zeros(4096, dtype=torch.uint8, device=cuda)
    assert _fused("q4_k", 1 | Y_Q8_1, w, w, x, None, out, K, n, n, 1) != 0       # mis-aligned GLU row partition
    assert _fused("q4_k", 0 | Y_Q8_1, w, None, x, None, out, K, n, 0, 1) != 0    # Q8_1 output outside the GLU
    assert _fused("q4_k", X_Q8_1, w, None, out, None, out, K, n, 0, 1, norm=x) != 0   # a norm needs raw input
    assert _fused("q4_k", 16, w, None, x, None, out, K, n, 0, 1) != 0            # unknown mode bit
    assert np.all(out.cpu().numpy() == 0)
