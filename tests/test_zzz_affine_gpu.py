"""Packed-affine GGUF path (a5) on the GPU: `mrs_gguf_affine_repack_*` + `marlin_affine_{u4,u8}_*` through
`packed_affine.PackedAffine`, in the shape of the reference's own tests (packed_affine.rs `run_case`,
`marlin_matches_dequantized_q4k`, `marlin_matches_dequantized_all_affine_formats`, `unaligned_width_uses_padded_packed_dispatch`).

  * repack: payload / scales / offsets read back from the device must equal the numpy restatement bit for bit;
  * matmul: against the float64 product with the packed weights rounded once to the activation format (what the kernel
    multiplies by), tolerance = one output rounding (2^-11 f16 / 2^-8 bf16) + f32 accumulation slack;
  * and the reference's own bar against the plain dequantised weights: max |diff| <= 0.08, mean <= 0.01.

The GEMM is the warpgroup-MMA kernel of the checkpoint-layout int4 path with the affine dequantiser; the per-format
arithmetic is also checked on the CPU (tests/test_affine_host.py runs the same csrc/affine.cuh code on the host)."""
import numpy as np
import pytest
import torch

import oracle
from oracle import affine_np as A
from mistralrs_b200 import packed_affine as PA

pytestmark = pytest.mark.gpu

TORCH = {"f16": torch.float16, "bf16": torch.bfloat16}


def _blocks(dtype, nblocks, rng):
    if dtype in oracle.F16_FIELDS:
        return oracle.random_blocks(dtype, nblocks, rng, scale_exp=(-7, -5))
    raw = rng.integers(0, 256, size=(nblocks, A.SPECS[dtype][2]), dtype=np.uint8)
    d = np.exp2(rng.uniform(-10, -8, size=nblocks))
    if dtype == "q8_1":
        raw[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(nblocks, 2)
        raw[:, 2:4] = 0
    else:
        raw[:, 0:4] = d.astype(np.float32).view(np.uint8).reshape(nblocks, 4)
    return raw


def _patterned(rows, cols, seed, scale):   # packed_affine.rs `patterned`
    i = np.arange(rows * cols, dtype=np.int64)
    return (np.sin(((i * 37 + seed * 17) % 251).astype(np.float32) * np.float32(0.071)) * np.float32(scale)).reshape(rows, cols)


def _round(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(TORCH[dt]).float().numpy()


def _run_case(cuda, dtype, dt, m, n, k, seed=0):
    rng = np.random.default_rng(1000 * A.SPECS[dtype][0] + seed)
    blocks = _blocks(dtype, n * k // A.SPECS[dtype][1], rng)
    packed = PA.PackedAffine(torch.from_numpy(blocks.reshape(-1)).to(cuda), dtype, (n, k), TORCH[dt])
    torch.cuda.synchronize()
    bits, group = A.SPECS[dtype][3], A.SPECS[dtype][4]
    epay, esc, eof = A.repack(dtype, blocks, n, k, packed.padded_n, dt == "bf16")
    assert np.array_equal(packed.payload.cpu().numpy().reshape(packed.padded_n, k * bits // 8), epay)
    assert np.array_equal(packed.scales.view(torch.int16).cpu().numpy().view(np.uint16).reshape(packed.padded_n, k // group), esc)
    assert np.array_equal(packed.offsets.view(torch.int16).cpu().numpy().view(np.uint16).reshape(packed.padded_n, k // group), eof)
    x = _round(_patterned(m, k, 29, 0.1), dt)
    y = packed.forward(torch.from_numpy(x).to(cuda).to(TORCH[dt]).reshape(1, m, k))
    assert tuple(y.shape) == (1, m, n) and y.dtype == TORCH[dt] and y.is_contiguous()
    y = y.float().cpu().numpy().reshape(m, n)
    w16 = _round(A.weights(dtype, blocks, n, k, dt == "bf16"), dt).astype(np.float64)
    ref = x.astype(np.float64) @ w16.T
    ulp = 2.0 ** (-11 if dt == "f16" else -8)
    tol = ulp * np.abs(ref) * 1.01 + 2e-6 * (np.abs(x).astype(np.float64) @ np.abs(w16).T) + 1e-6
    assert (np.abs(y - ref) <= tol).all(), float((np.abs(y - ref) / tol).max())
    if dtype in oracle.F16_FIELDS:      # the reference's own acceptance bar, against the plain dequantised weights
        wd = oracle.dequantize(dtype, blocks).reshape(n, k)
        plain = x.astype(np.float64) @ _round(wd, dt).astype(np.float64).T
        d = np.abs(y - plain)
        s = max(1.0, float(np.abs(wd).max()) / 0.04)      # the reference's limits are for |w| <= 0.04 (its `patterned` weights)
        assert d.max() <= 0.08 * s and d.mean() <= 0.01 * s, (float(d.max()), float(d.mean()), s)


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("m,n,k", [(1, 64, 256), (8, 128, 256), (16, 128, 256), (17, 192, 256), (33, 256, 256), (49, 320, 256), (65, 64, 512),
                                   (127, 192, 512)])
def test_marlin_matches_dequantized_q4k(cuda, dt, m, n, k):
    _run_case(cuda, "q4_k", dt, m, n, k)


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("dtype", list(A.SPECS))
def test_marlin_matches_dequantized_all_affine_formats(cuda, dtype, dt):
    _run_case(cuda, dtype, dt, 17, 128, 256)
    _run_case(cuda, dtype, dt, 17, 96, 256, seed=1)          # padded to 128, narrowed back


@pytest.mark.parametrize("dtype,m,n,k", [("q4_k", 300, 640, 1024), ("q6_k", 257, 520, 768), ("q8_0", 512, 1024, 2048), ("q2_k", 130, 72, 512)])
def test_multi_tile_shapes(cuda, dtype, m, n, k):             # several 256-row weight tiles x several 256-token tiles, ragged edges
    _run_case(cuda, dtype, "bf16", m, n, k)


def test_rejects_what_the_plan_rejects(cuda):
    z = torch.zeros(64 * 144, dtype=torch.uint8, device=cuda)
    with pytest.raises(ValueError):
        PA.PackedAffine(z, "q4_k", (64, 128), torch.bfloat16)          # K not a whole number of source blocks
    with pytest.raises(ValueError):
        PA.PackedAffine(z, "q4_k", (64, 256), torch.float32)           # 16-bit activations only
    p = PA.PackedAffine(z, "q4_k", (64, 256), torch.bfloat16)
    with pytest.raises(ValueError):
        p.forward(torch.zeros(4, 128, dtype=torch.bfloat16, device=cuda))
    with pytest.raises(ValueError):
        p.forward(torch.zeros(4, 256, dtype=torch.float16, device=cuda))
    from mistralrs_b200 import lib
    import ctypes
    assert lib().mrs_gguf_affine_repack_f16(ctypes.c_int32(1), ctypes.c_void_p(z.data_ptr()), ctypes.c_void_p(z.data_ptr()),
                                            ctypes.c_void_p(z.data_ptr()), ctypes.c_void_p(z.data_ptr()), 256, 64, 64, ctypes.c_size_t(0)) == -1


def test_dispatch_switches_to_packed_at_minimum_batch(cuda, monkeypatch):   # packed_affine.rs:1181-1201, and the bias is kept (:1018)
    from mistralrs_b200 import quant
    monkeypatch.setenv(PA.BACKEND_ENV, "on")
    n, k = 128, 256
    rng = np.random.default_rng(7)
    blocks = _blocks("q4_k", n * k // 256, rng)
    bias = torch.from_numpy(_patterned(1, n, 3, 0.05)[0]).to(cuda).to(torch.bfloat16)
    layer = quant.GgufMatMul(quant.QTensor(torch.from_numpy(blocks.reshape(-1)).to(cuda), "q4_k", (n, k)), bias)
    small = torch.from_numpy(_patterned(PA.GGUF_AFFINE_MIN_BATCH - 1, k, 81, 0.1)).to(cuda).to(torch.bfloat16)
    layer.forward(small)
    assert getattr(layer, "_packed", None) is None
    x = torch.from_numpy(_patterned(PA.GGUF_AFFINE_MIN_BATCH, k, 83, 0.1)).to(cuda).to(torch.bfloat16)
    y = layer.forward(x)
    assert layer._packed is not None
    monkeypatch.setenv(PA.BACKEND_ENV, "off")
    y_canonical = layer.forward(x)                       # same layer through MMVQ (batch 8): the two paths agree to activation-quantisation noise
    assert torch.allclose(y.float(), y_canonical.float(), atol=0.08, rtol=0.05)


def test_fast_mmq_named_entry_points(cuda):   # fast_mmq.rs:760-826 over the (already covered) prefill GEMM + GLU kernels
    from mistralrs_b200 import mmq, ops, quant
    rng = np.random.default_rng(21)
    K, I, M = 512, 768, 40
    mk = lambda n, k: quant.QTensor(torch.from_numpy(oracle.random_blocks("q4_k", n * k // 256, rng).reshape(-1)).to(cuda), "q4_k", (n, k))
    g, u, d = mk(I, K), mk(I, K), mk(K, I)
    x = torch.from_numpy(_patterned(M, K, 5, 0.5)).to(cuda).to(torch.bfloat16)
    q, k, v = mmq.fused_qkv(g, u, u, x)
    assert torch.equal(q, mmq.plain(g, x)) and torch.equal(k, v)
    glu = mmq.fused_glu(g, u, x, quant.GluActivationType.Silu)
    assert torch.equal(glu, ops.fused_glu(mmq.forward(g, x), mmq.forward(u, x), quant.GluActivationType.Silu))
    assert torch.equal(mmq.fused_ffn(g, u, d, x, quant.GluActivationType.Silu), mmq.forward(d, glu))


def test_apply_isq_requantises_through_the_device_decoders(cuda):   # gguf/mod.rs:633-708
    from mistralrs_b200 import quant
    rng = np.random.default_rng(9)
    n, k = 32, 512
    blocks = oracle.random_blocks("q4_k", n * k // 256, rng)
    layer = quant.GgufMatMul(quant.QTensor(torch.from_numpy(blocks.reshape(-1)).to(cuda), "q4_k", (n, k)))
    w = layer.dequantize_w()
    assert w.dtype == torch.float32 and np.array_equal(w.cpu().numpy(), oracle.dequantize("q4_k", blocks).reshape(n, k))
    out = layer.apply_isq("q8_0", cuda)
    assert out.w.dtype == "q8_0" and out.w.data.device.type == "cuda"
    import gguf
    from gguf import quants
    want = quants.quantize(oracle.dequantize("q4_k", blocks).reshape(n, k), gguf.GGMLQuantizationType.Q8_0).reshape(-1)
    assert np.array_equal(out.w.data.cpu().numpy(), want)
