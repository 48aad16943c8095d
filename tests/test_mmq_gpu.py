"""Prefill wgmma dequant-GEMM vs the oracle's EXACT product (f64 sum of deq(w)*x) — the
known-answer structure of the reference's own GEMM test (packed_affine.rs:967-1000:
quantized product == dequantize() . x, max abs <= 0.08, mean <= 0.01 on patterned inputs)."""
import numpy as np
import pytest
import torch

import oracle
from mistralrs_b200 import mmq, quant
from util import ALL_TYPES, make_acts, make_weight, to_dev

pytestmark = pytest.mark.gpu


def _check(dtype, M, N, K, dt, seed=0):
    cuda = torch.device("cuda:0")
    wb = make_weight(dtype, N, K, seed)
    x = make_acts(M, K, seed + 1, dt)
    w = quant.QTensor(to_dev(wb.reshape(-1), cuda), dtype, (N, K))
    y = mmq.forward(w, to_dev(x, cuda, dt)).float().cpu().numpy()
    ref = oracle.matmul_exact(dtype, wb, x, K, N)
    mag = np.abs(oracle.dequantize(dtype, wb).reshape(N, K)).astype(np.float64) @ np.abs(x).astype(np.float64).T  # sum |w||x|
    ulp = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11}[dt]
    # one output rounding + weight rounding to the operand format (2^-9 bf16 / 2^-12 f16 per
    # term, random sign -> well inside ulp * sum|w||x|) + f32 accumulation
    tol = ulp * np.abs(ref) * 1.01 + ulp * mag.T + 1e-6
    err = np.abs(y - ref)
    assert (err <= tol).all(), (dtype, M, N, K, float((err / tol).max()))


@pytest.mark.parametrize("dtype", ["q8_0", "q4_k", "q6_k"])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_main_types(cuda, dtype, dt):
    _check(dtype, 300, 520, 512, dt)      # ragged M and N (partial tiles)
    _check(dtype, 256, 256, 1024, dt, 3)  # exactly one tile, several ring wraps


@pytest.mark.parametrize("dtype", [t for t in ALL_TYPES if t not in ("q8_0", "q4_k", "q6_k")])
def test_other_types(cuda, dtype):
    _check(dtype, 130, 260, 256, "bf16", 5)


def test_reference_known_answer_shapes(cuda):
    # shapes of the reference's marlin_matches_dequantized_* tests, patterned inputs
    def patterned(shape, seed, scale):
        i = np.arange(int(np.prod(shape)))
        return (np.sin(((i * 37 + seed * 17) % 251) * 0.071) * scale).astype(np.float32).reshape(shape)
    for (m, n, k) in [(9, 64, 256), (64, 128, 512), (127, 192, 512)]:
        for dtype in ("q4_k", "q8_0", "q6_k"):
            wb = make_weight(dtype, n, k, 11)
            x = oracle.round_dtype(patterned((m, k), 3, 0.5), "bf16")
            w = quant.QTensor(to_dev(wb.reshape(-1), cuda), dtype, (n, k))
            y = mmq.forward(w, to_dev(x, cuda, "bf16")).float().cpu().numpy()
            ref = oracle.matmul_exact(dtype, wb, x, k, n)
            scale = np.abs(ref).max()
            assert np.abs(y - ref).max() <= 0.08 * max(scale, 1.0) / 8 and np.abs(y - ref).mean() <= 0.01 * max(scale, 1.0) / 8


def test_matches_decode_path_semantics(cuda):
    # GgufMatMul dispatch: batch 8 -> MMVQ (Q8_1 activations), batch 9 -> wgmma GEMM; both
    # must agree with the exact product within the reference's MMVQ-vs-dequant envelope
    K, N = 1024, 256
    wb = make_weight("q4_k", N, K, 2)
    w = quant.QTensor(to_dev(wb.reshape(-1), cuda), "q4_k", (N, K))
    lin = quant.GgufMatMul(w)
    x = make_acts(9, K, 4, "bf16")
    y9 = lin.forward(to_dev(x, cuda, "bf16")).float().cpu().numpy()
    y8 = lin.forward(to_dev(x[:8], cuda, "bf16")).float().cpu().numpy()
    ref = oracle.matmul_exact("q4_k", wb, x, K, N)
    scale = np.abs(ref).max()
    assert np.abs(y9 - ref).max() <= 2.0 ** -7 * scale
    assert np.abs(y8 - ref[:8]).max() <= 2e-2 * scale   # int8 activations: ~1/127 per-block noise


@pytest.mark.parametrize("dtype", ["q8_0", "q4_k", "q6_k"])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("M,N,K", [(300, 520, 2048), (64, 136, 4096), (129, 128, 2048)])
def test_second_generation_kernel(cuda, dtype, dt, M, N, K):
    """The k-quant "M" types on ragged token and row tiles (several 128-token tiles, a 64-token one, one token past a
    tile).  Against the exact product; bit for bit run to run (split-K partials are added in rank order); and bit for
    bit against the same product taken one 128-token launch at a time: a token row's f32 accumulation runs in k order
    whatever other tokens share the launch."""
    _check(dtype, M, N, K, dt, 7)
    wb = make_weight(dtype, N, K, 7)
    x = to_dev(make_acts(M, K, 8, dt), cuda, dt)
    w = quant.QTensor(to_dev(wb.reshape(-1), cuda), dtype, (N, K))
    y_all = mmq.forward(w, x)
    assert torch.equal(y_all, mmq.forward(w, x))
    full = M // 128 * 128   # (launches of <= 64 tokens may split K: another grouping of the same f32 sum)
    if full:
        y_cat = torch.cat([mmq.forward(w, x[i:i + 128]) for i in range(0, full, 128)])
        assert torch.equal(y_all[:full], y_cat), float((y_all[:full].float() - y_cat.float()).abs().max())
