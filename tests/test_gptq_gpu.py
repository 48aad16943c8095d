"""GPTQ / AWQ int4 linear (wgmma path, raw checkpoint tensors) vs the numpy oracle
(w = (q-8)*s symmetric GPTQ incl. act-order g_idx; w = (q-z)*s AWQ), f16 compute.
Synthetic tensors per SURVEY §8(d): qweight uniform u4, scales f16 2^U(-8,-6), g_idx = k/128 and a
random permutation (act-order)."""
import numpy as np
import pytest
import torch

from oracle import gptq as og
from mistralrs_b200 import gptq

pytestmark = pytest.mark.gpu


def _mk(K, N, group, seed):
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 16, size=(K, N))
    scales = np.exp2(rng.uniform(-8, -6, size=(K // group, N))).astype(np.float16)
    return rng, q, scales


@pytest.mark.parametrize("act_order", [False, True])
@pytest.mark.parametrize("M", [1, 32, 300])
def test_gptq_sym(cuda, act_order, M):
    K, N, group = 1024, 520, 128
    rng, q, scales = _mk(K, N, group, 1)
    g_idx = rng.permutation(K) // group if act_order else None
    qweight = og.pack_gptq(q)
    x = rng.standard_normal((M, K)).astype(np.float16)
    layer = gptq.GptqLayer(torch.from_numpy(qweight).to(cuda), torch.from_numpy(scales).to(cuda),
                           qzeros=None, g_idx=torch.from_numpy(g_idx.astype(np.int32)).to(cuda) if act_order else None,
                           group_size=group)
    y = layer.forward_raw(torch.from_numpy(x).to(cuda)).float().cpu().numpy()
    ref = og.gemm(x, og.dequant_gptq(qweight, scales, g_idx, group))
    tol = 2.0 ** -11 * np.abs(ref) * 1.01 + 2e-6 * (np.abs(x.astype(np.float64)) @ np.abs(og.dequant_gptq(qweight, scales, g_idx, group)).astype(np.float64)) + 1e-6
    assert (np.abs(y - ref) <= tol).all(), float((np.abs(y - ref) / tol).max())


def test_awq_zero_points(cuda):
    K, N, group, M = 512, 256, 128, 40
    rng, q, scales = _mk(K, N, group, 2)
    z = rng.integers(0, 16, size=(K // group, N))
    qweight, qzeros = og.pack_awq(q), og.pack_awq(z)
    x = rng.standard_normal((M, K)).astype(np.float16)
    layer = gptq.GptqLayer(torch.from_numpy(qweight).to(cuda), torch.from_numpy(scales).to(cuda),
                           qzeros=torch.from_numpy(qzeros).to(cuda), group_size=group, is_awq=True)
    xb = torch.from_numpy(x).to(cuda).to(torch.bfloat16)
    y = layer.forward(xb)                      # QuantMethod::forward: bf16 -> f16 -> bf16
    assert y.dtype == torch.bfloat16
    ref = og.gemm(xb.to(torch.float16).cpu().numpy(), og.dequant_awq(qweight, scales, qzeros, group))
    assert np.abs(y.float().cpu().numpy() - ref).max() <= 2.0 ** -7 * np.abs(ref).max()


def test_gptq_rejects_tp_and_cpu(cuda):
    qw = torch.zeros(16, 64, dtype=torch.int32)
    sc = torch.ones(1, 64, dtype=torch.float16)
    with pytest.raises(ValueError, match="only supported on CUDA"):
        gptq.GptqLayer(qw, sc)
    with pytest.raises(ValueError, match="tensor parallelism"):
        gptq.GptqLayer(qw.to(cuda), sc.to(cuda), world_size=2)
