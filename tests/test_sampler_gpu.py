"""Sampling tail (csrc/sampler.cu) behind the reference's sort.cu symbols: top-k + softmax statistics and
greedy top-1 over f32 logits, against a numpy restatement of the reference kernels' contract
((value desc, index asc) order, raw values, per-row denom / max) and against the stored outputs of the reference
kernels themselves, bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

from mistralrs_b200 import ops

pytestmark = pytest.mark.gpu


def _expected(x, k, inv_t):
    order = np.lexsort((np.arange(x.size), -x.astype(np.float64)))      # value desc, index asc
    order = [i for i in order if np.isfinite(x[i]) or x[i] == np.inf][:k]
    vals = np.full(k, -np.inf, dtype=np.float32); idx = np.zeros(k, dtype=np.int64)
    vals[:len(order)] = x[order]; idx[:len(order)] = order
    s = x.astype(np.float64) * inv_t
    gm = s.max()
    return vals, idx, np.exp(s - gm).sum(), gm


@pytest.mark.parametrize("ncols,k,temp", [(128256, 40, 0.7), (32000, 128, 1.0), (5000, 1, 2.0), (2048, 64, 0.3), (100, 50, 1.0)])
def test_topk_matches_contract(cuda, ncols, k, temp):
    rng = np.random.default_rng(ncols + k)
    # bf16-rounded logits: ties are common, which pins the (value desc, index asc) order
    x = torch.from_numpy(rng.standard_normal((3, ncols)).astype(np.float32) * 4).to(torch.bfloat16).float()
    vals, idx, denom, gmax = ops.cuda_topk_logits_f32_packed(x.to(cuda), k, temp)
    for r in range(3):
        ev, ei, ed, eg = _expected(x[r].numpy(), min(k, ncols), 1.0 / temp)
        assert np.array_equal(vals[r].cpu().numpy(), ev)
        assert np.array_equal(idx[r].cpu().numpy(), ei)
        assert abs(float(gmax[r]) - eg) <= 1e-6 * max(1.0, abs(eg))
        assert abs(float(denom[r]) - ed) <= 2e-5 * ed


def test_topk_and_top1_vs_reference_kernels(cuda):
    """Against the outputs of the reference's own sort.cu kernels on the same logits (tests/golden/ref_golden.npz,
    make_ref_golden.py)."""
    import os
    from mistralrs_b200 import lib
    ref = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_golden.npz"))
    rng = np.random.default_rng(5)
    ncols, k = 128256, 40
    nblocks = -(-ncols // 2048)
    x = torch.from_numpy(rng.standard_normal(ncols).astype(np.float32) * 3).to(torch.bfloat16).float().to(cuda)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    st = ctypes.c_int64(torch.cuda.current_stream().cuda_stream)
    L = lib()
    bv = torch.zeros(nblocks * k, dtype=torch.float32, device=cuda); bi = torch.zeros(nblocks * k, dtype=torch.int32, device=cuda)
    bm = torch.zeros(nblocks, dtype=torch.float32, device=cuda); bs = torch.zeros(nblocks, dtype=torch.float32, device=cuda)
    packed = torch.zeros(2 * k + 2, dtype=torch.float32, device=cuda)
    L.topk_large_f32_packed(P(x), P(bv), P(bi), P(bm), P(bs), P(packed), ncols, k, 2048, nblocks, ctypes.c_float(1.0 / 0.8), st)
    p1 = torch.zeros(2, dtype=torch.float32, device=cuda); tok = torch.zeros(1, dtype=torch.int32, device=cuda)
    L.top1_large_f32_packed(P(x), P(bv), P(bi), P(p1), P(tok), ncols, 2048, nblocks, st)
    torch.cuda.synchronize()
    pa, ta, ka = packed.cpu().numpy(), p1.cpu().numpy(), int(tok.item())
    pb, tb, kb = ref["sort_topk_packed"], ref["sort_top1_packed"], int(ref["sort_top1_token"][0])
    assert np.array_equal(pa[:2 * k], pb[:2 * k])                    # values and indices: bit-identical
    assert np.allclose(pa[2 * k:], pb[2 * k:], rtol=2e-5)            # denom / max: summation order
    assert np.array_equal(ta, tb) and ka == kb


def test_top1_nan_and_ties(cuda):
    x = torch.zeros(2, 5000, dtype=torch.float32)
    x[0, 1234] = 3.0; x[0, 4321] = 3.0          # tie -> first index
    x[1, 7] = float("nan")
    tok = ops.cuda_top1_logits_f32(x.to(cuda)).cpu().tolist()
    assert tok == [1234, 0xFFFFFFFF]
