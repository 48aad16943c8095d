"""Prompt attention kernel (csrc/prefill_attn.cu) vs a plain fp64 torch reference of the same op:
causal, GQA, ragged lengths, var-len batches, sliding window, soft-cap, both dtypes and head sizes."""
import numpy as np
import pytest
import torch

from mistralrs_b200 import paged_attn

pytestmark = pytest.mark.gpu


def _ref(q, k, v, scale, causal, window=None, softcap=None):
    T, H, D = q.shape
    g = H // k.shape[1]
    qq, kk, vv = q.double(), k.double().repeat_interleave(g, dim=1), v.double().repeat_interleave(g, dim=1)
    s = torch.einsum("thd,jhd->htj", qq, kk) * scale
    if softcap:
        s = softcap * torch.tanh(s / softcap)
    i = torch.arange(T, device=q.device)
    mask = torch.ones(T, T, dtype=torch.bool, device=q.device)
    if causal:
        mask &= i[None, :] <= i[:, None]
    if window is not None:
        mask &= i[None, :] >= i[:, None] - window
    s = s.masked_fill(~mask[None], float("-inf"))
    return torch.einsum("htj,jhd->thd", torch.softmax(s, dim=-1), vv)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("T,H,KVH,D", [(37, 4, 2, 128), (128, 8, 2, 64), (333, 8, 8, 128), (1100, 4, 1, 128)])
def test_causal_matches_reference(cuda, dt, T, H, KVH, D):
    gen = torch.Generator(device=cuda).manual_seed(T)
    q = torch.randn(T, H, D, device=cuda, generator=gen).to(dt)
    k = torch.randn(T, KVH, D, device=cuda, generator=gen).to(dt)
    v = torch.randn(T, KVH, D, device=cuda, generator=gen).to(dt)
    scale = 1.0 / np.sqrt(D)
    got = paged_attn.prefill_attention(q, k, v, scale).double()
    want = _ref(q, k, v, scale, True)
    ulp = 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -11
    # P is rounded to the activation dtype before PV (as flash-attention does) + one output rounding
    assert (got - want).abs().max().item() <= 3 * ulp * want.abs().max().item() + 1e-6


def test_window_softcap_noncausal(cuda):
    T, H, KVH, D = 300, 4, 2, 128
    gen = torch.Generator(device=cuda).manual_seed(1)
    q, k, v = (torch.randn(T, h, D, device=cuda, generator=gen).to(torch.bfloat16) for h in (H, KVH, KVH))
    scale = 1.0 / np.sqrt(D)
    for kw, ref_kw in ((dict(window_left=70), dict(causal=True, window=70)), (dict(softcap=20.0), dict(causal=True, softcap=20.0)),
                       (dict(causal=False), dict(causal=False))):
        got = paged_attn.prefill_attention(q, k, v, scale, **kw).double()
        want = _ref(q, k, v, scale, **ref_kw)
        assert (got - want).abs().max().item() <= 3 * 2.0 ** -8 * want.abs().max().item(), kw


def test_varlen_batch(cuda):
    lens = [5, 130, 64, 257]
    H, KVH, D = 8, 2, 128
    T = sum(lens)
    gen = torch.Generator(device=cuda).manual_seed(2)
    q, k, v = (torch.randn(T, h, D, device=cuda, generator=gen).to(torch.bfloat16) for h in (H, KVH, KVH))
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=cuda)
    scale = 1.0 / np.sqrt(D)
    got = paged_attn.prefill_attention(q, k, v, scale, cu_seqlens=cu, max_seqlen=max(lens)).double()
    off = 0
    for L in lens:
        want = _ref(q[off:off + L], k[off:off + L], v[off:off + L], scale, True)
        assert (got[off:off + L] - want).abs().max().item() <= 3 * 2.0 ** -8 * want.abs().max().item()
        off += L


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_both_kernels_head_128(cuda, dt):
    """Head size 128 without window / softcap runs on csrc/prefill_attn_tc.cu (wgmma, S and P in registers);
    mrs_prefill_attn_tc_debug(0, ...) keeps the call on csrc/prefill_attn.cu (mma.sync).  Both against the fp64
    reference, on a ragged multi-tile prompt, causal and not."""
    import ctypes
    from mistralrs_b200 import lib
    T, H, KVH, D = 700, 8, 2, 128
    gen = torch.Generator(device=cuda).manual_seed(9)
    q, k, v = (torch.randn(T, h, D, device=cuda, generator=gen).to(dt) for h in (H, KVH, KVH))
    scale = 1.0 / np.sqrt(D)
    ulp = 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -11
    try:
        for enable in (0, 1):
            lib().mrs_prefill_attn_tc_debug(ctypes.c_int32(enable), ctypes.c_uint32(0), ctypes.c_uint32(0))
            for causal in (True, False):
                got = paged_attn.prefill_attention(q, k, v, scale, causal=causal).double()
                want = _ref(q, k, v, scale, causal)
                assert torch.isfinite(got).all()
                assert (got - want).abs().max().item() <= 3 * ulp * want.abs().max().item() + 1e-6, (enable, causal)
    finally:
        lib().mrs_prefill_attn_tc_debug(ctypes.c_int32(1), ctypes.c_uint32(0), ctypes.c_uint32(0))
