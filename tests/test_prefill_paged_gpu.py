"""Paged prompt attention (mrs_prefill_attention_paged: new query tokens over K/V already in the HND page cache) vs a
plain fp64 torch reference that gathers the pages through the block table.  Both kernels (wgmma for head 128 without
window / softcap, mma.sync for the rest), var-len batches with cached prefixes, shuffled non-contiguous pages, NaN in
every cache slot no sequence owns, padded table rows, bit-equality with the fresh kernel, chunking, graph capture."""
import ctypes

import numpy as np
import pytest
import torch

from mistralrs_b200 import lib, paged_attn

pytestmark = pytest.mark.gpu

CACHED = [0, 1, 15, 16, 300, 1000]
QLENS = [1, 7, 128, 129, 700, 64]


def _ulp(dt):
    return 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -11


def _tc(enable):
    lib().mrs_prefill_attn_tc_debug(ctypes.c_int32(enable), ctypes.c_uint32(0), ctypes.c_uint32(0))


@pytest.fixture
def both_kernels():
    yield
    _tc(1)


def _setup(dev, dt, page, H, KVH, D, cached, qlens, seed, pad=-1, contiguous=False, extra_pages=3):
    """Cache [NB, KVH, page, D] filled with NaN except the rows each sequence owns (< kv_len); pages of all sequences
    shuffled over the pool (or in order when contiguous); table rows padded with `pad` past each sequence's pages."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    kv_lens = [c + q for c, q in zip(cached, qlens)]
    npages = [-(-L // page) for L in kv_lens]
    nb = sum(npages) + 5
    ids = np.arange(1, nb) if contiguous else np.random.default_rng(seed).permutation(np.arange(1, nb))
    width = max(npages) + extra_pages
    table = np.full((len(kv_lens), width), pad, dtype=np.int64)
    k_seq, v_seq, used = [], [], 0
    kc = torch.full((nb, KVH, page, D), float("nan"), dtype=dt, device=dev)
    vc = torch.full_like(kc, float("nan"))
    for b, L in enumerate(kv_lens):
        table[b, :npages[b]] = ids[used:used + npages[b]]
        used += npages[b]
        k = torch.randn(L, KVH, D, device=dev, generator=gen).to(dt)
        v = torch.randn(L, KVH, D, device=dev, generator=gen).to(dt)
        j = torch.arange(L, device=dev)
        blk = torch.as_tensor(table[b], device=dev)[j // page]
        kc[blk, :, j % page] = k
        vc[blk, :, j % page] = v
        k_seq.append(k); v_seq.append(v)
    q = torch.randn(sum(qlens), H, D, device=dev, generator=gen).to(dt)
    bt = torch.as_tensor(table.astype(np.int32), device=dev)
    cu_q = torch.tensor(np.concatenate([[0], np.cumsum(qlens)]), dtype=torch.int32, device=dev)
    cu_k = torch.tensor(np.concatenate([[0], np.cumsum(kv_lens)]), dtype=torch.int32, device=dev)
    return dict(q=q, kc=kc, vc=vc, bt=bt, cu_q=cu_q, cu_k=cu_k, k_seq=k_seq, v_seq=v_seq, qlens=list(qlens), kv_lens=kv_lens)


def _call(s, scale, causal=True, **kw):
    return paged_attn.prefill_attention_paged(s["q"], s["kc"], s["vc"], s["bt"], s["cu_q"], s["cu_k"], max(s["qlens"]),
                                              max(s["kv_lens"]), scale, causal=causal, **kw)


def _ref(q, k, v, scale, causal, window=None, softcap=None):
    """q [Tq, H, D] at positions kv_len - Tq .. kv_len - 1 over k / v [kv_len, KVH, D], fp64"""
    Tq, H, D = q.shape
    L = k.shape[0]
    g = H // k.shape[1]
    qq, kk, vv = q.double(), k.double().repeat_interleave(g, dim=1), v.double().repeat_interleave(g, dim=1)
    s = torch.einsum("thd,jhd->htj", qq, kk) * scale
    if softcap:
        s = softcap * torch.tanh(s / softcap)
    pos = torch.arange(Tq, device=q.device)[:, None] + (L - Tq)
    j = torch.arange(L, device=q.device)[None, :]
    mask = torch.ones(Tq, L, dtype=torch.bool, device=q.device)
    if causal:
        mask &= j <= pos
    if window is not None:
        mask &= j >= pos - window
    s = s.masked_fill(~mask[None], float("-inf"))
    return torch.einsum("htj,jhd->thd", torch.softmax(s, dim=-1), vv)


def _check(s, got, scale, causal, dt, what, **kw):
    assert torch.isfinite(got).all(), what
    off = 0
    for b, Lq in enumerate(s["qlens"]):
        want = _ref(s["q"][off:off + Lq], s["k_seq"][b], s["v_seq"][b], scale, causal,
                    window=kw.get("window_left"), softcap=kw.get("softcap"))
        err = (got[off:off + Lq].double() - want).abs().max().item()
        assert err <= 3 * _ulp(dt) * want.abs().max().item() + 1e-6, (what, b, err)
        off += Lq


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("H,KVH", [(8, 2), (4, 4)])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("page", [8, 16, 32])
def test_varlen_grid_matches_reference(cuda, both_kernels, page, dt, D, H, KVH, causal):
    s = _setup(cuda, dt, page, H, KVH, D, CACHED, QLENS, seed=page * 7 + D + H)
    scale = 1.0 / np.sqrt(D)
    for enable in ((1, 0) if D == 128 else (1,)):
        _tc(enable)
        _check(s, _call(s, scale, causal), scale, causal, dt, (enable, causal))


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("page", [8, 16, 32])
def test_window_and_softcap(cuda, page, D):
    dt = torch.bfloat16
    s = _setup(cuda, dt, page, 8, 2, D, CACHED, QLENS, seed=100 + page + D)
    scale = 1.0 / np.sqrt(D)
    for kw in (dict(window_left=70), dict(softcap=20.0), dict(window_left=200, softcap=30.0)):
        for causal in (True, False) if "window_left" not in kw else (True,):
            _check(s, _call(s, scale, causal, **kw), scale, causal, dt, kw, **kw)


@pytest.mark.parametrize("pad", [-1, 2 ** 31 - 1])
@pytest.mark.parametrize("D", [64, 128])
def test_garbage_outside_sequence_is_ignored(cuda, both_kernels, pad, D):
    """NaN in every slot no sequence owns (stale rows of each last page included), table rows padded with -1 or a
    huge id: output finite and equal to the reference, on both kernels."""
    dt = torch.bfloat16
    s = _setup(cuda, dt, 16, 8, 2, D, [3, 0, 250, 17], [5, 33, 140, 1], seed=pad & 0xFFFF, pad=pad, extra_pages=8)
    scale = 1.0 / np.sqrt(D)
    for enable in ((1, 0) if D == 128 else (1,)):
        _tc(enable)
        for causal in (True, False):
            _check(s, _call(s, scale, causal), scale, causal, dt, (enable, causal, pad))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", [64, 128])
def test_uncached_equals_fresh_kernel_bitwise(cuda, both_kernels, dt, D):
    """cached = 0 and a contiguous table: the same tiles in the same order with the same arithmetic as
    mrs_prefill_attention on the same k / v, so the outputs are identical on each kernel."""
    lens = [37, 300, 129, 1]
    s = _setup(cuda, dt, 16, 8, 2, D, [0] * len(lens), lens, seed=5 + D, contiguous=True)
    k, v = torch.cat(s["k_seq"]), torch.cat(s["v_seq"])
    scale = 1.0 / np.sqrt(D)
    for enable in ((1, 0) if D == 128 else (1,)):
        _tc(enable)
        for causal in (True, False):
            fresh = paged_attn.prefill_attention(s["q"], k, v, scale, causal=causal, cu_seqlens=s["cu_q"], max_seqlen=max(lens))
            paged = _call(s, scale, causal)
            assert torch.equal(fresh, paged), (enable, causal, (fresh.float() - paged.float()).abs().max().item())


@pytest.mark.parametrize("D", [64, 128])
def test_chunked_matches_one_shot(cuda, D):
    dt, page = torch.bfloat16, 16
    s = _setup(cuda, dt, page, 8, 2, D, [0], [1000], seed=11 + D)
    scale = 1.0 / np.sqrt(D)
    one = _call(s, scale)
    parts, done = [], 0
    for n in (300, 300, 400):
        cu_q = torch.tensor([0, n], dtype=torch.int32, device=cuda)
        cu_k = torch.tensor([0, done + n], dtype=torch.int32, device=cuda)
        parts.append(paged_attn.prefill_attention_paged(s["q"][done:done + n], s["kc"], s["vc"], s["bt"], cu_q, cu_k, n,
                                                        done + n, scale))
        done += n
    got = torch.cat(parts)
    assert (got.double() - one.double()).abs().max().item() <= 3 * _ulp(dt) * one.double().abs().max().item()
    _check(s, got, scale, True, dt, "chunked")


def test_graph_capture_replays_eager(cuda):
    dt = torch.bfloat16
    s = _setup(cuda, dt, 16, 8, 2, 128, [300, 16], [129, 7], seed=21)
    scale = 1.0 / np.sqrt(128)
    eager = _call(s, scale)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = _call(s, scale)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
