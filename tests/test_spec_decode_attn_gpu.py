"""Multi-query fused decode attention (mrs_paged_decode_fused_multi, the verify step of speculative decoding) against
a float64 restatement with a per-row causal mask: query row i of a sequence sits at position kv_len - q + i and sees
every key up to and including it.  Covers q 1..8, GQA groups 1 / 4 / 8, head 64 / 128, f16 / bf16, pages of 8 / 16 / 32,
var-len batches over shuffled pages, unsplit / cluster-merge / counter-merge plans, and NaN in every cache row the
kernel must not read (rows at or past kv_len - q before the call, slots no sequence owns)."""
import ctypes

import numpy as np
import pytest
import torch

from mistralrs_b200 import kv_index, lib, ops, paged_attn

pytestmark = pytest.mark.gpu

_DT = {torch.float16: 0, torch.bfloat16: 1}


def causal_ref(q, keys, vals, scale):
    """q [Q, H, D], keys / vals [kv_len, KVH, D] (all rows, the q new ones last) -> [Q, H, D] in float64"""
    Q, H, D = q.shape
    kv_len, KVH = keys.shape[0], keys.shape[1]
    g = H // KVH
    out = np.zeros((Q, H, D))
    for i in range(Q):
        n = kv_len - Q + i + 1
        for h in range(H):
            s = keys[:n, h // g].astype(np.float64) @ q[i, h].astype(np.float64) * scale
            p = np.exp(s - s.max())
            out[i, h] = (p / p.sum()) @ vals[:n, h // g].astype(np.float64)
    return out


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def call_multi(fn, qt, kn, vn, kc, vc, cos, sin, pos, slots, indptr, indices, last, req, tile, o_indptr, chunk, mask, out,
               tmp_v, tmp_s, counters, B, padded, H, KVH, D, bs, scale, dt, q_len=None):
    args = [_ptr(qt), _ptr(kn), _ptr(vn), _ptr(kc), _ptr(vc), _ptr(cos), _ptr(sin), _ptr(pos), _ptr(slots), _ptr(indptr),
            _ptr(indices), _ptr(last), _ptr(req), _ptr(tile), _ptr(o_indptr), _ptr(chunk), _ptr(mask), _ptr(out),
            _ptr(tmp_v), _ptr(tmp_s), _ptr(counters), B, padded, H, KVH, D, bs, ctypes.c_float(scale), ctypes.c_uint32(_DT[dt]), 0]
    if q_len is not None:
        args.append(q_len)
    rc = getattr(lib(), fn)(*args, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc


def setup(cuda, dt, D, group, Q, bs, ctx, plan, seed=0):
    """ctx: per-sequence kv_len (the q new rows included).  plan: 'unsplit' | 'split' (batch 1: cluster merge, batch > 1:
    counter merge) | 'counter' (the split plan with the cluster merge turned off)."""
    gen = torch.Generator().manual_seed(seed)
    B, KVH = len(ctx), 2
    H = KVH * group
    nblk = [-(-c // bs) for c in ctx]
    NB = sum(nblk) + 3
    perm = (torch.randperm(NB - 1, generator=gen) + 1).tolist()          # shuffled pages; some belong to nobody
    tables, o = [], 0
    for n in nblk:
        tables.append(perm[o:o + n]); o += n
    kc = torch.full((NB, KVH, bs, D), float("nan"), dtype=dt)
    vc = torch.full((NB, KVH, bs, D), float("nan"), dtype=dt)
    old_k = [torch.randn(c - Q, KVH, D, generator=gen).to(dt) for c in ctx]     # already rotated, in the cache
    old_v = [torch.randn(c - Q, KVH, D, generator=gen).to(dt) for c in ctx]
    for b in range(B):
        for t in range(ctx[b] - Q):
            kc[tables[b][t // bs], :, t % bs] = old_k[b][t]; vc[tables[b][t // bs], :, t % bs] = old_v[b][t]
    qt = torch.randn(B * Q, H, D, generator=gen).to(dt)
    kn = torch.randn(B * Q, KVH, D, generator=gen).to(dt)
    vn = torch.randn(B * Q, KVH, D, generator=gen).to(dt)
    max_pos = max(ctx) + 8
    inv = 1.0 / (10000.0 ** (np.arange(0, D, 2) / D))
    fr = np.arange(max_pos)[:, None] * inv[None, :]
    cos = torch.from_numpy(np.cos(fr)).to(dt).to(cuda); sin = torch.from_numpy(np.sin(fr)).to(dt).to(cuda)
    pos = torch.tensor([c - Q + i for c in ctx for i in range(Q)], dtype=torch.int32)
    slots = torch.tensor([tables[b][p // bs] * bs + p % bs for b in range(B) for p in range(ctx[b] - Q, ctx[b])], dtype=torch.int64)
    indptr, indices, last = kv_index.make_paged_kv_tensors(tables, ctx, bs, sum(nblk))
    split = None if plan == "unsplit" else -(-max(nblk) // 4)          # <= 4 tiles per sequence: a batch-1 cluster
    padded = B if plan == "unsplit" else sum(-(-n // split) for n in nblk)
    req, tile, o_indptr, chunk, mask = kv_index.make_paged_kv_decode_tensors(tables, ctx, bs, split, padded)
    T = lambda a, d=torch.int32: torch.as_tensor(np.asarray(a)).to(d).to(cuda)
    d = dict(qt=qt.to(cuda), kn=kn.to(cuda), vn=vn.to(cuda), kc=kc.to(cuda), vc=vc.to(cuda), cos=cos, sin=sin, pos=pos.to(cuda),
             slots=slots.to(cuda), indptr=T(indptr), indices=T(indices), last=T(last), req=T(req), tile=T(tile),
             o_indptr=T(o_indptr), chunk=T(chunk), mask=T(mask, torch.uint8), out=torch.zeros(B * Q, H, D, dtype=dt, device=cuda),
             tmp_v=None if plan == "unsplit" else torch.zeros(padded, Q * H, D, dtype=dt, device=cuda),
             tmp_s=None if plan == "unsplit" else torch.zeros(padded, Q * H, dtype=torch.float32, device=cuda),
             counters=torch.zeros(B * KVH * -(-group * Q // 16), dtype=torch.int32, device=cuda))
    meta = dict(B=B, padded=padded, H=H, KVH=KVH, D=D, bs=bs, scale=D ** -0.5, dt=dt)
    return d, meta, old_k, old_v, tables


def run(fn, d, meta, Q=None):
    call_multi(fn, d["qt"], d["kn"], d["vn"], d["kc"], d["vc"], d["cos"], d["sin"], d["pos"], d["slots"], d["indptr"],
               d["indices"], d["last"], d["req"], d["tile"], d["o_indptr"], d["chunk"], d["mask"], d["out"], d["tmp_v"],
               d["tmp_s"], d["counters"], meta["B"], meta["padded"], meta["H"], meta["KVH"], meta["D"], meta["bs"],
               meta["scale"], meta["dt"], Q)


CASES = [  # (dtype, D, group, q, page, ctx, plan)
    (torch.bfloat16, 128, 4, 4, 16, [300], "split"), (torch.bfloat16, 128, 4, 2, 16, [300], "split"),
    (torch.bfloat16, 128, 4, 8, 16, [131], "split"), (torch.float16, 128, 4, 3, 16, [77, 5, 200], "split"),
    (torch.float16, 64, 8, 5, 8, [40, 9], "split"), (torch.bfloat16, 64, 1, 7, 32, [70], "split"),
    (torch.bfloat16, 64, 1, 1, 32, [33, 64], "unsplit"), (torch.float16, 128, 8, 6, 32, [150, 12], "unsplit"),
    (torch.bfloat16, 64, 4, 8, 8, [8, 100], "unsplit"), (torch.float16, 64, 4, 2, 16, [17], "unsplit"),
    (torch.bfloat16, 128, 1, 4, 8, [260], "counter"), (torch.float16, 64, 8, 8, 16, [90], "counter"),
    (torch.bfloat16, 128, 8, 2, 32, [500], "split"), (torch.float16, 128, 1, 1, 8, [45, 46], "split"),
    (torch.bfloat16, 64, 4, 3, 16, [6, 3], "split"),
]


@pytest.mark.parametrize("dt,D,group,Q,bs,ctx,plan", CASES)
def test_multi_query_attention_matches_fp64(cuda, dt, D, group, Q, bs, ctx, plan):
    d, meta, old_k, old_v, tables = setup(cuda, dt, D, group, Q, bs, ctx, plan)
    # reference: the library's own RoPE (bit-identical to the kernel's, checked below) then float64 attention
    qr, kr = d["qt"].clone(), d["kn"].clone()
    ops.apply_rotary_qk(qr, kr, d["cos"], d["sin"], d["pos"], is_neox=True)
    want_kc, want_vc = d["kc"].clone(), d["vc"].clone()
    paged_attn.reshape_and_cache_flashinfer(kr, d["vn"].clone(), want_kc, want_vc, d["slots"])
    if plan == "counter":
        lib().mrs_set_attn_flags(2)
    try:
        run("mrs_paged_decode_fused_multi", d, meta, Q)
    finally:
        lib().mrs_set_attn_flags(0)
    torch.cuda.synchronize()
    got = d["out"].float().cpu().numpy()
    assert np.isfinite(got).all()
    qn, kn, vn = qr.float().cpu().numpy(), kr.float().cpu().numpy(), d["vn"].float().cpu().numpy()
    tol = {torch.float16: 2.0 ** -9, torch.bfloat16: 3 * 2.0 ** -8}[dt]
    for b, c in enumerate(ctx):
        keys = np.concatenate([old_k[b].float().numpy(), kn[b * Q:(b + 1) * Q]])
        vals = np.concatenate([old_v[b].float().numpy(), vn[b * Q:(b + 1) * Q]])
        want = causal_ref(qn[b * Q:(b + 1) * Q], keys, vals, meta["scale"])
        err = np.abs(got[b * Q:(b + 1) * Q] - want).max() / np.abs(want).max()
        assert err <= tol, (b, err)
    # the cache rows it writes: bit-identical to rotary_embedding_positions + reshape_and_cache_flashinfer (NaN included)
    assert torch.equal(d["kc"].view(torch.int16), want_kc.view(torch.int16))
    assert torch.equal(d["vc"].view(torch.int16), want_vc.view(torch.int16))
    assert int(d["counters"].abs().sum()) == 0


@pytest.mark.parametrize("plan,ctx,D", [("unsplit", [50, 7], 128), ("split", [300], 128), ("split", [90, 40], 64)])
def test_q1_is_bit_identical_to_single_query_kernel(cuda, plan, ctx, D):
    outs = []
    for fn in ("mrs_paged_decode_fused", "mrs_paged_decode_fused_multi"):
        d, meta, *_ = setup(cuda, torch.bfloat16, D, 4, 1, 16, ctx, plan, seed=3)
        run(fn, d, meta, 1 if fn.endswith("multi") else None)
        torch.cuda.synchronize()
        outs.append((d["out"].clone(), d["kc"].clone(), d["vc"].clone()))
    for a, b in zip(*outs):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_graph_replay_matches_eager(cuda):
    d, meta, *_ = setup(cuda, torch.bfloat16, 128, 4, 4, 16, [200], "split", seed=5)
    run("mrs_paged_decode_fused_multi", d, meta, 4)
    torch.cuda.synchronize()
    eager = d["out"].clone()
    d["out"].zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run("mrs_paged_decode_fused_multi", d, meta, 4)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager, d["out"])
