"""Every decode and prompt attention entry point under score-shaped inputs (tests/attn_cases.py): rising, falling,
sink, needle, shifted by +-100 nats and poisoned (every position the kernel must not see scores 200 over every visible
key), against a float64 reference, element-wise within a bound computed from the inputs.  Covers split plans with a
sliding window or soft-cap, vLLM v2 with sinks, HND decode with GQA groups above 16, contexts up to 32768, the fused
decode kernels (unsplit, cluster merge, counter merge, strided QKV views, interleaved RoPE), the verify kernel with
poisoned future draft rows, and prompt attention up to a 4096-token prompt at 32 / 8 heads."""
import ctypes

import numpy as np
import pytest
import torch

import attn_cases as ac
from mistralrs_b200 import kv_index, lib, ops, paged_attn

pytestmark = pytest.mark.gpu

NAN = float("nan")


def _t(a, dev, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t.to(ac.TORCH_DT[dt]) if dt else t


def _check(what, got, want, st, dt, n, softcap=None):
    got = got.double().cpu().numpy() if torch.is_tensor(got) else got
    tol = ac.tolerance(want, st, dt, n, softcap)
    assert np.isfinite(got).all(), what
    r = ac.err_ratio(got, want, tol)
    assert r <= 1.0, (what, r)
    return r


def _profiles(needles):
    for prof in ac.PROFILES:
        if prof == "needle":
            for j in needles:
                yield prof, j
        else:
            yield prof, None


# ---------------------------------------------------------------- decode problems over the HND / vLLM caches
def _decode_problem(rng, prof, ctx, H, KVH, D, dt, window_left=None, needle=None, poison_v=ac.POISON_V):
    """Per sequence: q [H, D], k / v [ctx, KVH, D] rounded to dt, visible mask; plus the fill rows for every cache slot
    no sequence owns (poison rows under 'poison', NaN otherwise)."""
    scale = D ** -0.5
    seqs = []
    for b, c in enumerate(ctx):
        j = np.arange(c)
        lo = max(0, c - 1 - window_left) if window_left is not None else 0
        vis = j >= lo
        q = ac.round_to(ac.make_queries(rng, prof, H, KVH, D, scale), dt)
        nd = None if needle is None else min(needle, c - 1) if needle != "win_lo" else lo
        t = ac.target_scores(prof, c, vis, nd)
        k = ac.make_keys(rng, prof, q, KVH, t, scale)
        v = ac.make_values(rng, c, KVH, D, vis, prof == "poison", poison_v)
        seqs.append((q, k, v, vis))
    if prof == "poison":
        fk, fv = ac.poison_rows(rng, seqs[0][0], KVH, 60.0, scale, poison_v)
    else:
        fk, fv = np.full((KVH, D), NAN, np.float32), np.full((KVH, D), NAN, np.float32)
    return seqs, fk, fv, scale


def _to_cache(x, cache_dt, qdt, scale_f):
    """numpy rows -> the dtype the cache stores, and their values as the kernel reads them (float32)"""
    if cache_dt == "fp8":
        t = (torch.from_numpy(x) / scale_f).to(torch.float8_e4m3fn)
        return t, t.float().numpy() * scale_f
    t = torch.from_numpy(x).to(ac.TORCH_DT[qdt])
    return t, t.float().numpy()


def _hnd_cache(dev, rng, seqs, fk, fv, page, KVH, D, dt, cache_dt=None, k_scale=1.0, v_scale=1.0, extra=3):
    """HND cache [NB, KVH, page, D]: each sequence's pages drawn from a shuffled pool, every other slot (stale rows of
    each last page, pages nobody owns) holding the fill rows.  Returns caches, tables, and each sequence's k / v as the
    kernel reads them (after the cache's rounding)."""
    npg = [-(-len(s[1]) // page) for s in seqs]
    NB = sum(npg) + extra
    perm = rng.permutation(NB)
    kc = np.ascontiguousarray(np.broadcast_to(fk[None, :, None, :], (NB, KVH, page, D)), dtype=np.float32)
    vc = np.ascontiguousarray(np.broadcast_to(fv[None, :, None, :], (NB, KVH, page, D)), dtype=np.float32)
    tables, o = [], 0
    for (q, k, v, vis), n in zip(seqs, npg):
        t = perm[o:o + n]; o += n
        tables.append([int(x) for x in t])
        j = np.arange(len(k))
        kc[t[j // page], :, j % page] = k
        vc[t[j // page], :, j % page] = v
    kt, kr = _to_cache(kc, cache_dt, dt, k_scale)
    vt, vr = _to_cache(vc, cache_dt, dt, v_scale)
    ks = [kr[np.array(t)[np.arange(len(s[1])) // page], :, np.arange(len(s[1])) % page] for t, s in zip(tables, seqs)]
    vs = [vr[np.array(t)[np.arange(len(s[1])) // page], :, np.arange(len(s[1])) % page] for t, s in zip(tables, seqs)]
    spare = [int(x) for x in perm[o:]]
    return kt.to(dev), vt.to(dev), tables, ks, vs, spare


def _decode_ref(seqs, ks, vs, scale, softcap=None, sinks=None):
    out = []
    for (q, _, _, vis), k, v in zip(seqs, ks, vs):
        out.append(ac.reference(q[None], k, v, scale, vis[None], softcap, sinks))
    return out


def _plan(tables, ctx, page, split, KVH):
    """split: None (unsplit), 'planner' (the serving planner's chunk), or pages per tile"""
    if split == "planner":
        split = kv_index.decode_split_pages(page, len(ctx), KVH, max(ctx))
    ntiles = sum(1 if not split else -(-max(-(-c // page), 1) // split) for c in ctx)
    padded = ntiles + (2 if split else 0)        # graph padding tiles, mask 0
    return split, padded, kv_index.make_paged_kv_decode_tensors(tables, ctx, page, split, padded)


def _flashinfer(dev, q, kc, vc, tables, ctx, page, split, scale, window_left=None, softcap=None, k_scale=1.0, v_scale=1.0):
    indptr, indices, last = kv_index.make_paged_kv_tensors(tables, ctx, page, sum(len(t) for t in tables))
    split, padded, (req, tile, o_indptr, chunk, mask) = _plan(tables, ctx, page, split, kc.shape[1])
    d = lambda a: _t(a, dev)
    return paged_attn.flashinfer_decode(q, kc, vc, d(indptr), d(indices), d(last), d(req), d(tile), d(o_indptr), d(chunk),
                                        d(mask), scale, window_left=window_left, logits_soft_cap=softcap,
                                        k_scale=k_scale, v_scale=v_scale)


HND_CASES = [  # (dt, D, KVH, group, page, ctx, splits, flags, cache)
    ("bf16", 128, 2, 4, 16, [300, 1100], (None, 4, "planner"), 0, None),
    ("f16", 64, 2, 8, 16, [700, 37], (None, 4), 0, None),
    ("bf16", 128, 1, 1, 32, [520], (None, 2), 0, None),
    ("f16", 128, 1, 24, 16, [400], (None, 4), 0, None),
    ("bf16", 64, 1, 32, 8, [333, 90], (None, 8), 0, None),
    ("f16", 256, 2, 4, 16, [300], (None, 4), 1, None),          # SIMT kernel
    ("f32", 128, 2, 4, 16, [300], (None, 4), 1, None),
    ("bf16", 128, 2, 4, 16, [300, 45], (None, 4), 0, "fp8"),     # FP8 cache: SIMT kernel
]


@pytest.mark.parametrize("case", HND_CASES, ids=lambda c: f"{c[0]}-D{c[1]}-g{c[3]}-p{c[4]}-f{c[7]}-{c[8]}")
def test_flashinfer_decode_profiles(cuda, case):
    dt, D, KVH, group, page, ctx, splits, flags, cache = case
    H = KVH * group
    ks_, vs_ = (0.1, 0.04) if cache == "fp8" else (1.0, 1.0)
    worst = 0.0
    lib().mrs_set_attn_flags(flags)
    try:
        for i, (prof, nd) in enumerate(_profiles([0, page - 1, page, 4 * page, 10 ** 9])):
            rng = np.random.default_rng(i)
            seqs, fk, fv, scale = _decode_problem(rng, prof, ctx, H, KVH, D, dt, needle=nd,
                                                  poison_v=16.0 if cache == "fp8" else ac.POISON_V)
            kc, vc, tables, ks, vs, _ = _hnd_cache(cuda, rng, seqs, fk, fv, page, KVH, D, dt, cache, ks_, vs_)
            refs = _decode_ref(seqs, ks, vs, scale)
            q = _t(np.stack([s[0] for s in seqs]), cuda, dt)
            for split in splits:
                got = _flashinfer(cuda, q, kc, vc, tables, ctx, page, split, scale, k_scale=ks_, v_scale=vs_)
                torch.cuda.synchronize()
                for b, (o, st) in enumerate(refs):
                    worst = max(worst, _check((prof, nd, split, b), got[b:b + 1].float().cpu().numpy(), o, st, dt, ctx[b]))
    finally:
        lib().mrs_set_attn_flags(0)
    print(f"\nflashinfer_decode {case}: worst err/tol {worst:.3f}")


@pytest.mark.parametrize("flags", [0, 1])
def test_flashinfer_decode_split_window_and_softcap(cuda, flags):
    """window_left and soft-cap in split plans: tiles wholly outside the window leave a partial with lse -inf"""
    dt, D, KVH, group, page, ctx = "bf16", 128, 2, 4, 16, [700, 300]
    H = KVH * group
    worst = 0.0
    lib().mrs_set_attn_flags(flags)
    try:
        for i, (prof, nd) in enumerate(_profiles(["win_lo", 699])):
            for window_left, softcap in ((100, None), (255, None), (None, 30.0), (100, 30.0)):
                rng = np.random.default_rng(10 * i + (window_left or 0))
                seqs, fk, fv, scale = _decode_problem(rng, prof, ctx, H, KVH, D, dt, window_left, nd)
                kc, vc, tables, ks, vs, _ = _hnd_cache(cuda, rng, seqs, fk, fv, page, KVH, D, dt)
                q = _t(np.stack([s[0] for s in seqs]), cuda, dt)
                refs = _decode_ref(seqs, ks, vs, scale, softcap)
                for split in (None, 4, 2):
                    got = _flashinfer(cuda, q, kc, vc, tables, ctx, page, split, scale, window_left, softcap)
                    torch.cuda.synchronize()
                    for b, (o, st) in enumerate(refs):
                        worst = max(worst, _check((prof, nd, window_left, softcap, split, b), got[b:b + 1].float().cpu().numpy(),
                                                  o, st, dt, ctx[b], softcap))
    finally:
        lib().mrs_set_attn_flags(0)
    print(f"\nflashinfer_decode split + window / softcap, flags {flags}: worst err/tol {worst:.3f}")


def test_flashinfer_decode_32k_context(cuda):
    """A 32768-token context at 32 / 8 heads through the serving planner (batch 1 and 2)"""
    dt, D, KVH, group, page = "bf16", 128, 8, 4, 16
    H = KVH * group
    worst = 0.0
    for ctx in ([32768], [32768, 5000]):
        split = kv_index.decode_split_pages(page, len(ctx), KVH, max(ctx))
        profs = [("ramp_up", None), ("poison", None), ("shift-100", None), ("needle", split * page),
                 ("normal", None)] if len(ctx) == 1 else [("ramp_down", None)]
        for i, (prof, nd) in enumerate(profs):
            rng = np.random.default_rng(100 + i)
            seqs, fk, fv, scale = _decode_problem(rng, prof, ctx, H, KVH, D, dt, needle=nd)
            kc, vc, tables, ks, vs, _ = _hnd_cache(cuda, rng, seqs, fk, fv, page, KVH, D, dt)
            q = _t(np.stack([s[0] for s in seqs]), cuda, dt)
            got = _flashinfer(cuda, q, kc, vc, tables, ctx, page, "planner", scale)
            for b in range(len(ctx)):      # float64 on the device: the whole context is visible to the one query row
                o, st = _prompt_ref(q[b:b + 1], _t(ks[b], cuda), _t(vs[b], cuda), scale, False)
                worst = max(worst, _prompt_check((ctx, prof, nd, b), got[b:b + 1], o, st, dt, ctx[b]))
            del kc, vc
    print(f"\nflashinfer_decode 32k: worst err/tol {worst:.3f}")


# ---------------------------------------------------------------- vLLM paged_attention v1 / v2
def _vllm_cache(kc, vc, dt):
    """HND [NB, KVH, BS, D] -> vLLM K [NB, KVH, D/x, BS, x], V [NB, KVH, D, BS]"""
    NB, KVH, BS, D = kc.shape
    x = 16 // kc.element_size()
    return (kc.reshape(NB, KVH, BS, D // x, x).permute(0, 1, 3, 2, 4).contiguous(),
            vc.permute(0, 1, 3, 2).contiguous())


@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_vllm_paged_attention_profiles(cuda, dt):
    """v1 (one partition) and v2 (512-token partitions merged by merge_partials_kernel), with sinks that sit near the
    top score or dominate it, soft-cap, needles at 511 / 512, and padded block-table entries on a poisoned page"""
    D, KVH, group, BS = 128, 2, 4, 16
    H = KVH * group
    worst = {"v1": 0.0, "v2": 0.0}
    for i, (prof, nd) in enumerate(_profiles([0, 511, 512, 10 ** 9])):
        for ctx, ver in (([300, 512], "v1"), ([1100, 600, 513], "v2")):
            rng = np.random.default_rng(7 * i + len(ctx))
            seqs, fk, fv, scale = _decode_problem(rng, prof, ctx, H, KVH, D, dt, needle=nd)
            kc, vc, tables, ks, vs, spare = _hnd_cache(cuda, rng, seqs, fk, fv, BS, KVH, D, dt)
            kv, vv = _vllm_cache(kc, vc, dt)
            width = max(len(t) for t in tables) + 2
            bt = np.array([t + [spare[0]] * (width - len(t)) for t in tables], dtype=np.int32)   # padding: a page nobody owns
            q = _t(np.stack([s[0] for s in seqs]), cuda, dt)
            top = {"shift+100": 100.0, "shift-100": -100.0, "ramp_up": 60.0, "ramp_down": 60.0, "needle": 45.0}.get(prof, 3.0)
            for sinks, softcap in ((None, None), (np.full(H, top, np.float32), None),
                                   (np.full(H, top + 20.0, np.float32), None), (None, 30.0)):
                max_ctx = 512 if ver == "v1" else 4096
                got = paged_attn.paged_attention(q, None, None, kv, vv, _t(bt, cuda), _t(np.array(ctx, np.int32), cuda), None,
                                                 max_ctx, scale, softcapping=softcap or 1.0,
                                                 sinks=None if sinks is None else _t(sinks, cuda)).float().cpu().numpy()
                for b, (o, st) in enumerate(_decode_ref(seqs, ks, vs, scale, softcap, sinks)):
                    worst[ver] = max(worst[ver], _check((ver, prof, nd, sinks is not None and sinks[0], softcap, b),
                                                        got[b:b + 1], o, st, dt, ctx[b], softcap))
    print(f"\npaged_attention {dt}: worst err/tol {worst}")


# ---------------------------------------------------------------- fused decode (RoPE + cache write + attention + merge)
def _ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _fused_setup(dev, rng, prof, dt, D, KVH, group, Q, page, ctx, plan, needle=None, interleaved=False):
    """ctx: per-sequence kv_len including the Q new rows.  Queries share a low-frequency direction so every verify row
    sees nearly the same scores; cached keys are built from q after the library's own RoPE, new keys from the raw q
    (RoPE keeps q.k)."""
    B, H = len(ctx), KVH * group
    scale = D ** -0.5
    tdt = ac.TORCH_DT[dt]
    max_pos = max(ctx) + 8
    inv = 1.0 / (10000.0 ** (np.arange(0, D, 2) / D))
    fr = np.arange(max_pos)[:, None] * inv[None, :]
    cos, sin = _t(np.cos(fr), dev).to(tdt), _t(np.sin(fr), dev).to(tdt)
    pos = np.array([c - Q + i for c in ctx for i in range(Q)], np.int32)
    q_raw = []
    for b in range(B):
        q0 = ac.make_queries(rng, prof, H, KVH, D, scale, low_freq=True)
        q_raw += [q0 + (0.1 * rng.standard_normal(q0.shape) if i else 0) for i in range(Q)]
    q_raw = ac.round_to(np.stack(q_raw), dt)                                          # [B * Q, H, D]
    qr = _t(q_raw, dev, dt)
    dummy = torch.zeros(B * Q, KVH, D, dtype=tdt, device=dev)
    ops.apply_rotary_qk(qr, dummy, cos, sin, _t(pos, dev), is_neox=not interleaved)
    q_rot = qr.float().cpu().numpy()
    seqs, k_new, v_new = [], [], []
    for b, c in enumerate(ctx):
        j = np.arange(c)
        t = ac.target_scores(prof, c, np.ones(c, bool), None if needle is None else min(needle, c - 1))
        if prof == "poison":           # draft row j scores 20 j over draft row j - 1: row i must not see rows after i
            t[c - Q:] = 210.0 + 20.0 * np.arange(Q)
        kc_b = ac.make_keys(rng, prof, q_rot[b * Q:(b + 1) * Q].mean(0), KVH, t[:c - Q], scale)
        kn_b = ac.make_keys(rng, prof, q_raw[b * Q:(b + 1) * Q].mean(0), KVH, t[c - Q:], scale)
        v_b = ac.make_values(rng, c, KVH, D)
        seqs.append((ac.round_to(kc_b, dt), ac.round_to(v_b, dt)))
        k_new.append(ac.round_to(kn_b, dt)); v_new.append(v_b[c - Q:])
    if prof == "poison":
        fk, fv = ac.poison_rows(rng, q_rot[:1].mean(0).reshape(H, D), KVH, 500.0, scale)
    else:
        fk, fv = np.full((KVH, D), NAN, np.float32), np.full((KVH, D), NAN, np.float32)
    # cache: the cached rows of each sequence; its new rows' slots and every slot nobody owns hold the fill rows
    cache_seqs = [(None, np.concatenate([k, np.broadcast_to(fk, (Q, KVH, D))]), np.concatenate([v[:len(v) - Q],
                   np.broadcast_to(fv, (Q, KVH, D))]), None) for (k, v) in seqs]
    kc, vc, tables, _, _, _ = _hnd_cache(dev, rng, cache_seqs, fk, fv, page, KVH, D, dt)
    nblk = [len(t) for t in tables]
    slots = np.array([tables[b][p // page] * page + p % page for b in range(B) for p in range(ctx[b] - Q, ctx[b])], np.int64)
    indptr, indices, last = kv_index.make_paged_kv_tensors(tables, ctx, page, sum(nblk))
    split = {"unsplit": None, "split": -(-max(nblk) // 4), "counter": -(-max(nblk) // 4), "many": 1}[plan]
    padded = B if split is None else sum(-(-n // split) for n in nblk)
    req, tile, o_indptr, chunk, mask = kv_index.make_paged_kv_decode_tensors(tables, ctx, page, split, padded)
    T = lambda a, d=torch.int32: torch.as_tensor(np.asarray(a)).to(d).to(dev)
    d = dict(q=_t(q_raw, dev, dt), kn=_t(np.stack([r for k in k_new for r in k]), dev, dt),
             vn=_t(np.stack([r for v in v_new for r in v]), dev, dt), kc=kc, vc=vc, cos=cos, sin=sin, pos=T(pos),
             slots=T(slots, torch.int64), indptr=T(indptr), indices=T(indices), last=T(last), req=T(req), tile=T(tile),
             o_indptr=T(o_indptr), chunk=T(chunk), mask=T(mask, torch.uint8),
             out=torch.zeros(B * Q, H, D, dtype=tdt, device=dev),
             tmp_v=None if split is None else torch.zeros(padded, Q * H, D, dtype=tdt, device=dev),
             tmp_s=None if split is None else torch.zeros(padded, Q * H, dtype=torch.float32, device=dev),
             counters=torch.zeros(B * KVH * -(-group * Q // 16), dtype=torch.int32, device=dev))
    meta = dict(B=B, padded=padded, H=H, KVH=KVH, D=D, page=page, scale=scale, dt=dt, Q=Q, interleaved=interleaved)
    return d, meta, seqs


def _fused_call(d, m, fn, qkv=None):
    common = [_ptr(d["kc"]), _ptr(d["vc"]), _ptr(d["cos"]), _ptr(d["sin"]), _ptr(d["pos"]), _ptr(d["slots"]),
              _ptr(d["indptr"]), _ptr(d["indices"]), _ptr(d["last"]), _ptr(d["req"]), _ptr(d["tile"]), _ptr(d["o_indptr"]),
              _ptr(d["chunk"]), _ptr(d["mask"]), _ptr(d["out"]), _ptr(d["tmp_v"]), _ptr(d["tmp_s"]), _ptr(d["counters"]),
              m["B"], m["padded"], m["H"], m["KVH"], m["D"], m["page"], ctypes.c_float(m["scale"]),
              ctypes.c_uint32({"f16": 0, "bf16": 1}[m["dt"]]), 2 if m["interleaved"] else 0]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if fn == "strided":
        q, k, v = qkv
        rc = lib().mrs_paged_decode_fused_strided(_ptr(q), _ptr(k), _ptr(v), *common, ctypes.c_int64(q.stride(0)),
                                                  ctypes.c_int64(k.stride(0)), st)
    elif fn == "multi":
        rc = lib().mrs_paged_decode_fused_multi(_ptr(d["q"]), _ptr(d["kn"]), _ptr(d["vn"]), *common, m["Q"], st)
    else:
        rc = lib().mrs_paged_decode_fused(_ptr(d["q"]), _ptr(d["kn"]), _ptr(d["vn"]), *common, st)
    assert rc == 0, rc


def _fused_check(what, d, m, seqs, fn, ctx, flags=0):
    dev = d["q"].device
    Q = m["Q"]
    qr, kr = d["q"].clone(), d["kn"].clone()
    ops.apply_rotary_qk(qr, kr, d["cos"], d["sin"], d["pos"], is_neox=not m["interleaved"])
    want_kc, want_vc = d["kc"].clone(), d["vc"].clone()
    paged_attn.reshape_and_cache_flashinfer(kr, d["vn"].clone(), want_kc, want_vc, d["slots"])
    qkv = None
    if fn == "strided":      # q, k_new, v_new as views into one fused-QKV row [B, (H + 2 KVH) D]
        H, KVH, D = m["H"], m["KVH"], m["D"]
        row = torch.cat([d["q"].reshape(m["B"], -1), d["kn"].reshape(m["B"], -1), d["vn"].reshape(m["B"], -1)], 1).contiguous()
        qkv = (row[:, :H * D], row[:, H * D:(H + KVH) * D], row[:, (H + KVH) * D:])
    lib().mrs_set_attn_flags(flags)
    try:
        _fused_call(d, m, fn, qkv)
    finally:
        lib().mrs_set_attn_flags(0)
    torch.cuda.synchronize()
    got = d["out"].double().cpu().numpy()
    qn, kn, vn = qr.float().cpu().numpy(), kr.float().cpu().numpy(), d["vn"].float().cpu().numpy()
    worst = 0.0
    for b, c in enumerate(ctx):
        keys = np.concatenate([seqs[b][0], kn[b * Q:(b + 1) * Q]])
        vals = np.concatenate([seqs[b][1][:c - Q], vn[b * Q:(b + 1) * Q]])
        mask = np.arange(c)[None, :] <= (c - Q + np.arange(Q))[:, None]
        o, st = ac.reference(qn[b * Q:(b + 1) * Q], keys, vals, m["scale"], mask)
        worst = max(worst, _check((what, b), got[b * Q:(b + 1) * Q], o, st, m["dt"], c))
    # the cache rows the kernel writes: bit-identical to rotary_embedding_positions + reshape_and_cache_flashinfer
    assert torch.equal(d["kc"].view(torch.int16), want_kc.view(torch.int16)), what
    assert torch.equal(d["vc"].view(torch.int16), want_vc.view(torch.int16)), what
    assert int(d["counters"].abs().sum()) == 0, what
    return worst


FUSED_CASES = [  # (dt, D, KVH, group, page, ctx, plan, flags, fn, interleaved)
    ("bf16", 128, 2, 4, 16, [300], "unsplit", 0, "fused", False),
    ("bf16", 128, 2, 4, 16, [300], "split", 0, "fused", False),            # cluster merge (batch 1, 4 tiles)
    ("f16", 128, 2, 4, 16, [300], "split", 2, "fused", False),             # counter merge (flag 2)
    ("f16", 64, 2, 8, 16, [700, 45, 300], "split", 0, "fused", False),     # counter merge (batch 3)
    ("bf16", 128, 2, 4, 16, [1100], "many", 0, "fused", False),            # counter merge (69 tiles)
    ("bf16", 128, 2, 4, 16, [300, 77], "split", 0, "fused", True),         # interleaved RoPE
    ("bf16", 128, 8, 4, 16, [600, 40], "split", 0, "strided", False),      # GPTQ decode step's call
    ("f16", 64, 2, 4, 8, [129], "unsplit", 0, "strided", True),
]


@pytest.mark.parametrize("case", FUSED_CASES, ids=lambda c: f"{c[8]}-{c[0]}-D{c[1]}-{c[6]}-f{c[7]}-il{int(c[9])}")
def test_fused_decode_profiles(cuda, case):
    dt, D, KVH, group, page, ctx, plan, flags, fn, il = case
    worst = 0.0
    for i, (prof, nd) in enumerate(_profiles([0, page, 64, min(ctx) - 2, min(ctx) - 1])):   # min(ctx) - 1: the new token
        rng = np.random.default_rng(50 + i)
        d, m, seqs = _fused_setup(cuda, rng, prof, dt, D, KVH, group, 1, page, ctx, plan, nd, il)
        worst = max(worst, _fused_check((prof, nd), d, m, seqs, fn, ctx, flags))
    print(f"\nmrs_paged_decode_{fn} {case}: worst err/tol {worst:.3f}")


MULTI_CASES = [  # (dt, D, KVH, group, Q, page, ctx, plan, flags)
    ("bf16", 128, 2, 4, 4, 16, [300], "split", 0),       # cluster
    ("f16", 128, 2, 4, 3, 16, [77, 5, 200], "split", 0),  # counter (batch 3)
    ("bf16", 64, 2, 8, 8, 8, [90], "counter", 2),          # counter, 4 sub-tiles of 16 rows
    ("f16", 64, 2, 1, 7, 32, [70], "unsplit", 0),
    ("bf16", 128, 2, 4, 1, 16, [1100], "many", 0),
]


@pytest.mark.parametrize("case", MULTI_CASES, ids=lambda c: f"{c[0]}-D{c[1]}-g{c[3]}-q{c[4]}-{c[7]}")
def test_fused_multi_query_profiles(cuda, case):
    """Verify attention: under 'poison' draft row j scores 20 j above draft row j - 1 and 200 above every cached key,
    so a row that sees a later draft row returns that row's V; needles on the first and last draft rows"""
    dt, D, KVH, group, Q, page, ctx, plan, flags = case
    worst = 0.0
    c0 = min(ctx)
    for i, (prof, nd) in enumerate(_profiles([0, c0 - Q, c0 - 1, page])):
        rng = np.random.default_rng(80 + i)
        d, m, seqs = _fused_setup(cuda, rng, prof, dt, D, KVH, group, Q, page, ctx, plan, nd)
        worst = max(worst, _fused_check((prof, nd), d, m, seqs, "multi", ctx, flags))
    print(f"\nmrs_paged_decode_fused_multi {case}: worst err/tol {worst:.3f}")


# ---------------------------------------------------------------- prompt attention
def _tc(enable):
    lib().mrs_prefill_attn_tc_debug(ctypes.c_int32(enable), ctypes.c_uint32(0), ctypes.c_uint32(0))


def _prompt_problem(rng, prof, Tq, L, H, KVH, D, dt, causal=True, window_left=None, needle=None):
    """q [Tq, H, D] at positions L - Tq .. L - 1 over keys [L, KVH, D].  Every row shares its KV head's direction, so
    the per-key profile holds for every row that sees the key.  'poison' adds, for a spread of rows r, a key in r's
    causal future (offsets 1, 2, 17, 63) and, with a window, the key just outside it, that score 200 over everything
    r sees: each on its own direction w_r orthogonal to the rest, so no other row notices it."""
    scale = D ** -0.5
    q0 = ac.make_queries(rng, prof, H, KVH, D, scale)
    q = q0[None] + (0.1 * rng.standard_normal((Tq, H, D)) if prof != "normal" else rng.standard_normal((Tq, H, D)) - q0[None])
    t = ac.target_scores(prof if prof != "poison" else "normal", L, np.ones(L, bool), needle)
    k = ac.make_keys(rng, prof, q0, KVH, t, scale)
    v = ac.make_values(rng, L, KVH, D)
    if prof == "poison":
        off = L - Tq
        g = H // KVH
        # per KV head an orthonormal basis whose first vector is the head's direction u: w_n = basis[:, n + 1]
        basis = [np.linalg.qr(np.column_stack([q0[kvh * g:(kvh + 1) * g].mean(0), rng.standard_normal((D, D - 1))]))[0]
                 for kvh in range(KVH)]
        pairs = []
        for r in np.unique(np.linspace(0, Tq - 2, 24).astype(int)):
            for dj in ((1, 2, 17, 63) if causal else ()):
                if r + off + dj < L:
                    pairs.append((r, r + off + dj))
            if window_left is not None and r + off - window_left - 1 >= 0:
                pairs.append((r, r + off - window_left - 1))
        pairs = pairs[:D // 2]
        a = ac.SCORE_GAIN / scale
        for n, (r, j) in enumerate(pairs):
            for kvh in range(KVH):
                w = basis[kvh][:, n + 1]
                q[r, kvh * g:(kvh + 1) * g] += a * w
                k[j, kvh] += 210.0 / (scale * a) * w
            v[j] = 30.0 * np.sign(v[j])
    return ac.round_to(q, dt), ac.round_to(k, dt), ac.round_to(v, dt), scale


def _prompt_ref(q, k, v, scale, causal, window_left=None, softcap=None):
    """fp64 on the device, one head at a time; s2 (sum p |v - o|) is bounded by s1 + |o|.  Returns (o, tol input dict)"""
    Tq, H, D = q.shape
    L, KVH = k.shape[0], k.shape[1]
    g = H // KVH
    pos = torch.arange(Tq, device=q.device)[:, None] + (L - Tq)
    j = torch.arange(L, device=q.device)[None, :]
    mask = torch.ones(Tq, L, dtype=torch.bool, device=q.device)
    if causal:
        mask &= j <= pos
    if window_left is not None:
        mask &= j >= pos - window_left
    o = torch.empty(Tq, H, D, dtype=torch.float64, device=q.device)
    s1, fl = torch.empty_like(o), torch.empty_like(o)
    qk = torch.empty(Tq, H, dtype=torch.float64, device=q.device)
    for h in range(H):
        qh, kh, vh = q[:, h].double(), k[:, h // g].double(), v[:, h // g].double()
        s = qh @ kh.T * scale
        if softcap:
            s = softcap * torch.tanh(s / softcap)
        p = torch.softmax(s.masked_fill(~mask, float("-inf")), dim=-1)
        o[:, h] = p @ vh
        s1[:, h] = p @ vh.abs()
        fl[:, h] = torch.where(p < np.exp(-80.0), p, 0.0) @ vh.abs()
        qk[:, h] = ((qh.abs() @ kh.abs().T) * scale).masked_fill(~mask, 0.0).amax(1)
    return o, dict(s1=s1, s2=s1 + o.abs(), flush=fl, qk=qk)


def _prompt_check(what, got, o, st, dt, n, softcap=None):
    assert torch.isfinite(got).all(), what
    tol = ac.tolerance(o, st, dt, n, softcap)
    r = ((got.double() - o).abs() / tol).max().item()
    assert r <= 1.0, (what, r)
    return r


PROMPT_CASES = [  # (dt, D, T, H, KVH, tc)
    ("bf16", 128, 700, 8, 2, 1), ("f16", 128, 333, 4, 4, 1), ("bf16", 128, 700, 8, 2, 0), ("f16", 64, 520, 8, 2, 1),
]


@pytest.mark.parametrize("case", PROMPT_CASES, ids=lambda c: f"{c[0]}-D{c[1]}-T{c[2]}-tc{c[5]}")
def test_prefill_attention_profiles(cuda, case):
    dt, D, T, H, KVH, tc = case
    worst = 0.0
    try:
        _tc(tc)
        for i, (prof, nd) in enumerate(_profiles([0, 63, 64, 128, T - 1])):
            for causal, window_left, softcap in ((True, None, None), (False, None, None), (True, 100, None), (True, None, 30.0)):
                rng = np.random.default_rng(i * 13 + (window_left or 0))
                q, k, v, scale = _prompt_problem(rng, prof, T, T, H, KVH, D, dt, causal, window_left, nd)
                qt, kt, vt = _t(q, cuda, dt), _t(k, cuda, dt), _t(v, cuda, dt)
                got = paged_attn.prefill_attention(qt, kt, vt, scale, causal=causal, window_left=window_left, softcap=softcap)
                o, st = _prompt_ref(qt, kt, vt, scale, causal, window_left, softcap)
                worst = max(worst, _prompt_check((prof, nd, causal, window_left, softcap), got, o, st, dt, T, softcap))
    finally:
        _tc(1)
    print(f"\nprefill_attention {case}: worst err/tol {worst:.3f}")


def test_prefill_attention_4096_prompt(cuda):
    """Config 3's shape: a 4096-token prompt at 32 / 8 heads, head 128 (the wgmma kernel), 32 K/V tiles per row"""
    dt, D, T, H, KVH = "bf16", 128, 4096, 32, 8
    worst = 0.0
    for i, prof in enumerate(("ramp_up", "poison")):
        rng = np.random.default_rng(400 + i)
        q, k, v, scale = _prompt_problem(rng, prof, T, T, H, KVH, D, dt)
        qt, kt, vt = _t(q, cuda, dt), _t(k, cuda, dt), _t(v, cuda, dt)
        got = paged_attn.prefill_attention(qt, kt, vt, scale)
        o, st = _prompt_ref(qt, kt, vt, scale, True)
        worst = max(worst, _prompt_check(prof, got, o, st, dt, T))
    print(f"\nprefill_attention T=4096: worst err/tol {worst:.3f}")


def test_prefill_attention_varlen_batch(cuda):
    dt, D, H, KVH = "bf16", 128, 8, 2
    lens = [5, 130, 64, 257]
    worst = 0.0
    for i, prof in enumerate(("ramp_up", "ramp_down", "poison", "shift+100", "shift-100")):
        rng = np.random.default_rng(500 + i)
        parts = [_prompt_problem(rng, prof, L, L, H, KVH, D, dt) for L in lens]
        scale = parts[0][3]
        qt, kt, vt = (_t(np.concatenate([p[x] for p in parts]), cuda, dt) for x in range(3))
        cu = _t(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32), cuda)
        got = paged_attn.prefill_attention(qt, kt, vt, scale, cu_seqlens=cu, max_seqlen=max(lens))
        off = 0
        for L in lens:
            o, st = _prompt_ref(qt[off:off + L], kt[off:off + L], vt[off:off + L], scale, True)
            worst = max(worst, _prompt_check((prof, L), got[off:off + L], o, st, dt, L))
            off += L
    print(f"\nprefill_attention var-len: worst err/tol {worst:.3f}")


@pytest.mark.parametrize("page", [8, 16, 32])
@pytest.mark.parametrize("D,tc", [(128, 1), (128, 0), (64, 1)])
def test_prefill_attention_paged_profiles(cuda, page, D, tc):
    """New rows over a cached prefix in shuffled pages: needles on page boundaries of the prefix, and under 'poison' the
    stale rows of each last page, every page nobody owns and the padded table entries hold keys 200 over everything"""
    dt, H, KVH = "bf16", 8, 2
    cached, qlens = [300, 0, 17], [129, 40, 7]
    worst = 0.0
    try:
        _tc(tc)
        for i, (prof, nd) in enumerate(_profiles([0, page - 1, page, 2 * page, 299])):
            rng = np.random.default_rng(600 + i + page)
            probs = [_prompt_problem(rng, prof, ql, c + ql, H, KVH, D, dt, needle=min(nd, c + ql - 1) if nd is not None else None)
                     for c, ql in zip(cached, qlens)]
            scale = probs[0][3]
            if prof == "poison":
                fk, fv = ac.poison_rows(rng, probs[0][0].mean(0), KVH, 60.0, scale)
            else:
                fk, fv = np.full((KVH, D), NAN, np.float32), np.full((KVH, D), NAN, np.float32)
            seqs = [(None, p[1], p[2], None) for p in probs]
            kc, vc, tables, _, _, spare = _hnd_cache(cuda, rng, seqs, fk, fv, page, KVH, D, dt, extra=4)
            width = max(len(t) for t in tables) + 3
            bt = _t(np.array([t + [spare[0]] * (width - len(t)) for t in tables], np.int32), cuda)
            kv_lens = [c + ql for c, ql in zip(cached, qlens)]
            qt = _t(np.concatenate([p[0] for p in probs]), cuda, dt)
            cu_q = _t(np.concatenate([[0], np.cumsum(qlens)]).astype(np.int32), cuda)
            cu_k = _t(np.concatenate([[0], np.cumsum(kv_lens)]).astype(np.int32), cuda)
            for causal in (True, False):
                got = paged_attn.prefill_attention_paged(qt, kc, vc, bt, cu_q, cu_k, max(qlens), max(kv_lens), scale, causal=causal)
                off = 0
                for b, p in enumerate(probs):
                    kk, vv = _t(p[1], cuda, dt), _t(p[2], cuda, dt)
                    o, st = _prompt_ref(qt[off:off + qlens[b]], kk, vv, scale, causal)
                    worst = max(worst, _prompt_check((prof, nd, causal, b), got[off:off + qlens[b]], o, st, dt, kv_lens[b]))
                    off += qlens[b]
    finally:
        _tc(1)
    print(f"\nprefill_attention_paged page {page} D {D} tc {tc}: worst err/tol {worst:.3f}")
