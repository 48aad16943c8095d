"""Decode GEMV (mmvq.cu) at the launch shapes of the Llama-3-8B decode chain, where the kernel takes paths the
small-shape tests in test_mmvq_gpu.py never reach:

* clamped grids: more passes than `ctas_per_sm x SMs` CTAs, so every CTA owns `vrows * cta / ncta` rows, a range
  that is not a whole number of 16-row (GLU: 8-row) passes, and its last pass runs with padding slots;
* the two-type QKV grid (q||k Q4_K, v Q6_K) cut down to one wave;
* the one-CTA-per-SM plan with a deeper ring (long K at batch 5-8);
* the long-segment variant (UPL x 2) of a >= 128 MiB lm_head, at its default threshold;
* the fused RMSNorm -> Q8_1 prologue in every activation dtype, past the register-resident chunks (K > 4096);
* batch columns in the NCOLS = 4 / 8 instantiations, and weights whose address breaks the type's alignment.

Every launch goes through the public entries (`mrs_mmvq_fused`, `mrs_mmvq_fused_qkv_mixed`) with the default plan:
the process-wide switches are not touched, so the three-CTA-per-SM plan (reachable only through
`mrs_set_mmvq_ctas_per_sm`) is not tested here.  `_plan` restates the host planning rule of mmvq.cu, and each test
asserts that its launch takes the path it is meant to.

Oracle checks feed the kernel the oracle's own Q8_1 bytes, so the exact value `oracle.mmvq_q8_1` differs from the
kernel's only by f32 summation order (at most 5e-6 of the largest output) and by the output rounding.  Every element
must lie between the kernel's epilogue applied to y - delta and to y + delta: within the summation allowance of the
exact result, rounded exactly as the kernel rounds.  Outputs start as NaN and sit in 8-column buffers whose unused
columns must stay NaN, so a missed row or a stray column write fails the check.

Row reductions are fixed for a given segment length (lanes in K order, then one butterfly), so results must not
depend on the grid, the batch instantiation, the weight alignment or the run: those checks are bit for bit.

The fused prologue's activation image is read back through a probe matrix: Q8_0 rows with d = 1 and a single q = 1,
so output i is d_x(block) * q_x(i), exact in f32.  All K elements are probed."""
import ctypes
import os
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import oracle
from mistralrs_b200 import GGML, lib, quant
from util import TORCH_DT, make_acts, make_weight, to_dev

pytestmark = pytest.mark.gpu

X_Q8_1 = 4
PLAIN, GLU, QKV = 0, 1, 2
DT_CODE = {"f16": 0, "bf16": 1, "f32": 2}
U32 = 2.0 ** -24
EPS = 1e-5
H, FF, KV, VOCAB = 4096, 14336, 1024, 128256  # Llama-3-8B

# mmvq_types.cuh: block elements, block bytes, 32-weight units per block, aux floats per unit, alignment of the
# FAST path, units per lane per K segment; LONG: the type has the long-segment variant (HasLong)
QTYPE = {
    "q4_k": SimpleNamespace(QK=256, BYTES=144, UPB=8, AUX=4, WALIGN=16, UPL=2, LONG=True),
    "q5_k": SimpleNamespace(QK=256, BYTES=176, UPB=8, AUX=4, WALIGN=16, UPL=4, LONG=False),
    "q6_k": SimpleNamespace(QK=256, BYTES=210, UPB=8, AUX=2, WALIGN=2, UPL=2, LONG=True),
    "q8_0": SimpleNamespace(QK=32, BYTES=34, UPB=1, AUX=1, WALIGN=2, UPL=2, LONG=False),
    "q3_k": SimpleNamespace(QK=256, BYTES=110, UPB=8, AUX=4, WALIGN=2, UPL=8, LONG=False),
    "q4_0": SimpleNamespace(QK=32, BYTES=18, UPB=1, AUX=2, WALIGN=2, UPL=4, LONG=False),
    "q5_0": SimpleNamespace(QK=32, BYTES=22, UPB=1, AUX=2, WALIGN=2, UPL=4, LONG=False),
}


# ------------------------------------------------------------------------------------------------ planning rule
def _dev():
    return torch.cuda.get_device_properties(0)


def _plan(t, K, b, vrows, mode=PLAIN, wbytes=0, aligned=True):
    """launch_type / plan8 / launch_one of mmvq.cu with the default switches: which variant, how many CTAs per SM,
    how deep a ring, and the grid."""
    q, props = QTYPE[t], _dev()
    ncols = 1 if b == 1 else 2 if b == 2 else 4 if b <= 4 else 8
    upl = 2 * q.UPL if (q.LONG and aligned and ncols == 1 and wbytes >= 128 << 20) else q.UPL
    seg_units = 32 * upl
    seg_blocks = seg_units // q.UPB
    stage = 16 * ((seg_blocks * q.BYTES + 45) & ~15)
    npos = -(-(K // q.QK) // seg_blocks) * seg_units
    xbytes = 256 + ncols * npos * (32 + 4 * q.AUX) + 128
    smax = props.shared_memory_per_block_optin
    ctas, budget, full = 2, smax // 2 - 1024, smax - 1024
    nst = 12
    while nst > 2 and xbytes + nst * stage > budget:
        nst -= 1
    if xbytes + nst * stage > budget:
        ctas = 1
        while nst < 4 and xbytes + (nst + 1) * stage <= full:
            nst += 1
    P = 8 if mode & 3 == GLU else 16
    want = -(-vrows // P)
    grid = max(1, min(want, ctas * props.multi_processor_count))
    return SimpleNamespace(ok=xbytes + nst * stage <= smax, ctas=ctas, nst=nst, upl=upl, P=P, want=want, grid=grid,
                           vrows=vrows, clamped=want > grid)


def _cta_rows(pl, c):
    return pl.vrows * c // pl.grid, pl.vrows * (c + 1) // pl.grid


def _assert_partial_passes(pl):
    # clamped: the CTA ranges are not whole passes, so last passes run with padding slots
    assert pl.clamped, pl
    assert any((b - a) % pl.P for a, b in (_cta_rows(pl, c) for c in range(pl.grid))), pl


# ------------------------------------------------------------------------------------------------ launches
def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _addr(t, off=0):
    return ctypes.c_void_p(0 if t is None else t.data_ptr() + off)


def _fused(t, mode, dt, ws, x, outs, K, ns, b, norm=None, resid=None, woff=0):
    """mrs_mmvq_fused; ws / outs / ns are lists of up to three (weights are uint8 tensors, `woff` bytes in)."""
    ws, outs, ns = list(ws) + [None] * (3 - len(ws)), list(outs) + [None] * (3 - len(outs)), list(ns) + [0] * (3 - len(ns))
    return lib().mrs_mmvq_fused(
        ctypes.c_int(GGML[t]), ctypes.c_int(mode), ctypes.c_int(DT_CODE[dt]), *(_addr(w, woff) for w in ws), _addr(x),
        _addr(norm), ctypes.c_float(EPS), _addr(resid), *(_addr(o) for o in outs), ctypes.c_int(K),
        *(ctypes.c_int(n) for n in ns), ctypes.c_int(b), ctypes.c_int(0), ctypes.c_int(0), _stream())


def _out(n, dt):
    """an 8-column NaN-filled output; a batch-b launch must write columns 0..b-1 and nothing else"""
    return torch.full((8, n), float("nan"), dtype=TORCH_DT[dt], device="cuda")


def _used(o, b):
    rest = o[b:].float()
    assert torch.isnan(rest).all(), "a launch wrote outside its batch columns"
    return o[:b]


def _run(t, mode, dt, ws, x, ns, b, K, **kw):
    """one launch into fresh NaN outputs; returns the b used columns of each output"""
    outs = [_out(n, dt) for n in (ns if mode & 3 == QKV else ns[:1])]
    rc = _fused(t, mode, dt, ws, x, outs, K, ns, b, **kw)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return [_used(o, b) for o in outs]


def _np(t):
    return t.float().cpu().numpy()


# ------------------------------------------------------------------------------------------------ oracle side
_WCACHE = {}


def _weight(t, n, K, seed):
    key = (t, n, K, seed)
    if key not in _WCACHE:
        if len(_WCACHE) > 8:
            _WCACHE.clear()
        wb = make_weight(t, n, K, seed).reshape(n, -1)
        _WCACHE[key] = (wb, torch.from_numpy(wb.reshape(-1)).cuda())
    return _WCACHE[key]


def _image(x):
    """oracle Q8_1 bytes of x [b, K] and the same bytes on the device"""
    img, _ = oracle.quantize_q8_1(x, k_padded=x.shape[1])
    return img, torch.from_numpy(img).cuda()


def _image_values(img, b, K):
    """(d, q) of a Q8_1 image: d [b, K/32] (f16 widened), q [b, K]"""
    blk = img.reshape(b, K // 32, 36)
    d = blk[..., :2].copy().view(np.float16)[..., 0].astype(np.float64)
    q = blk[..., 4:].view(np.int8).reshape(b, K).astype(np.float64)
    return d, q


def _exact(t, wb, img, K, b):
    """oracle.mmvq_q8_1 (f64, the reference's integer-dot arithmetic), rows split over threads"""
    n = wb.shape[0]
    step = -(-n // (os.cpu_count() or 1))
    parts = [(r, min(n, r + step)) for r in range(0, n, step)]
    with ThreadPoolExecutor(len(parts)) as ex:
        outs = ex.map(lambda p: oracle.mmvq_q8_1(t, wb[p[0]:p[1]], img, K, p[1] - p[0], K // 32, b), parts)
    return np.concatenate(list(outs), axis=1)


def _rnd(v, dt):
    return oracle.round_dtype(np.asarray(v).astype(np.float32), dt)


def _assert_epilogue(got, y, dt, resid=None, slack=0.0, what=""):
    """got [b, n] (kernel, widened) against the exact y [b, n]: got must lie between epi(y - delta) and
    epi(y + delta), epi = round to dt [then + residual in f32, rounded to dt again], delta = 5e-6 of the largest |y|
    (f32 summation order) plus `slack`.  Implies |got - ref| <= ulp(dt) * |ref| * 1.01 + 5e-6 * scale per element."""
    delta = 5e-6 * np.abs(y).max() + slack

    def epi(v):
        v = _rnd(v, dt)
        return v if resid is None else _rnd(v + resid.astype(np.float32), dt)

    lo, hi = epi(y - delta), epi(y + delta)
    ok = (got >= lo) & (got <= hi)
    if not ok.all():
        i = np.argwhere(~ok)[:5]
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.size} outside the bound, e.g. "
                             + ", ".join(f"[{c},{r}] got {got[c, r]!r} want {y[c, r]!r}" for c, r in i))


def _silu64(g):
    return g * 0.5 * (1.0 + np.tanh(0.5 * g)), 0.5 * (1.0 + np.tanh(0.5 * g))


def _assert_glu(got, g, u, dt, what=""):
    """fused SiLU GLU against oracle.fused_glu(round(gate), round(up)).  Gate and up carry the 5e-6 summation
    allowance; the kernel's silu uses __expf / __fdividef (the reference's fast math), relative error at most
    2^-24 (4 + 1.2 |g| / (1 + e^g))."""
    dg, du = 5e-6 * np.abs(g).max(), 5e-6 * np.abs(u).max()
    ref = oracle.fused_glu(_rnd(g, dt), _rnd(u, dt), 0, dt).astype(np.float64)
    silu, sig = _silu64(g)
    fm = U32 * (8 + 1.2 * np.abs(g) * (1.0 - sig))
    if dt == "f32":
        # propagated bound: |silu'| <= 1.1
        tol = fm * np.abs(silu * u) + 1.1 * dg * np.abs(u) + (np.abs(silu) + 1.1 * dg) * du + 1.01 * U32 * np.abs(ref)
        ok = np.abs(got - ref) <= tol
    else:
        # 16-bit: the issue-style bound, or (where gate, up or the activation lie within their error of a rounding
        # boundary) exactly one of the roundings the kernel may have taken
        ok = np.abs(got - ref) <= 2.0 ** -8 * 1.01 * np.abs(ref) + 5e-6 * np.abs(ref).max()
        for gc in (_rnd(g - dg, dt), _rnd(g + dg, dt)):
            s, _ = _silu64(gc.astype(np.float64))
            for a in (_rnd(s * (1 - fm), dt), _rnd(s * (1 + fm), dt)):
                for uc in (_rnd(u - du, dt), _rnd(u + du, dt)):
                    ok |= got == _rnd(a * uc, dt)
    if not ok.all():
        i = np.argwhere(~ok)[:5]
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.size} outside the bound, e.g. "
                             + ", ".join(f"[{c},{r}] got {got[c, r]!r} want {ref[c, r]!r}" for c, r in i))


def _row_slice(t, w, K, r0, r1):
    rb = K // QTYPE[t].QK * QTYPE[t].BYTES
    return w[r0 * rb:r1 * rb]


def _assert_rows_match_slices(t, mode, dt, ws, x, pl, K, b, got, n, **kw):
    """rows around CTA boundaries of a clamped launch == a small unclamped launch on that row slice, bit for bit"""
    for c in sorted({1, pl.grid // 3, pl.grid // 2, pl.grid - 1}):
        a, _ = _cta_rows(pl, c)
        r0, r1 = max(0, a - 12), min(n, a + 36)
        small = _plan(t, K, b, r1 - r0, mode)
        assert not small.clamped and small.upl == QTYPE[t].UPL
        part = _run(t, mode, dt, [_row_slice(t, w, K, r0, r1) for w in ws], x, [r1 - r0] * len(ws), b, K, **kw)[0]
        assert torch.equal(part, got[:, r0:r1]), (t, mode, c, r0, r1)


# ================================================================================================ 1. oracle checks
@pytest.mark.parametrize("b,dt", [(1, "f32"), (2, "f32"), (3, "f32"), (5, "f32"), (8, "f32"), (3, "bf16")])
def test_clamped_plain(cuda, b, dt):
    # ffn_up-shaped plain GEMV: 14336 rows -> 896 passes on at most 2 x SMs CTAs
    N, K = FF, H
    pl = _plan("q4_k", K, b, N)
    _assert_partial_passes(pl)
    wb, w = _weight("q4_k", N, K, 100)
    x = make_acts(b, K, 101, "f32")
    img, yd = _image(x)
    got = _run("q4_k", X_Q8_1, dt, [w], yd, [N], b, K)[0]
    _assert_epilogue(_np(got), _exact("q4_k", wb, img, K, b), dt, what=f"plain b={b} {dt}")
    assert torch.equal(got, _run("q4_k", X_Q8_1, dt, [w], yd, [N], b, K)[0])  # re-run
    _assert_rows_match_slices("q4_k", X_Q8_1, dt, [w], yd, pl, K, b, got, N)


@pytest.mark.parametrize("b,dt", [(1, "f32"), (4, "f32"), (6, "f32"), (7, "f32"), (8, "f32"), (1, "bf16")])
def test_clamped_glu(cuda, b, dt):
    # gate||up of the FFN: 14336 rows at 8 per pass
    N, K = FF, H
    pl = _plan("q4_k", K, b, N, GLU)
    _assert_partial_passes(pl)
    (gb, g), (ub, u) = _weight("q4_k", N, K, 110), _weight("q4_k", N, K, 111)
    x = make_acts(b, K, 112, "f32")
    img, yd = _image(x)
    got = _run("q4_k", GLU | X_Q8_1, dt, [g, u], yd, [N, N], b, K)[0]
    _assert_glu(_np(got), _exact("q4_k", gb, img, K, b), _exact("q4_k", ub, img, K, b), dt, f"glu b={b} {dt}")
    assert torch.equal(got, _run("q4_k", GLU | X_Q8_1, dt, [g, u], yd, [N, N], b, K)[0])
    _assert_rows_match_slices("q4_k", GLU | X_Q8_1, dt, [g, u], yd, pl, K, b, got, N)


def _qkv_oracle(ns, b, seed, dt="f32", t="q4_k"):
    K = H
    ws = [_weight(t, n, K, seed + i) for i, n in enumerate(ns)]
    pl = _plan(t, K, b, sum(ns), QKV)
    x = make_acts(b, K, seed + 5, "f32")
    img, yd = _image(x)
    got = _run(t, QKV | X_Q8_1, dt, [w for _, w in ws], yd, ns, b, K)
    for name, o, (wb, _) in zip("qkv", got, ws):
        _assert_epilogue(_np(o), _exact(t, wb, img, K, b), dt, what=f"qkv {name} b={b} {ns}")
    return pl, got


@pytest.mark.parametrize("b", [1, 3, 8])
def test_clamped_qkv(cuda, b):
    ns = [H, KV, KV]
    pl, _ = _qkv_oracle(ns, b, 120)
    _assert_partial_passes(pl)


def _straddling_qkv_rows():
    """q/k/v row counts (near 4096/1024/1024) for which the q/k and the k/v boundaries both fall inside a CTA's
    range and inside one of its 16-row passes, and the grid is clamped"""
    for nk in range(KV, KV + 64):
        for nq in range(H, H + 256):
            pl = _plan("q4_k", H, 1, nq + 2 * nk, QKV)
            if not pl.clamped:
                continue
            cuts = [_cta_rows(pl, c)[0] for c in range(pl.grid)]
            if all(bd not in cuts and (bd - max(c for c in cuts if c < bd)) % 16 for bd in (nq, nq + nk)):
                return [nq, nk, nk]
    raise AssertionError("no straddling q/k/v split found")


@pytest.mark.parametrize("b", [1, 3])
def test_row_ranges_cross_qkv_boundaries(cuda, b):
    # one 16-row pass holds rows of two matrices (different weight pointers, destinations and row strides)
    ns = _straddling_qkv_rows()
    pl, _ = _qkv_oracle(ns, b, 130)
    _assert_partial_passes(pl)


def test_trimmed_dual_grid(cuda):
    # Q4_K_M attention input: q||k Q4_K and v Q6_K as one grid; 320 + 64 wanted CTAs > 2 x SMs -> trimmed
    K, (nq, nk, nv) = H, (H, KV, KV)
    sms = _dev().multi_processor_count
    ga, gb = -(-(nq + nk) // 16), -(-nv // 16)
    assert ga + gb > 2 * sms and _plan("q4_k", K, 1, nq + nk, QKV).ctas == 2 and _plan("q6_k", K, 1, nv).ctas == 2
    (wqb, wq), (wkb, wk), (wvb, wv) = _weight("q4_k", nq, K, 140), _weight("q4_k", nk, K, 141), _weight("q6_k", nv, K, 142)
    tq, tk, tv = (quant.QTensor(w, t, (n, K)) for w, t, n in ((wq, "q4_k", nq), (wk, "q4_k", nk), (wv, "q6_k", nv)))
    # raw f32 activations without a norm: the image is what the standalone quantiser makes of x
    x = to_dev(make_acts(1, K, 143, "f32"), cuda, "f32")
    img = quant.quantize_q8_1(x).cpu().numpy()
    got = quant.fused_qkv_mixed(tq, tk, tv, x)
    for name, o, (t, wb) in zip("qkv", got, (("q4_k", wqb), ("q4_k", wkb), ("q6_k", wvb))):
        _assert_epilogue(_np(o), _exact(t, wb, img, K, 1), "f32", what=f"dual {name}")
    # with the norm: the trimmed grid == the q||k launch + the v launch it stands for
    xb = to_dev(make_acts(1, K, 144, "bf16"), cuda, "bf16")
    nw = to_dev(1.0 + 0.1 * make_acts(1, K, 145, "bf16")[0], cuda, "bf16")
    q, k, v = quant.fused_qkv_mixed(tq, tk, tv, xb, norm_w=nw, eps=EPS)
    q2, k2 = quant.mmvq_fused(tq, xb, mode=2, w1=tk, norm_w=nw, eps=EPS)[:2]
    assert torch.equal(q, q2) and torch.equal(k, k2) and torch.equal(v, quant.mmvq_fused(tv, xb, norm_w=nw, eps=EPS))


@pytest.mark.parametrize("t", ["q4_k", "q6_k", "q8_0"])
@pytest.mark.parametrize("b", [5, 6, 7, 8])
def test_one_cta_per_sm(cuda, t, b):
    # ffn_down: K = 14336; 8 columns of its activation image and two ring stages do not fit twice per SM
    N, K = H, FF
    pl = _plan(t, K, b, N)
    assert pl.ctas == 1, pl
    wb, w = _weight(t, N, K, 150)
    x = make_acts(b, K, 151, "f32")
    img, yd = _image(x)
    outs = [_out(N, "f32")]
    rc = _fused(t, X_Q8_1, "f32", [w], yd, outs, K, [N], b)
    if not pl.ok:
        assert rc == 9, rc  # cudaErrorInvalidConfiguration: the image does not fit even once
        return
    assert rc == 0, rc
    torch.cuda.synchronize()
    _assert_epilogue(_np(_used(outs[0], b)), _exact(t, wb, img, K, b), "f32", what=f"down {t} b={b}")


def test_long_segments_lm_head(cuda):
    # Q6_K output.weight: 128256 x 4096 = 411 MiB of weights -> K segments of 4 units per lane
    N, K = VOCAB, H
    wbytes = N * (K // 256) * 210
    pl = _plan("q6_k", K, 1, N, wbytes=wbytes)
    assert pl.upl == 4 and pl.ctas == 2, pl
    _assert_partial_passes(pl)
    wb = make_weight("q6_k", N, K, 160).reshape(N, -1)
    w = torch.from_numpy(wb.reshape(-1)).cuda()
    x = make_acts(1, K, 161, "f32")
    img, yd = _image(x)
    got = _run("q6_k", X_Q8_1, "f32", [w], yd, [N], 1, K)[0]
    _assert_epilogue(_np(got), _exact("q6_k", wb, img, K, 1), "f32", what="lm_head")
    # No bitwise check against row slices here: a slice is a short-segment launch, and the two variants hand the
    # chunks of a block to different lanes (16 blocks per segment instead of 8), so their f32 partial sums, and the
    # last bit of a row, may differ.  The clamped short-segment launches above carry the row-partition check.


# ================================================================================================ 2. invariance
@pytest.mark.parametrize("what", ["plain", "glu", "qkv", "prologue", "prologue_qkv"])
def test_batch_columns_equal_batch1(cuda, what):
    # column j of a batch-b launch (NCOLS = 2 / 4 / 8 with column masking) == the batch-1 launch on column j
    K = H
    if what in ("plain", "prologue"):
        mode, ns, seeds = PLAIN, [FF], [170]
    elif what == "glu":
        mode, ns, seeds = GLU, [FF, FF], [171, 172]
    else:
        mode, ns, seeds = QKV, [H, KV, KV], [173, 174, 175]
    ws = [_weight("q4_k", n, K, s)[1] for n, s in zip(ns, seeds)]
    xr = to_dev(make_acts(8, K, 176, "bf16"), cuda, "bf16")
    raw = what.startswith("prologue")
    if raw:
        nw = to_dev(1.0 + 0.1 * make_acts(1, K, 177, "bf16")[0], cuda, "bf16")
        x, kw = xr, {"norm": nw}
        if mode == PLAIN:
            kw["resid"] = to_dev(make_acts(8, ns[0], 178, "bf16"), cuda, "bf16")
    else:
        mode |= X_Q8_1
        x, kw = quant.quantize_q8_1(xr).view(8, -1), {}

    def launch(cols):
        xx = x[cols].contiguous()
        k = dict(kw, resid=kw["resid"][cols].contiguous()) if "resid" in kw else kw
        return _run("q4_k", mode, "bf16", ws, xx, ns, len(cols), K, **k)

    one = [launch([j]) for j in range(8)]
    for b in range(2, 9):
        many = launch(list(range(b)))
        for j in range(b):
            for m, (o1, ob) in enumerate(zip(one[j], many)):
                assert torch.equal(ob[j], o1[0]), (what, b, j, m)


@pytest.mark.parametrize("t,off", [("q4_k", 2), ("q5_k", 2), ("q8_0", 1), ("q6_k", 1), ("q3_k", 1), ("q4_0", 1),
                                   ("q5_0", 1)])
@pytest.mark.parametrize("b", [1, 3])
def test_unaligned_weights(cuda, t, off, b):
    # weights at an address that breaks WALIGN take the FAST = false loads; same arithmetic.  At an odd address the
    # f16 scale of Q8_0 / Q4_0 / Q5_0 / Q3_K / Q6_K blocks sits at an odd shared-memory address too
    N, K = 2000, H
    assert off % QTYPE[t].WALIGN
    wb, w = _weight(t, N, K, 180)
    shifted = torch.zeros(w.numel() + 16, dtype=torch.uint8, device=cuda)
    base = (-shifted.data_ptr()) % 16
    shifted[base + off:base + off + w.numel()] = w
    xr = to_dev(make_acts(b, K, 181, "bf16"), cuda, "bf16")
    nw = to_dev(1.0 + 0.1 * make_acts(1, K, 182, "bf16")[0], cuda, "bf16")
    yq = quant.quantize_q8_1(xr)
    for mode, x, kw in ((X_Q8_1, yq, {}), (PLAIN, xr, {"norm": nw})):
        a = _run(t, mode, "bf16", [w], x, [N], b, K, **kw)[0]
        u = _run(t, mode, "bf16", [shifted], x, [N], b, K, woff=base + off, **kw)[0]
        assert torch.equal(a, u), (t, off, b, mode)
        assert torch.equal(u, _run(t, mode, "bf16", [shifted], x, [N], b, K, woff=base + off, **kw)[0])


# ================================================================================================ 3. fused prologue
_PROBES = {}


def _probe_weights(K):
    """Q8_0 [K, K]: row i holds d = 1 and q = 1 at column i, zero elsewhere"""
    if K not in _PROBES:
        p = np.zeros((K, K // 32, 34), dtype=np.uint8)
        r = np.arange(K)
        p[r, r // 32, 1] = 0x3C  # f16 1.0
        p[r, r // 32, 2 + r % 32] = 1
        _PROBES[K] = torch.from_numpy(p.reshape(-1)).cuda()
    return _PROBES[K]


def _qround(t):
    return np.sign(t) * np.floor(np.abs(t) + 0.5)  # roundf: ties away from zero


def _probe(x, nw, dt, b, K):
    """Read back the prologue's Q8_1 image of (RMSNorm'd) x through the probe matrix and check it (_check_image).
    Returns kernel image - oracle image [b, K] (exact for f32) and the oracle image bytes."""
    pl = _plan("q8_0", K, b, K)
    xd = to_dev(x, "cuda", dt)
    nwd = None if nw is None else to_dev(nw, "cuda", dt)
    outs = [_out(K, dt)]
    rc = _fused("q8_0", PLAIN, dt, [_probe_weights(K)], xd, outs, K, [K], b, norm=nwd)
    if not pl.ok:
        assert rc == 9, rc
        return None, None
    assert rc == 0, rc
    torch.cuda.synchronize()
    return _check_image(_np(_used(outs[0], b)).astype(np.float64), x, nw, dt, b, K)


def _check_image(got, x, nw, dt, b, K):
    """got [b, K] = d_x * q_x of the kernel's image against quantize_q8_1(round_dt(rms_norm_f64(x) * w)).  An element
    may take another value only where the normalised value lies within its f32 error of a dtype rounding boundary, or
    v / d within the fast divisions' error of a q rounding boundary, and a block's d only where amax / 127 lies within
    that error of an f16 rounding boundary."""
    x64 = x.astype(np.float64)
    if nw is None:
        v64, en = x64, 0.0
    else:
        v64 = x64 / np.sqrt((x64 * x64).mean(axis=1, keepdims=True) + EPS) * nw.astype(np.float64)
        # kernel: f32 sum of squares (<= K / 256 + 13 sequential adds), rsqrtf (2 ulp), two products
        en = U32 * (K / 512 + 16)
    img, _ = oracle.quantize_q8_1(_rnd(v64, dt), k_padded=K)
    d_ref, q_ref = _image_values(img, b, K)
    x_ref = (d_ref[..., None] * q_ref.reshape(b, -1, 32)).reshape(b, K)

    vl, vh = _rnd(v64 * (1 - en), dt).astype(np.float64), _rnd(v64 * (1 + en), dt).astype(np.float64)
    alo = np.minimum(np.abs(vl), np.abs(vh)).reshape(b, -1, 32).max(-1)
    ahi = np.maximum(np.abs(vl), np.abs(vh)).reshape(b, -1, 32).max(-1)
    qmin = np.full((b, K), np.inf)
    qmax = np.full((b, K), -np.inf)
    for a in (alo, ahi):
        ae = np.repeat(a, 32, axis=1)
        for v in (vl, vh):
            for s in (1 - 6 * U32, 1 + 6 * U32):  # two __fdividef, 2 ulp each, and the oracle's IEEE divisions
                q = _qround(v * 127.0 / ae * s)
                qmin, qmax = np.minimum(qmin, q), np.maximum(qmax, q)
    gotb = got.reshape(b, -1, 32)
    block_ok = np.zeros(d_ref.shape, dtype=bool)
    for a in (alo, ahi):
        for s in (1 - 3 * U32, 1 + 3 * U32):
            dh = (a / 127.0 * s).astype(np.float32).astype(np.float16).astype(np.float64)[..., None]
            el = np.zeros(gotb.shape, dtype=bool)
            for k in range(3):
                q = np.minimum(qmin + k, qmax).reshape(gotb.shape)
                el |= gotb == _rnd(dh * q, dt)
            block_ok |= el.all(-1)
    if not block_ok.all():
        c, blk = np.argwhere(~block_ok)[0]
        sl = slice(32 * blk, 32 * blk + 32)
        raise AssertionError(f"prologue image {dt} K={K} b={b} norm={nw is not None}: {int((~block_ok).sum())} blocks "
                             f"off, e.g. column {c} block {blk}: got {got[c, sl]} want {_rnd(x_ref[c, sl], dt)}")
    # flips are the exception, not the rule
    assert (got != _rnd(x_ref, dt)).mean() < 2e-2, (dt, K, b)
    return got - x_ref, img


@pytest.mark.parametrize("K", [2048, 4096, 5120, 8192, 14336])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("b", [1, 3, 8])
def test_prologue_image(cuda, K, dt, norm, b):
    x = make_acts(b, K, 190 + K % 97, dt)
    nw = oracle.round_dtype(1.0 + 0.1 * make_acts(1, K, 191, "f32")[0], dt) if norm else None
    _probe(x, nw, dt, b, K)


@pytest.mark.parametrize("t", ["q4_k", "q6_k", "q8_0"])
@pytest.mark.parametrize("K", [H, FF])
@pytest.mark.parametrize("b", [1, 3, 8])
def test_fused_launch_vs_oracle(cuda, t, K, b):
    # RMSNorm + Q8_1 + GEMV + residual in one launch (plain and QKV) against oracle.mmvq_q8_1 on the oracle's image;
    # the allowance for the elements where the probe saw the kernel's image differ is sum_i |w_i| * |dx_i|
    x = make_acts(b, K, 200, "f32")
    nw = 1.0 + 0.1 * make_acts(1, K, 201, "f32")[0]
    dx, img = _probe(x, nw, "f32", b, K)
    assert dx is not None, "the Q8_0 probe must fit wherever the launches under test do"
    for mode, ns in ((PLAIN, [1024]), (QKV, [512, 128, 128])):
        pl = _plan(t, K, b, sum(ns), mode)
        ws = [_weight(t, n, K, 202 + i) for i, n in enumerate(ns)]
        res = make_acts(b, max(ns), 205, "f32")
        outs = [_out(n, "f32") for n in ns]
        rc = _fused(t, mode, "f32", [w for _, w in ws], to_dev(x, cuda, "f32"), outs, K, ns, b,
                    norm=to_dev(nw, cuda, "f32"), resid=to_dev(res, cuda, "f32"))
        if not pl.ok:
            assert rc == 9, (rc, pl)
            continue
        assert rc == 0, rc
        torch.cuda.synchronize()
        nz = np.flatnonzero(np.abs(dx).max(axis=0))
        for m, (o, (wb, _), n) in enumerate(zip(outs, ws, ns)):
            wd = oracle.dequantize(t, wb).reshape(n, K)[:, nz].astype(np.float64)
            slack = (np.abs(dx[:, nz]) @ np.abs(wd).T) * (1 + 2.0 ** -20)
            # the epilogue adds residual[j * n_m + r] for matrix m (row stride n_m)
            r = res.reshape(-1)[:b * n].reshape(b, n)
            _assert_epilogue(_np(_used(o, b)), _exact(t, wb, img, K, b), "f32", resid=r, slack=slack,
                             what=f"fused {t} K={K} b={b} mode={mode} m={m}")
