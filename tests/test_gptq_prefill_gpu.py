"""GPTQ prompt prefill: the whole-K and GLU-epilogue forms of the W4A16 GEMM (`pdl` bits 1 and 2 of
mrs_w4a16_gemm_pdl), `mrs_gptq_prefill_step` through `GptqPrefill.forward` / `forward_batch` against the CPU oracle
in both cache layouts, batch independence, chunked prompts, the hand-off to a GptqRunner's rows, and the C entry's
rejections."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from oracle import gptq as og
from oracle.gptq_model import OracleGptq
from mistralrs_b200 import gptq_model as G
from mistralrs_b200 import lib
from mistralrs_b200.model import rope_tables

pytestmark = pytest.mark.gpu

TDT = {"f16": torch.float16, "bf16": torch.bfloat16}
ULP = {"f16": 2.0 ** -11, "bf16": 2.0 ** -8}
# last-row / all-row logits against the oracle fed token by token, as a share of the logit scale (the decode test's
# bound in f16; bf16 activations carry 8 bits, so roundings that differ between f32 and f64 accumulation weigh 8x more)
LOGIT_TOL = {"f16": 3e-3, "bf16": 2.4e-2}


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------- the W4A16 GEMM flags
def _tiles(q, scales, dt, cuda):
    """q [K, N] nibbles, f16 scales [K/group, N] -> (int4 tiles, scales in dt) as GptqWeights uploads them"""
    K, N = q.shape
    qw = torch.from_numpy(og.pack_gptq(q)).to(cuda)
    tiles = torch.empty(K // 16, N * 16 // 8, dtype=torch.int32, device=cuda)
    lib().gptq_marlin_repack(ctypes.c_void_p(qw.data_ptr()), ctypes.c_void_p(0), ctypes.c_void_p(tiles.data_ptr()),
                             ctypes.c_int(K), ctypes.c_int(N), ctypes.c_int(4), ctypes.c_int64(torch.cuda.current_stream().cuda_stream))
    return tiles, torch.from_numpy(scales).to(cuda).to(TDT[dt])


def _gemm(x, tiles, scales, N, group, flags):
    M, K = x.shape
    y = torch.full((M, N // 2 if flags & 4 else N), float("nan"), dtype=x.dtype, device=x.device)
    rc = lib().mrs_w4a16_gemm_pdl(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(tiles.data_ptr()),
                                  ctypes.c_void_p(scales.data_ptr()), ctypes.c_void_p(0), ctypes.c_void_p(y.data_ptr()),
                                  M, K, N, group, 0 if x.dtype == torch.float16 else 1, 0, flags, _stream())
    assert rc == 0, rc
    return y


def _deq(q, scales, group, dt):
    """the weights as the GEMM's MMA operands hold them: (q - 8) * s rounded once to dt"""
    s = torch.from_numpy(scales).to(TDT[dt]).float().numpy()
    w = (q - 8).astype(np.float32) * s[np.arange(q.shape[0]) // group]
    return torch.from_numpy(w).to(TDT[dt]).float().numpy()


def _mk(K, N, group, seed):
    rng = np.random.default_rng(seed)
    return rng, rng.integers(0, 16, size=(K, N)), np.exp2(rng.uniform(-8, -6, size=(K // group, N))).astype(np.float16)


@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_whole_k_rows_do_not_depend_on_m(cuda, dt):
    """With bit 1 a row of Y is the same for every M (no K split at 64 rows or fewer), and within the oracle bound."""
    K, N, group = 1024, 576, 128                     # 4.5 row tiles: split over K at small M without the bit
    rng, q, scales = _mk(K, N, group, 11)
    tiles, sc = _tiles(q, scales, dt, cuda)
    x = torch.from_numpy(rng.standard_normal((300, K)).astype(np.float32)).to(cuda).to(TDT[dt])
    full = _gemm(x, tiles, sc, N, group, 2)
    for M in (1, 7, 33, 64, 65):
        assert torch.equal(_gemm(x[:M].contiguous(), tiles, sc, N, group, 2), full[:M]), M
    wd = _deq(q, scales, group, dt)
    xs = x.float().cpu().numpy()
    ref = xs.astype(np.float64) @ wd.astype(np.float64)
    tol = ULP[dt] * np.abs(ref) * 1.01 + 2e-6 * (np.abs(xs).astype(np.float64) @ np.abs(wd)) + 1e-6
    assert (np.abs(full.float().cpu().numpy() - ref) <= tol).all()


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("M", [1, 40, 300, 2048])
def test_glu_epilogue_matches_gemm_then_split_glu(cuda, dt, M):
    """bit 2 over gate||up (I = 320: a ragged last 64-row pair) == the plain whole-K GEMM + fused_split_glu, bit for bit;
    the plain GEMM stays within the oracle bound."""
    K, I, group = 512, 320, 64
    rng, q, scales = _mk(K, 2 * I, group, 12 + M)
    tiles, sc = _tiles(q, scales, dt, cuda)
    x = torch.from_numpy((0.5 * rng.standard_normal((M, K))).astype(np.float32)).to(cuda).to(TDT[dt])
    glu = _gemm(x, tiles, sc, 2 * I, group, 2 | 4)
    gate_up = _gemm(x, tiles, sc, 2 * I, group, 2)
    want = torch.empty(M, I, dtype=x.dtype, device=cuda)
    lib().mrs_split_glu_pdl(ctypes.c_void_p(gate_up.data_ptr()), ctypes.c_void_p(want.data_ptr()), ctypes.c_uint32(M),
                            ctypes.c_uint32(I), 0, 0 if dt == "f16" else 1, 0, _stream())
    torch.cuda.synchronize()
    assert torch.equal(glu, want)
    wd = _deq(q, scales, group, dt)
    xs = x.float().cpu().numpy()
    ref = xs.astype(np.float64) @ wd.astype(np.float64)
    tol = ULP[dt] * np.abs(ref) * 1.01 + 2e-6 * (np.abs(xs).astype(np.float64) @ np.abs(wd)) + 1e-6
    assert (np.abs(gate_up.float().cpu().numpy() - ref) <= tol).all()


def test_gemm_flag_rejections(cuda):
    K, N, group = 256, 128, 64
    _, q, scales = _mk(K, N, group, 13)
    tiles, sc = _tiles(q, scales, "f16", cuda)
    x = torch.zeros(4, K, dtype=torch.float16, device=cuda)
    y = torch.zeros(4, N, dtype=torch.float16, device=cuda)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    assert lib().mrs_w4a16_gemm_pdl(P(x), P(tiles), P(sc), None, P(y), 4, K, N, group, 0, 0, 8, _stream()) == 1
    assert lib().mrs_w4a16_gemm_pdl(P(x), P(tiles), P(sc), None, P(y), 4, K, 120, group, 0, 0, 4, _stream()) == 1
    w = torch.zeros(N, K, dtype=torch.float16, device=cuda)
    assert lib().mrs_dense_linear_pdl(P(x), P(w), P(y), 4, K, N, 0, 4, _stream()) == 1
    assert lib().mrs_dense_linear_pdl(P(x), P(w), P(y), 4, K, N, 0, 2, _stream()) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------- the model against the oracle
class _F64(np.ndarray):
    """an f64 array whose astype(np.float64) is itself: the oracle converts the lm_head at every step"""

    def astype(self, dtype, *a, **kw):
        return self if np.dtype(dtype) == np.float64 else np.ndarray.astype(self, dtype, *a, **kw)


class Oracle(OracleGptq):
    """OracleGptq whose linears take the weights rounded once to the activation format (the device's scales are the
    checkpoint's f16 scales converted to it), in f32 products (the bounds here are far above f32 rounding)."""

    def _lin(self, l, name, x):
        key = (l, name)
        if key not in self._deq:
            qw, sc = self.hw[key]
            q = np.empty((qw.shape[0] * 8, qw.shape[1]), dtype=np.int32)
            for j in range(8):
                q[j::8] = (qw.view(np.uint32) >> np.uint32(4 * j)) & 0xF
            self._deq[key] = _deq(q, sc, self.cfg.group_size, self.dt)
        return oracle.round_dtype(np.asarray(x, dtype=np.float32) @ self._deq[key], self.dt)


def _oracle(w, dt):
    cos, sin = rope_tables(w.cfg)
    host = dict(w.host)
    host[(0, "lm_head")] = np.asarray(host[(0, "lm_head")], dtype=np.float64).view(_F64)
    return Oracle(w.cfg, host, cos, sin, dt)


def _feed(w, dt, prompt):
    """the oracle fed `prompt` token by token: (oracle, [len, vocab] logits)"""
    r = _oracle(w, dt)
    return r, np.stack([r.step([t], pos)[0] for pos, t in enumerate(prompt)])


def _near_tie(want_row, err, dt):
    top2 = np.sort(want_row)[-2:]
    return top2[1] - top2[0] <= max(8 * ULP[dt] * np.abs(want_row).max(), 2 * err)


def _prompts(vocab, n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, vocab, size=int(rng.integers(lo, hi + 1))).tolist() for _ in range(n)]


def _own_tables(n, blocks):
    return [list(range(1 + blocks * i, 1 + blocks * (i + 1))) for i in range(n)]


def _cache_rows(run, l, table, length):
    """(K, V) rows 0 .. length - 1 of a sequence in layer l of a runner's cache, [length, kv_heads * head_dim]"""
    bs = run.cfg.block_size
    blk = torch.tensor([table[p // bs] for p in range(length)], device=run.dev)
    off = torch.arange(length, device=run.dev) % bs
    kc, vc = run.k_cache[l], run.v_cache[l]
    if run.layout == "hnd":                    # [NB, KVH, BS, D]
        k, v = kc[blk, :, off], vc[blk, :, off]
    else:                                      # K [NB, KVH, D/8, BS, 8], V [NB, KVH, D, BS]
        k, v = kc[blk, :, :, off], vc[blk, :, :, off]
    return k.reshape(length, -1).float().cpu().numpy(), v.reshape(length, -1).float().cpu().numpy()


@pytest.mark.parametrize("layout", ["hnd", "vllm"])
@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_ragged_prompts_match_oracle(cuda, layout, dt):
    """Three ragged prompts of 3..40 tokens in one forward_batch into a runner's cache: last-row logits within the
    bound of the oracle fed token by token, first tokens its argmax off near-ties, the cache rows its K / V; then
    forward(all_logits=True) for one prompt: every row within the bound."""
    cfg = G.GptqConfig.tiny_test()
    w = G.GptqWeights(cfg, cuda, dtype=TDT[dt], keep_host=True)
    run = G.GptqRunner(w, batch=3, max_ctx=128, cache_layout=layout)
    pre = G.GptqPrefill(w, max_tokens=128, runner=run)
    prompts = _prompts(cfg.vocab, 3, 3, 40, seed=21)
    prompts[0] = prompts[0][:3]                          # the shortest allowed length is in the call
    logits, first = pre.forward_batch(prompts)
    got = logits.float().cpu().numpy()
    worst = 0.0
    for i, p in enumerate(prompts):
        r, want = _feed(w, dt, p)
        scale = np.abs(want[-1]).max()
        err = np.abs(got[i] - want[-1]).max() / scale
        worst = max(worst, err)
        assert err <= LOGIT_TOL[dt], (i, err)
        if int(first[i]) != int(np.argmax(want[-1])):
            assert _near_tie(want[-1], err * scale, dt), i
        for l in range(cfg.n_layers):
            k, v = _cache_rows(run, l, run.tables[i], len(p))
            wk, wv = np.concatenate(r.k[l]), np.concatenate(r.v[l])
            for g_, w_ in ((k, wk), (v, wv)):
                assert np.abs(g_ - w_).max() <= 16 * ULP[dt] * np.abs(w_).max(), (i, l)
    p = prompts[2]
    all_rows = pre.forward(p, all_logits=True).float().cpu().numpy()
    _, want = _feed(w, dt, p)
    err = np.abs(all_rows - want).max() / np.abs(want).max()
    assert err <= LOGIT_TOL[dt], err
    print(f"gptq prefill ({layout}, {dt}): worst last-row logit error {worst:.2e}, all rows {err:.2e} of the logit scale")


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("n,lo,hi", [(3, 2, 20), (9, 2, 40), (40, 2, 40)])
def test_batch_matches_one_at_a_time(cuda, dt, n, lo, hi):
    """Every GEMM runs over whole K and each sequence's attention on its own: K/V rows in every layer and last-row
    logits are bit-identical to n single-sequence calls into identical tables.  n = 3 has at most 60 rows, where a
    K split would otherwise be picked."""
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda, dtype=TDT[dt])
    prompts = _prompts(w.cfg.vocab, n, lo, hi, seed=30 + n)
    tables = _own_tables(n, 3)
    a, b = (G.GptqPrefill(w, max_tokens=48 * max(n, 2)) for _ in range(2))
    logits, first = a.forward_batch(prompts, tables=tables)
    singles = torch.stack([b.forward(p, table=t) for p, t in zip(prompts, tables)])
    torch.cuda.synchronize()
    for l in range(w.cfg.n_layers):
        assert torch.equal(a.k_cache[l], b.k_cache[l]) and torch.equal(a.v_cache[l], b.v_cache[l]), l
    assert torch.equal(logits, singles)
    assert torch.equal(first, torch.argmax(logits.float(), dim=-1).to(torch.int32).cpu())


def test_chunked_prompt_matches_one_shot(cuda):
    """A 37-token prompt as a 20-token chunk (final=False) and the rest over the cached rows (paged prompt attention):
    last-row logits within the bound of the one-shot run, the same first token off near-ties.  The vLLM layout
    refuses cached rows with a ValueError before anything runs."""
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda)
    prompt = _prompts(w.cfg.vocab, 1, 37, 37, seed=40)[0]
    one, chunked = (G.GptqPrefill(w, max_tokens=64) for _ in range(2))
    want = one.forward(prompt).float()
    assert chunked.forward_batch([prompt[:20]], final=False) is None
    got_logits, first = chunked.forward_batch([prompt[20:]], cached=[20])
    got = got_logits[0].float()
    scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale
    assert err <= LOGIT_TOL["f16"], err
    if int(first[0]) != int(torch.argmax(want)):
        assert _near_tie(want.cpu().numpy(), err * scale, "f16")
    for l in range(w.cfg.n_layers):
        for c1, c2 in ((one.k_cache[l], chunked.k_cache[l]), (one.v_cache[l], chunked.v_cache[l])):
            assert float((c1.float() - c2.float()).abs().max()) <= 8 * ULP["f16"] * float(c1.float().abs().max()), l
    run = G.GptqRunner(w, batch=2, max_ctx=64, cache_layout="vllm")
    pre = G.GptqPrefill(w, max_tokens=64, runner=run)
    with pytest.raises(ValueError, match="HND"):
        pre.forward_batch([prompt[20:]], cached=[20])
    with pytest.raises(ValueError, match="HND"):
        pre.forward(prompt[20:], cached=20)
    torch.cuda.synchronize()
    assert all(int(c.abs().sum()) == 0 for c in run.k_cache)


# ---------------------------------------------------------------- hand-off to a decode runner
@pytest.mark.parametrize("layout", ["hnd", "vllm"])
def test_hand_off_gives_oracle_greedy_stream(cuda, layout):
    """forward_batch(slots=...) into a captured batch-4 runner, then 6 graph replays: each row's tokens are the
    oracle's greedy stream until a near-tie (after which the two may fork); steps_taken follows the longest context."""
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda, keep_host=True)
    run = G.GptqRunner(w, batch=4, max_ctx=128, cache_layout=layout)
    run.capture()
    pre = G.GptqPrefill(w, max_tokens=128, runner=run)
    prompts = _prompts(w.cfg.vocab, 4, 2, 24, seed=50)
    _, first = pre.forward_batch(prompts, slots=[2, 0, 3, 1])
    assert run.steps_taken == max(len(p) for p in prompts)
    rows = {2: 0, 0: 1, 3: 2, 1: 3}                     # runner row -> sequence
    stream = [first.tolist()]
    for _ in range(6):
        run.replay()
        torch.cuda.synchronize()
        stream.append([int(run.meta["token_ids"][r]) for r in sorted(rows, key=rows.get)])
    run.check_overflow()
    assert run.steps_taken == max(len(p) for p in prompts) + 6
    for i, p in enumerate(prompts):
        r, want = _feed(w, "f16", p)
        pos, logit = len(p), want[-1]
        for step in range(7):
            tok = stream[step][i]
            if tok != int(np.argmax(logit)):
                assert _near_tie(logit, 3e-3 * np.abs(logit).max(), "f16"), (i, step)
                break
            logit = r.step([tok], pos)[0]
            pos += 1


def test_refill_two_slots_between_replays(cuda):
    """After 3 replays at batch 4, two new prompts are admitted into rows 1 and 3, then 3 more replays: rows 0 and 2
    are bit-identical to a run without the admission, rows 1 and 3 to a run that admitted the new prompts first."""
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda)
    B, slots, keep = 4, [1, 3], [0, 2]
    prompts = _prompts(w.cfg.vocab, B, 2, 20, seed=60)
    fresh = _prompts(w.cfg.vocab, 2, 2, 20, seed=61)
    runs = [G.GptqRunner(w, batch=B, max_ctx=128) for _ in range(3)]
    pres = [G.GptqPrefill(w, max_tokens=128, runner=r) for r in runs]
    for r in runs:
        r.capture()
    for pre in pres:
        pre.forward_batch(prompts, slots=range(B))
    pres[2].forward_batch(fresh, slots=slots)

    def replay(r):
        r.replay()
        torch.cuda.synchronize()
        return r.logits().clone()
    for _ in range(3):
        replay(runs[0]), replay(runs[1])
    pres[0].forward_batch(fresh, slots=slots)
    for step in range(3):
        got, plain, ref = replay(runs[0]), replay(runs[1]), replay(runs[2])
        assert torch.equal(got[keep], plain[keep]), step
        assert torch.equal(got[slots], ref[slots]), step


# ---------------------------------------------------------------- rejections
@pytest.mark.parametrize("case", ["n0", "n257", "t_lt_n", "null_x", "null_qkv", "null_tables", "null_layers", "dtype",
                                  "lm_rows", "dest_rows", "paged2", "paged_vllm", "hidden"])
def test_prefill_step_rejects(cuda, case):
    """Each bad field alone gives cudaErrorInvalidValue (1) before anything is launched: the caches stay untouched."""
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda)
    pre = G.GptqPrefill(w, max_tokens=64)
    p, _, keep = pre.make_plan([[1, 2, 3], [4, 5]], [1, 0], _own_tables(2, 1), lm_rows=1)
    s = G._Step.from_buffer_copy(pre.step_struct)
    dummy = torch.zeros(64, dtype=torch.int32, device=cuda)
    if case == "n0":
        p.n_seqs = 0
    elif case == "n257":
        p.n_seqs = 257
    elif case == "t_lt_n":
        p.total_tokens = 1
    elif case == "null_x":
        p.x = None
    elif case == "null_qkv":
        p.q = None
    elif case == "null_tables":
        p.block_tables = None
    elif case == "null_layers":
        s.layers = None
    elif case == "dtype":
        s.act_dtype = 2
    elif case == "lm_rows":
        p.lm_rows = 3
    elif case == "dest_rows":
        p.lm_rows, p.dest_rows = 2, dummy.data_ptr()
    elif case == "paged2":
        p.paged = 2
    elif case == "paged_vllm":
        s.cache_layout = 0
    elif case == "hidden":
        s.hidden = w.cfg.hidden - 4
    torch.cuda.synchronize()
    rc = lib().mrs_gptq_prefill_step(ctypes.byref(s), ctypes.byref(p), _stream())
    torch.cuda.synchronize()
    assert rc == 1, rc
    assert all(int(c.abs().sum()) == 0 for c in pre.k_cache)


def test_python_rejections(cuda):
    """The checks shared with LlamaPrefill raise the same ValueErrors for GPTQ, before anything is launched."""
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda)
    pre = G.GptqPrefill(w, max_tokens=64)
    for args, kw, match in [([], {}, "1..256"), ([[1, 2], [3, 4]], {}, "own tables"),
                            ([[1, 2], [3, 4]], dict(tables=_own_tables(2, 2), slots=[0, 1]), "runner"),
                            ([list(range(40)), list(range(40))], dict(tables=_own_tables(2, 3)), "max_tokens"),
                            ([[1, 2, 512]], {}, "token ids")]:
        with pytest.raises(ValueError, match=match):
            pre.forward_batch(args, **kw)
    with pytest.raises(ValueError, match="GptqPrefill.forward"):
        pre.forward([1])
    run = G.GptqRunner(w, batch=2, max_ctx=32)
    with pytest.raises(ValueError, match="block table"):
        G.GptqPrefill(w, max_tokens=64, runner=run)
    torch.cuda.synchronize()
    assert all(int(c.abs().sum()) == 0 for c in pre.k_cache)


# ---------------------------------------------------------------- real size
def test_mistral_7b_shapes(cuda):
    """Two Mistral-7B GPTQ g128 layers, 8 prompts of 128 tokens in one step: finite, non-degenerate last-row logits
    within the bound of the oracle fed token by token."""
    cfg = G.GptqConfig.mistral_7b(n_layers=2, max_pos=256)
    w = G.GptqWeights(cfg, cuda, keep_host=True)
    B, L = 8, 128
    rng = np.random.default_rng(70)
    prompts = [rng.integers(0, cfg.vocab, size=L).tolist() for _ in range(B)]
    pre = G.GptqPrefill(w, max_tokens=B * L)
    logits, first = pre.forward_batch(prompts, tables=_own_tables(B, L // cfg.block_size))
    got = logits.float().cpu().numpy()
    ref = _oracle(w, "f16")
    for pos in range(L):
        want = ref.step([p[pos] for p in prompts], pos)
    assert np.isfinite(got).all() and np.isfinite(want).all()
    scale = np.abs(want).max()
    assert scale > 1e-3 and np.unique(want).size > 1000 and np.unique(got).size > 1000, "degenerate logits"
    err = np.abs(got - want).max() / scale
    assert err <= LOGIT_TOL["f16"], err
    for b in range(B):
        if int(first[b]) != int(np.argmax(want[b])):
            assert _near_tie(want[b], np.abs(got[b] - want[b]).max(), "f16"), b
    print(f"gptq prefill, Mistral-7B shapes: logit error {err:.2e} of the logit scale")
