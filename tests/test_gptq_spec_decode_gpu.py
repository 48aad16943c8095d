"""Speculative decoding of a GPTQ / AWQ model: mrs_paged_decode_fused_multi_strided (the multi-query fused attention
reading q, k and v inside the q||k||v rows of the fused QKV GEMM), mrs_gptq_verify_step through GptqVerifier against
the CPU oracle and a plain GptqRunner teacher-forced through the same rows, speculative_generate from prompts handed
over by GptqPrefill, graph / PDL bit-identity, overflow, host traffic and Mistral-7B shapes.  The argument checks at the
end run without a GPU."""
import collections
import ctypes
import itertools
import types

import numpy as np
import pytest
import torch

from mistralrs_b200 import gptq_model as G
from mistralrs_b200 import lib
from mistralrs_b200 import model as M
from test_gptq_prefill_gpu import LOGIT_TOL, TDT, _feed, _near_tie, _oracle, _prompts
from test_spec_decode_attn_gpu import _DT, _ptr, run as run_attention, setup as setup_attention
from test_spec_decode_host import accept_np
from test_spec_decode_model_gpu import TIE, truncate


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------- strided multi-query attention
def _ctx(B, q, seed):
    return [q + (37 * b + 11 * seed) % 150 for b in range(B)]     # kv lengths of q .. q + 149, the q new rows included


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("group", [1, 4, 8])
@pytest.mark.parametrize("Q", [2, 4, 8])
def test_strided_multi_query_attention_is_bit_identical(cuda, D, group, Q):
    """the same q, k and v once in contiguous buffers (mrs_paged_decode_fused_multi) and once inside [R, nqkv] q||k||v
    rows (mrs_paged_decode_fused_multi_strided): output and cache writes bit-identical, counters left zero, at B 1, 9
    and 64 in split and unsplit plans"""
    dt = torch.bfloat16 if (D + group + Q) % 2 else torch.float16
    for B, plan in itertools.product((1, 9, 64), ("split", "unsplit")):
        d, meta, *_ = setup_attention(cuda, dt, D, group, Q, 16, _ctx(B, Q, D + group), plan, seed=B + Q)
        H, KVH = meta["H"], meta["KVH"]
        R, nq, nkv = B * Q, H * D, KVH * D
        qkv = torch.cat([d["qt"].view(R, nq), d["kn"].view(R, nkv), d["vn"].view(R, nkv)], dim=1).contiguous()
        kc, vc = d["kc"].clone(), d["vc"].clone()
        out = torch.full_like(d["out"], float("nan"))
        tmp_v = None if d["tmp_v"] is None else torch.zeros_like(d["tmp_v"])
        tmp_s = None if d["tmp_s"] is None else torch.zeros_like(d["tmp_s"])
        counters = torch.zeros_like(d["counters"])
        run_attention("mrs_paged_decode_fused_multi", d, meta, Q)
        rc = lib().mrs_paged_decode_fused_multi_strided(
            _ptr(qkv), ctypes.c_void_p(qkv.data_ptr() + 2 * nq), ctypes.c_void_p(qkv.data_ptr() + 2 * (nq + nkv)),
            _ptr(kc), _ptr(vc), _ptr(d["cos"]), _ptr(d["sin"]), _ptr(d["pos"]), _ptr(d["slots"]), _ptr(d["indptr"]),
            _ptr(d["indices"]), _ptr(d["last"]), _ptr(d["req"]), _ptr(d["tile"]), _ptr(d["o_indptr"]), _ptr(d["chunk"]),
            _ptr(d["mask"]), _ptr(out), _ptr(tmp_v), _ptr(tmp_s), _ptr(counters), B, meta["padded"], H, KVH, D,
            meta["bs"], ctypes.c_float(meta["scale"]), ctypes.c_uint32(_DT[dt]), 0, Q, ctypes.c_int64(qkv.stride(0)),
            ctypes.c_int64(qkv.stride(0)), _stream())
        assert rc == 0, rc
        torch.cuda.synchronize()
        if plan == "split" and B > 1:
            assert meta["padded"] > B
        for a, b in ((d["out"], out), (d["kc"], kc), (d["vc"], vc)):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (B, plan)
        assert torch.isfinite(out).all(), (B, plan)
        assert int(counters.abs().sum()) == 0 and int(d["counters"].abs().sum()) == 0


# ---------------------------------------------------------------- verify rows on the tiny model
def _prefill_ragged(w, run, seed, lo=2, hi=24):
    """ragged prompts handed to every row of `run` by GptqPrefill.forward_batch(slots=...), a few rows per call:
    (prompts, first tokens)"""
    prompts = _prompts(w.cfg.vocab, run.B, lo, hi, seed)
    pre = G.GptqPrefill(w, max_tokens=run.max_ctx, runner=run)
    first = []
    per_call = max(1, run.max_ctx // hi)
    for i in range(0, run.B, per_call):
        _, f = pre.forward_batch(prompts[i:i + per_call], slots=list(range(i, min(i + per_call, run.B))))
        first += f.tolist()
    assert run.context_lens.cpu().tolist() == [len(p) for p in prompts]
    return prompts, first


def _models(cuda, dt, B, seed, max_ctx=128):
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda, dtype=TDT[dt], keep_host=True)
    run = G.GptqRunner(w, batch=B, max_ctx=max_ctx)
    plain = G.GptqRunner(w, batch=B, max_ctx=max_ctx)     # plain decode teacher-forced through the same rows
    prompts, first = _prefill_ragged(w, run, seed)
    assert _prefill_ragged(w, plain, seed) == (prompts, first)
    return w, run, plain, prompts, first


def _plain_rows(plain, ctx, fed):
    """plain decode of fed[b][0..q-1] from context ctx[b]: logits [B, q, vocab]"""
    plain.context_lens.copy_(torch.tensor(ctx, dtype=torch.int32))
    rows = []
    for i in range(len(fed[0])):
        plain.set_tokens([f[i] for f in fed])
        plain.advance(); plain.forward()
        rows.append(plain.logits().float().cpu().numpy())
    return np.stack(rows, axis=1)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("B", [1, 4, 32, 33])
@pytest.mark.parametrize("q", [2, 4, 8])
def test_verify_rows_match_oracle_and_plain_decode(cuda, dt, B, q):
    w, run, plain, prompts, anchors = _models(cuda, dt, B, seed=3 * B + q)
    cfg, k, tol = w.cfg, q - 1, LOGIT_TOL[dt]
    refs = [_feed(w, dt, p)[0] for p in prompts]       # the oracle after each prompt
    ctx = [len(p) for p in prompts]
    ver = G.GptqVerifier(run, draft_len=k)
    ver.sync_from_runner()
    worst = 0.0
    for step in range(3):
        # the greedy continuation of the plain runner (its cache rows past the context are overwritten below)
        plain.context_lens.copy_(torch.tensor(ctx, dtype=torch.int32))
        plain.set_tokens(anchors)
        greedy = []
        for i in range(k):
            plain.advance(); plain.forward()
            greedy.append(plain.meta["token_ids"].cpu().tolist())
        drafts, fed = [], []
        for b in range(B):
            mode = (b + step) % 3                    # greedy / wrong from a position on / all wrong
            d = [greedy[i][b] for i in range(k)]
            if mode == 1:
                j = (b // 3) % k
                d[j:] = [(t + 1) % cfg.vocab for t in d[j:]]
            elif mode == 2:
                d = [(t + 7) % cfg.vocab for t in d]
            drafts.append(d)
            fed.append([anchors[b]] + d)
        ver.set_drafts(drafts)
        ver.step()
        torch.cuda.synchronize()
        got = ver.logits().float().cpu().numpy().reshape(B, q, -1)
        acc, em = ver.fetch()
        assert np.isfinite(got).all()
        # the kernels' own argmax through the greedy rule: accepted, emitted, rolled-back lengths, next anchors
        want_acc, want_em, want_ctx, want_rows = accept_np(got.argmax(axis=2).reshape(-1), np.array(fed).reshape(-1),
                                                           [0] * B, [c + q for c in ctx], q)
        assert acc == want_acc.tolist() and sum(em, []) == want_em.tolist(), step
        assert run.context_lens.cpu().tolist() == want_ctx.tolist(), step
        assert ver.meta["token_ids"].cpu().tolist() == want_rows.tolist(), step
        ref_plain = _plain_rows(plain, ctx, fed)
        for b in range(B):
            want = np.stack([refs[b].step([fed[b][i]], ctx[b] + i)[0] for i in range(q)])   # teacher-forced
            scale = np.abs(want).max()
            errs = np.abs(got[b] - want).max(axis=1) / scale
            worst = max(worst, errs.max())
            assert (errs <= tol).all(), (step, b, errs)
            assert np.abs(got[b] - ref_plain[b]).max() / scale <= tol, (step, b)
            # the greedy rule on the oracle's choices, unless a row up to the decision is a near-tie
            want_a = 0
            while want_a < k and fed[b][want_a + 1] == int(np.argmax(want[want_a])):
                want_a += 1
            if not any(_near_tie(want[i], errs[i] * scale, dt) for i in range(min(want_a + 1, q))):
                assert acc[b] == want_a, (step, b, acc[b], want_a)
            ctx[b] += 1 + acc[b]
            truncate(refs[b], ctx[b])                # the rejected rows leave the oracle too
            anchors[b] = em[b][acc[b]]
        if B >= 3:
            assert len(set(acc)) > 1, acc           # sequences accept different numbers of drafts
        if step == 1:                                # a plain step of the whole batch between verify steps
            ver.sync_to_runner()
            run.step()
            torch.cuda.synchronize()
            got1 = run.logits().float().cpu().numpy()
            ref1 = _plain_rows(plain, ctx, [[a] for a in anchors])[:, 0]
            for b in range(B):
                want1 = refs[b].step([anchors[b]], ctx[b])[0]
                scale = np.abs(want1).max()
                assert np.abs(got1[b] - want1).max() / scale <= tol, (step, b)
                assert np.abs(got1[b] - ref1[b]).max() / scale <= tol, (step, b)
                ctx[b] += 1
            anchors = run.meta["token_ids"].cpu().tolist()
            ver.sync_from_runner()
    assert run.context_lens.cpu().tolist() == ctx
    assert int(run.error_flag.item()) == 0
    assert int(ver.buf["attn_counters"].abs().sum()) == 0
    print(f"gptq verify {dt} B={B} q={q}: worst logit error {worst:.3e} of the scale")


# ---------------------------------------------------------------- generation from prompts
def _plain_greedy(w, B, seed, n, max_ctx):
    """the B-row runner's own greedy streams after the prompts: (prompts, first tokens, tokens [B][n], top-2 margins)"""
    run = G.GptqRunner(w, batch=B, max_ctx=max_ctx)
    prompts, first = _prefill_ragged(w, run, seed, hi=12)
    toks, margins = [[] for _ in range(B)], [[] for _ in range(B)]
    for _ in range(n):
        run.step()
        lg = run.logits().float().cpu().numpy()
        for b, t in enumerate(run.meta["token_ids"].cpu().tolist()):
            toks[b].append(t)
            top2 = np.sort(lg[b])[-2:]
            margins[b].append((top2[1] - top2[0]) / np.abs(lg[b]).max())
    return prompts, first, toks, margins


@pytest.mark.gpu
@pytest.mark.parametrize("B,k", [(16, 3), (4, 7)])
def test_speculative_generate_from_prompts_matches_plain_greedy(cuda, B, k):
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda)
    vocab, n, seed, max_ctx = w.cfg.vocab, 40, 80 + B, 256
    prompts, first, plain, margins = _plain_greedy(w, B, seed, n, max_ctx)
    calls = itertools.count()

    def propose(history):
        # drafts from the plain trajectory: correct, wrong from a seeded position, or all wrong; speculative_generate
        # asks for sequences 0 .. B-1 in order, once per step
        b = next(calls) % B
        at = len(history) - 1
        rng = np.random.default_rng(1000 * b + at)
        d = [plain[b][at + i] if at + i < n else 0 for i in range(k)]
        mode = rng.integers(0, 3)
        if mode == 1:
            j = int(rng.integers(0, k))
            d[j:] = [(t + 1) % vocab for t in d[j:]]
        elif mode == 2:
            d = [(t + 7) % vocab for t in d]
        return d

    run = G.GptqRunner(w, batch=B, max_ctx=max_ctx)
    assert _prefill_ragged(w, run, seed, hi=12) == (prompts, first)
    ver = G.GptqVerifier(run, draft_len=k)
    streams, steps = M.speculative_generate(ver, first, n, propose)
    assert len(steps) < n
    counts = np.array(steps)
    assert (counts >= 0).all() and (counts <= k).all()
    assert (counts != counts[:, :1]).any()                     # accepted counts differ between sequences
    for b in range(B):
        for i, (x, y) in enumerate(zip(streams[b], plain[b])):
            if x != y:    # only a near-tie of the plain step may flip a token (then the trajectories part)
                assert margins[b][i] <= TIE, (b, i, x, y)
                break


@pytest.mark.gpu
def test_generate_host_traffic_at_256_sequences(cuda):
    """per step: one H2D copy of the drafts, one graph launch, one D2H copy of the results (plus, before the loop, the
    first tokens' H2D copy and the D2D copy that hands the anchors to the verifier).  The CUDA runtime calls are counted
    exactly.  The device's copy records are only bounded: in a long-running process the profiler's device timestamps
    drift from the host's by about 1 ms per 100 s and some copy records go missing (the runtime calls stay complete)."""
    w = G.GptqWeights(G.GptqConfig.tiny_test(n_layers=1), cuda)
    B, k = 256, 3
    run = G.GptqRunner(w, batch=B, max_ctx=64)
    ver = G.GptqVerifier(run, draft_len=k)
    ver.capture()
    first = [(5 * b + 1) % w.cfg.vocab for b in range(B)]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        streams, steps = M.speculative_generate(ver, first, 6, lambda h: [h[-1]] * k)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    n = len(steps)
    assert sum(s.startswith("cudaMemcpy") for s in names) == 2 * n + 2, names
    assert sum(s == "cudaGraphLaunch" for s in names) == n
    kinds = collections.Counter(s.split(" (")[0] for s in names if s.startswith("Memcpy "))
    assert set(kinds) <= {"Memcpy HtoD", "Memcpy DtoH", "Memcpy DtoD"}, kinds
    assert kinds["Memcpy HtoD"] <= n + 1 and kinds["Memcpy DtoH"] <= n and kinds["Memcpy DtoD"] <= 1, kinds
    assert all(len(s) == 6 for s in streams)


# ---------------------------------------------------------------- bit-identity
def _random_caches(run, seed):
    gen = torch.Generator(device=run.dev).manual_seed(seed)
    for c in run.k_cache + run.v_cache:
        c.copy_(torch.randn(c.shape, generator=gen, device=run.dev).to(c.dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("B,k", [(16, 3), (33, 7)])
def test_graph_and_pdl_bit_identical(cuda, B, k):
    """eager steps on the PDL chain, eager steps with skip_mask bit 2 (plain stream order) and graph replays of the
    chain give the same logits, results, lengths and anchors, bit for bit; a plain step in between too"""
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda, dtype=torch.bfloat16)
    vocab = w.cfg.vocab
    lens = [20 + 7 * b % 90 for b in range(B)]
    pairs = []
    for chain in (True, False, True):
        r = G.GptqRunner(w, batch=B, max_ctx=256)
        _random_caches(r, 1)
        r.reset(lens)
        r.set_tokens([(13 * b + 2) % vocab for b in range(B)])
        v = G.GptqVerifier(r, k)
        if not chain:
            r.step_struct.skip_mask = v.step_struct.skip_mask = 4
        v.sync_from_runner()
        pairs.append((r, v))
    assert pairs[0][0].padded_tiles > B, "expected a split-KV plan"
    pairs[2][1].capture()
    rng = np.random.default_rng(0)
    for step in range(5):
        drafts = rng.integers(0, vocab, size=(B, k)).tolist()
        if step % 2:                                 # propose what the last step emitted: partial accepts
            em = pairs[0][1].fetch()[1]
            drafts = [[t if t >= 0 else 0 for t in e[1:]] for e in em]
        for i, (r, v) in enumerate(pairs):
            v.set_drafts(drafts)
            if i == 2:
                v.replay()
            else:
                v.step()
        torch.cuda.synchronize()
        (r0, v0) = pairs[0]
        for r, v in pairs[1:]:
            assert torch.equal(v0.logits(), v.logits()), step
            assert torch.equal(v0.results, v.results), step
            assert torch.equal(r0.context_lens, r.context_lens), step
            assert torch.equal(v0.meta["token_ids"], v.meta["token_ids"]), step
        if step == 2:                                # and a plain step in between, also identical
            for r, v in pairs:
                v.sync_to_runner(); r.step(); v.sync_from_runner()
            torch.cuda.synchronize()
            assert all(torch.equal(r0.logits(), r.logits()) for r, _ in pairs[1:])
    for r, v in pairs:
        assert int(r.error_flag.item()) == 0 and int(v.buf["attn_counters"].abs().sum()) == 0


# ---------------------------------------------------------------- overflow
@pytest.mark.gpu
def test_overflow_freezes_one_sequence(cuda):
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda)
    B, k = 12, 3
    run = G.GptqRunner(w, batch=B, max_ctx=32)
    ver = G.GptqVerifier(run, draft_len=k)
    run.set_tokens([3 + b for b in range(B)]); ver.sync_from_runner()
    lens = [10 + b for b in range(B)]
    lens[4] = 29                                     # 29 + 4 rows > 32: sequence 4 is frozen
    run.context_lens.copy_(torch.tensor(lens, dtype=torch.int32))
    caches = [c.clone() for c in run.k_cache + run.v_cache]
    ver.set_drafts([[1, 2, 3]] * B)
    ver.step()
    torch.cuda.synchronize()
    acc, em = ver.fetch()
    assert acc[4] == -1 and em[4] == [-1] * (k + 1)
    assert all(acc[b] >= 0 for b in range(B) if b != 4)
    assert int(run.context_lens[4]) == 29 and int(run.error_flag.item()) & 1
    assert int(ver.meta["token_ids"][4 * (k + 1)]) == 7                # the frozen sequence keeps its anchor
    bs = w.cfg.block_size
    own = {run.tables[b][p // bs] * bs + p % bs for b in range(B) if b != 4 for p in range(lens[b], lens[b] + k + 1)}
    for before, after in zip(caches, run.k_cache + run.v_cache):
        changed = (before != after).any(dim=-1).any(dim=1)           # [blocks, slots in a block]
        slots = {int(b) * bs + int(o) for b, o in torch.nonzero(changed).tolist()}
        assert slots <= own, sorted(slots - own)


# ---------------------------------------------------------------- real size
@pytest.mark.gpu
def test_mistral_7b_shapes_verify(cuda):
    """two Mistral-7B GPTQ g128 layers, B = 32, q = 4 (128 rows through every GEMM): finite, non-degenerate logits on
    every row, against a plain runner teacher-forced through the same rows and the oracle.  With synthetic weights the
    attention scores at these shapes are large, so at a two-key context a one-ulp difference in q or k moves a row's
    logits by several times the decode bound, in plain decode as much as in the verify step.  So a row is within the
    bound of the oracle, or no further from it than twice plain decode's own distance on that row (and so no further
    from plain decode than three times that distance); the same argmax as plain decode off near-ties."""
    cfg = G.GptqConfig.mistral_7b(n_layers=2, max_pos=64)
    w = G.GptqWeights(cfg, cuda, keep_host=True)
    B, q = 32, 4
    run = G.GptqRunner(w, batch=B, max_ctx=32)
    plain = G.GptqRunner(w, batch=B, max_ctx=32)
    ver = G.GptqVerifier(run, draft_len=q - 1)
    rng = np.random.default_rng(9)
    fed = rng.integers(0, cfg.vocab, size=(B, q))
    run.set_tokens(fed[:, 0].tolist()); ver.sync_from_runner()
    ver.set_drafts(fed[:, 1:].tolist())
    ver.step()
    torch.cuda.synchronize()
    got = ver.logits().float().cpu().numpy().reshape(B, q, -1)
    acc, em = ver.fetch()
    ref_plain = _plain_rows(plain, [0] * B, fed.tolist())
    ref = _oracle(w, "f16")
    want = np.stack([ref.step(fed[:, i].tolist(), i) for i in range(q)], axis=1)   # every sequence starts at 0
    assert np.isfinite(got).all() and np.isfinite(ref_plain).all() and np.isfinite(want).all()
    scale = np.abs(want).max()
    assert scale > 1e-3 and np.unique(want).size > 1000 and np.unique(got).size > 1000, "degenerate logits"
    tol = LOGIT_TOL["f16"]
    for i in range(q):
        err = np.abs(got[:, i] - want[:, i]).max() / scale
        plain_err = np.abs(ref_plain[:, i] - want[:, i]).max() / scale
        diff = np.abs(got[:, i] - ref_plain[:, i]).max() / scale
        print(f"row {i}: verify {err:.2e}, plain {plain_err:.2e} of the logit scale from the oracle; apart {diff:.2e}")
        assert err <= max(tol, 2 * plain_err), (i, err, plain_err)
        assert diff <= max(tol, 3 * plain_err), (i, diff, plain_err)
        for b in range(B):
            if int(got[b, i].argmax()) != int(ref_plain[b, i].argmax()):
                assert _near_tie(ref_plain[b, i], np.abs(got[b, i] - ref_plain[b, i]).max(), "f16"), (i, b)
    want_acc, want_em, want_ctx, _ = accept_np(got.argmax(axis=2).reshape(-1), fed.reshape(-1), [0] * B, [q] * B, q)
    assert acc == want_acc.tolist() and sum(em, []) == want_em.tolist()
    assert run.context_lens.cpu().tolist() == want_ctx.tolist()


# ---------------------------------------------------------------- argument checks (no GPU)
def _stub(B=16, head_dim=64, dt=torch.float16, layout="hnd", max_ctx=64):
    return types.SimpleNamespace(B=B, cfg=G.GptqConfig.tiny_test(head_dim=head_dim), dt=dt, layout=layout, max_ctx=max_ctx)


def test_gptq_verifier_args_at_every_batch():
    for B in range(1, 257):
        for k in range(1, 8):
            assert G.check_gptq_verifier_args(_stub(B=B), k) == k


@pytest.mark.parametrize("kw,k,msg", [
    ({}, 8, "draft_len must be 1..7"), (dict(B=1), 0, "draft_len"), (dict(layout="vllm"), 3, "HND"),
    (dict(head_dim=96), 3, "head_dim"), (dict(head_dim=256), 1, "head_dim"), (dict(dt=torch.float32), 3, "f16 / bf16"),
    (dict(max_ctx=7), 7, "shorter than one verify step"), (dict(B=256, max_ctx=1), 1, "shorter than one verify step")])
def test_gptq_verifier_rejects_before_any_allocation(kw, k, msg):
    # the stub runner has no device state at all: reaching an allocation or a launch would fail differently
    with pytest.raises(ValueError, match=msg):
        G.GptqVerifier(_stub(**kw), draft_len=k)


def test_gptq_verify_step_rejects_bad_arguments():
    """mrs_gptq_verify_step returns cudaErrorInvalidValue before any launch; every case differs from a well-formed
    two-layer batch-16 step in one field (the device pointers are never dereferenced)"""
    L = lib()
    bufs = (ctypes.c_int32 * 64)()
    p = lambda i: ctypes.addressof(bufs) + 4 * i
    layers = (G._Layer * 2)()

    def call(q_len=4, ctx=True, acc=True, em=True, **fields):
        s = G._Step()
        s.batch, s.n_layers, s.head_dim, s.cache_layout, s.act_dtype, s.hidden = 16, 2, 128, 1, 1, 4096
        s.layers = ctypes.cast(layers, ctypes.POINTER(G._Layer))
        s.token_ids, s.out_token = p(0), p(8)
        for n, v in fields.items():
            setattr(s, n, v)
        return L.mrs_gptq_verify_step(ctypes.byref(s), q_len, ctypes.c_void_p(p(24) if ctx else 0),
                                      ctypes.c_void_p(p(32) if acc else 0), ctypes.c_void_p(p(40) if em else 0), None)

    bad = [dict(batch=0), dict(batch=257), dict(q_len=1), dict(q_len=9), dict(q_len=0), dict(cache_layout=0),
           dict(head_dim=96), dict(head_dim=256), dict(act_dtype=2), dict(act_dtype=3), dict(hidden=4092),
           dict(layers=None), dict(n_layers=0), dict(out_token=p(0)), dict(ctx=False), dict(acc=False), dict(em=False)]
    for kw in bad:
        assert call(**kw) == 1, kw
