"""Speculative decoding for batches of 9..256 sequences: verify steps on the dequant-GEMM chain (the route of the
runner's own plain step above 8 sequences), with B*q rows through every linear and mrs_paged_decode_fused_multi over
the B sequences.  The oracle is the exact-GEMM one of the batched decode tests, teacher-forced through the same rows.
The argument checks at the end run without a GPU."""
import ctypes

import numpy as np
import pytest
import torch

from mistralrs_b200 import lib, model as M
from oracle.model import OracleLlama
from test_batched_decode_gpu import LOGIT_TOL, Q8_0_LOGIT_TOL, TDT, _cfg, _near_tie, _oracles, _prefill_ragged
from test_spec_decode_attn_gpu import test_multi_query_attention_matches_fp64 as check_multi_query_attention
from test_spec_decode_host import _runner, accept_np
from test_spec_decode_model_gpu import TIE, _plain_greedy, truncate


# ---------------------------------------------------------------- attention at batched verify shapes
def _ragged(B, q, seed):
    return [q + (37 * b + 11 * seed) % 150 for b in range(B)]     # kv lengths of q .. q + 149, the q new rows included


ATTN_CASES = [  # (dtype, D, group, q, page, B, plan)
    (torch.bfloat16, 128, 4, 4, 16, 9, "split"), (torch.float16, 64, 8, 8, 16, 9, "unsplit"),
    (torch.float16, 64, 1, 2, 8, 9, "split"), (torch.bfloat16, 64, 1, 2, 16, 16, "split"),
    (torch.float16, 128, 1, 4, 8, 16, "unsplit"), (torch.bfloat16, 128, 8, 8, 32, 16, "split"),
    (torch.float16, 64, 4, 2, 16, 64, "split"), (torch.bfloat16, 64, 8, 4, 16, 64, "unsplit"),
    (torch.float16, 128, 4, 8, 16, 64, "split"), (torch.bfloat16, 128, 1, 2, 32, 64, "unsplit"),
    (torch.bfloat16, 64, 4, 8, 8, 64, "split"), (torch.float16, 128, 8, 2, 16, 16, "unsplit"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dt,D,group,q,bs,B,plan", ATTN_CASES)
def test_multi_query_attention_at_batched_shapes(cuda, dt, D, group, q, bs, B, plan):
    """the fp64 causal reference, cache writes bit-identical to RoPE + reshape_and_cache, NaN in every cache row the
    kernel must not read; split plans of more than one sequence merge through the counters"""
    check_multi_query_attention(cuda, dt, D, group, q, bs, _ragged(B, q, group + D), plan)


# ---------------------------------------------------------------- verify rows on tiny models
def _models(cuda, quant_, dt, B, seed, max_ctx=64):
    w = M.LlamaWeights(_cfg(quant_, dt), cuda, dtype=TDT[dt], keep_host=True)
    run = M.LlamaRunner(w, batch=B, max_ctx=max_ctx, pdl=True)
    plain = M.LlamaRunner(w, batch=B, max_ctx=max_ctx, pdl=True)   # plain decode teacher-forced through the same rows
    prompts = _prefill_ragged(w, run, B, seed)
    assert _prefill_ragged(w, plain, B, seed) == prompts
    return w, run, plain, prompts


# every (B, q) on both models, each model in one dtype; the other dtype of each on the anti-diagonal of B x q
VERIFY_CASES = ([(quant_, dt, B, q) for quant_, dt in (("q4_k_m", "bf16"), ("q8_0", "f16"))
                 for B in (9, 16, 33) for q in (2, 4, 8)] +
                [(quant_, dt, B, q) for quant_, dt in (("q4_k_m", "f16"), ("q8_0", "bf16"))
                 for B, q in ((9, 8), (16, 4), (33, 2))])


@pytest.mark.gpu
@pytest.mark.parametrize("quant_,dt,B,q", VERIFY_CASES)
def test_verify_rows_match_oracle_and_plain_decode(cuda, quant_, dt, B, q):
    w, run, plain, prompts = _models(cuda, quant_, dt, B, seed=B + q)
    cfg, k = w.cfg, q - 1
    refs = _oracles(w, prompts, dt)
    ver = M.LlamaVerifier(run, draft_len=k)
    anchors = [p[-1] for p in prompts]
    ctx = [len(p) - 1 for p in prompts]
    run.set_tokens(anchors)
    ver.sync_from_runner()
    tol = Q8_0_LOGIT_TOL if quant_ == "q8_0" else LOGIT_TOL
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
        plain.context_lens.copy_(torch.tensor(ctx, dtype=torch.int32))
        ref_plain = []
        for i in range(q):
            plain.set_tokens([fed[b][i] for b in range(B)])
            plain.advance(); plain.forward()
            ref_plain.append(plain.logits().float().cpu().numpy())
        ref_plain = np.stack(ref_plain, axis=1)
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
        assert len(set(acc)) > 1, acc               # sequences accept different numbers of drafts
        if step == 1:                                # a plain step of the whole batch between verify steps
            ver.sync_to_runner()
            run.step()
            torch.cuda.synchronize()
            got1 = run.logits().float().cpu().numpy()
            plain.context_lens.copy_(torch.tensor(ctx, dtype=torch.int32))
            plain.set_tokens(anchors)
            plain.advance(); plain.forward()
            ref1 = plain.logits().float().cpu().numpy()
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
    print(f"{quant_} {dt} B={B} q={q}: worst logit error {worst:.3e} of the scale")


# ---------------------------------------------------------------- generation
@pytest.mark.gpu
@pytest.mark.parametrize("quant_,B,k", [("q4_k_m", 16, 3), ("q8_0", 9, 7)])
def test_speculative_generate_matches_plain_greedy(cuda, quant_, B, k):
    cfg = M.LlamaConfig.tiny_test(quant=quant_)
    w = M.LlamaWeights(cfg, cuda)
    first, n = [(17 + 61 * b) % cfg.vocab for b in range(B)], 40
    plain, margins = _plain_greedy(cuda, w, B, first, n)       # the B-sequence runner's own greedy streams

    def propose(history):
        # drafts from the plain trajectory: correct, wrong from a seeded position, or all wrong
        b = first.index(history[0])
        at = len(history) - 1
        rng = np.random.default_rng(1000 * history[0] + at)
        d = [plain[b][at + i] if at + i < n else 0 for i in range(k)]
        mode = rng.integers(0, 3)
        if mode == 1:
            j = int(rng.integers(0, k))
            d[j:] = [(t + 1) % cfg.vocab for t in d[j:]]
        elif mode == 2:
            d = [(t + 7) % cfg.vocab for t in d]
        return d

    run = M.LlamaRunner(w, batch=B, max_ctx=512)
    ver = M.LlamaVerifier(run, draft_len=k)
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
    """per step: one H2D copy of the drafts, one graph launch, one D2H copy of the results (plus the first tokens'
    H2D copy before the loop)"""
    cfg = M.LlamaConfig.tiny_test(quant="q8_0", n_layers=1)
    w = M.LlamaWeights(cfg, cuda)
    B, k = 256, 3
    run = M.LlamaRunner(w, batch=B, max_ctx=64)
    ver = M.LlamaVerifier(run, draft_len=k)
    ver.capture()
    first = [(5 * b + 1) % cfg.vocab for b in range(B)]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        streams, steps = M.speculative_generate(ver, first, 6, lambda h: [h[-1]] * k)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    n = len(steps)
    assert sum("Memcpy HtoD" in s for s in names) == n + 1, names
    assert sum("Memcpy DtoH" in s for s in names) == n
    assert sum(s == "cudaGraphLaunch" for s in names) == n
    assert all(len(s) == 6 for s in streams)


# ---------------------------------------------------------------- bit-identity
def _random_caches(run, seed):
    gen = torch.Generator(device=run.dev).manual_seed(seed)
    for c in run.k_cache + run.v_cache:
        c.copy_(torch.randn(c.shape, generator=gen, device=run.dev).to(c.dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("B,k", [(16, 3), (33, 7)])
def test_graph_and_pdl_bit_identical(cuda, B, k):
    w = M.LlamaWeights(_cfg("q4_k_m", "bf16"), cuda)
    vocab = w.cfg.vocab
    lens = [20 + 7 * b % 90 for b in range(B)]
    pairs = []
    for pdl in (False, True, True):
        r = M.LlamaRunner(w, batch=B, max_ctx=256, pdl=pdl)
        _random_caches(r, 1)
        r.reset(lens)
        r.set_tokens([(13 * b + 2) % vocab for b in range(B)])
        v = M.LlamaVerifier(r, k)
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
    for r, _ in pairs:
        assert int(r.error_flag.item()) == 0 and int(r.buf["attn_counters"].abs().sum()) == 0


# ---------------------------------------------------------------- overflow
@pytest.mark.gpu
def test_overflow_freezes_one_sequence(cuda):
    w = M.LlamaWeights(_cfg("q8_0", "bf16"), cuda)
    B, k = 12, 3
    run = M.LlamaRunner(w, batch=B, max_ctx=32)
    ver = M.LlamaVerifier(run, draft_len=k)
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
def test_llama3_8b_shapes_verify(cuda):
    """two real-size Q4_K_M layers (layer 1 keeps attn_v / ffn_down in Q6_K) and the Q6_K lm_head, B = 16, q = 4,
    every row against the exact-GEMM oracle teacher-forced through the same rows"""
    cfg = M.LlamaConfig.llama3_8b(n_layers=2, max_pos=64)
    w = M.LlamaWeights(cfg, cuda, dtype=torch.bfloat16, keep_host=True)
    B, q = 16, 4
    run = M.LlamaRunner(w, batch=B, max_ctx=32, pdl=True)
    ver = M.LlamaVerifier(run, draft_len=q - 1)
    cos, sin = M.rope_tables(cfg)
    ref = OracleLlama(cfg, w.host, M.tensor_type, cos, sin, "bf16", exact_gemm=True)
    rng = np.random.default_rng(8)
    fed = rng.integers(0, cfg.vocab, size=(B, q))
    run.set_tokens(fed[:, 0].tolist()); ver.sync_from_runner()
    ver.set_drafts(fed[:, 1:].tolist())
    ver.step()
    torch.cuda.synchronize()
    got = ver.logits().float().cpu().numpy().reshape(B, q, -1)
    acc, em = ver.fetch()
    for i in range(q):                               # every sequence starts at 0: row i of all of them is at position i
        want = ref.step(fed[:, i].tolist(), i)
        assert np.isfinite(want).all()
        scale = np.abs(want).max()
        assert scale > 1e-3 and np.unique(want).size > 1000, "degenerate logits"
        err = np.abs(got[:, i] - want).max() / scale
        assert err <= LOGIT_TOL, (i, err)
        for b in range(B):
            if int(got[b, i].argmax()) != int(np.argmax(want[b])):
                assert _near_tie(want[b], np.abs(got[b, i] - want[b]).max(), "bf16"), (i, b)
    want_acc, want_em, want_ctx, _ = accept_np(got.argmax(axis=2).reshape(-1), fed.reshape(-1), [0] * B, [q] * B, q)
    assert acc == want_acc.tolist() and sum(em, []) == want_em.tolist()
    assert run.context_lens.cpu().tolist() == want_ctx.tolist()


# ---------------------------------------------------------------- argument checks (no GPU)
def test_verifier_args_at_batched_sizes():
    for B in (9, 10, 16, 33, 64, 128, 256):
        for k in range(1, 8):
            assert M.check_verifier_args(_runner(B=B), k) == k
    for B in range(1, 9):                            # up to 8 sequences: the GEMV route's 8 rows, as before
        for k in range(1, 8):
            if B * (k + 1) > 8:
                with pytest.raises(ValueError, match="exceeds the 8 rows"):
                    M.check_verifier_args(_runner(B=B), k)
            else:
                assert M.check_verifier_args(_runner(B=B), k) == k


@pytest.mark.parametrize("kw,k,msg", [
    (dict(B=16), 8, "draft_len must be 1..7"), (dict(B=9), 0, "draft_len"), (dict(B=16, tp=2), 3, "single-GPU"),
    (dict(B=64, peer=object()), 1, "single-GPU"), (dict(B=256, ar=object()), 7, "single-GPU"),
    (dict(B=16, head_dim=96), 3, "head_dim"), (dict(B=33, dt=torch.float32), 3, "f16 / bf16"),
    (dict(B=16, fused=0), 3, "fused attention"), (dict(B=16, max_ctx=7), 7, "shorter than one verify step")])
def test_batched_verifier_rejects_before_any_allocation(kw, k, msg):
    # the stub runner has no device state at all: reaching an allocation or a launch would fail differently
    with pytest.raises(ValueError, match=msg):
        M.LlamaVerifier(_runner(**kw), draft_len=k)


def test_verify_step_rejects_bad_arguments():
    """mrs_llama_verify_step returns cudaErrorInvalidValue before any launch; every case differs from a well-formed
    batch-16 step in one field (the pointers are never dereferenced)"""
    L = lib()
    bufs = (ctypes.c_int32 * 64)()
    p = lambda i: ctypes.addressof(bufs) + 4 * i

    def call(q_len=4, ctx=True, acc=True, em=True, **fields):
        s = M._Step()
        s.batch, s.head_dim, s.fused_attention, s.act_dtype = 16, 128, 1, 1
        s.token_ids, s.out_token, s.h = p(0), p(8), p(16)
        for n, v in fields.items():
            setattr(s, n, v)
        return L.mrs_llama_verify_step(ctypes.byref(s), q_len, ctypes.c_void_p(p(24) if ctx else 0),
                                       ctypes.c_void_p(p(32) if acc else 0), ctypes.c_void_p(p(40) if em else 0), None)

    bad = [dict(q_len=1), dict(q_len=9), dict(q_len=0), dict(h=None), dict(act_dtype=2), dict(act_dtype=3),
           dict(fused_attention=0), dict(head_dim=96), dict(head_dim=256), dict(out_token=p(0)), dict(ctx=False),
           dict(acc=False), dict(em=False), dict(batch=257), dict(batch=0),
           dict(batch=2, q_len=5), dict(batch=8, q_len=2)]           # up to 8 sequences: still at most 8 rows
    for kw in bad:
        assert call(**kw) == 1, kw
    ctx_ = M._TpCtx()
    assert call(tp=ctypes.addressof(ctx_)) == 1
    assert call(all_reduce=M._AR_FN(lambda *a: None)) == 1
