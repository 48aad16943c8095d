"""Speculative decoding end to end (LlamaVerifier / mrs_llama_verify_step) on the tiny Llama-shaped model against the
CPU oracle: every verify row's logits match the oracle teacher-forced through the same rows, drafts are accepted by the
greedy rule, rejected rows are rolled back, and speculative generation gives the tokens of plain greedy decoding."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.model import OracleLlama
from mistralrs_b200 import lib, model as M
from test_spec_decode_host import accept_np

pytestmark = pytest.mark.gpu

TOL = 4.1 * 2.0 ** -7          # logit error bound of the decode parity tests (bf16 logits)
TIE = 4 * 2.0 ** -7            # top-2 margin below which an argmax may legitimately flip


def truncate(ref, n):
    """roll the oracle's dense cache back to its first n rows"""
    for l in range(len(ref.k)):
        ref.k[l] = ref.k[l][:n]; ref.v[l] = ref.v[l][:n]


def near_tie(logits, scale, err=0.0):
    """top-2 margin within the bf16 tie margin, or within twice the row's own error against the oracle"""
    top2 = np.sort(logits)[-2:]
    return top2[1] - top2[0] <= max(TIE, 2 * err) * scale


def make(cuda, quant, B, max_ctx=64):
    # the layer counts of the decode parity test (test_model_gpu.py), whose error bound TOL is
    cfg = M.LlamaConfig.tiny_test(quant=quant, n_layers=8 if quant == "q4_k_m" else 2)
    w = M.LlamaWeights(cfg, cuda, keep_host=True)
    run = M.LlamaRunner(w, batch=B, max_ctx=max_ctx)
    cos, sin = M.rope_tables(cfg)
    refs = [OracleLlama(cfg, w.host, M.tensor_type, cos, sin, "bf16") for _ in range(B)]
    return cfg, w, run, refs


@pytest.mark.parametrize("quant", ["q4_k_m", "q8_0"])
@pytest.mark.parametrize("B,q", [(1, 2), (1, 4), (1, 8), (2, 2), (2, 4)])
def test_verify_logits_acceptance_and_rollback(cuda, quant, B, q):
    cfg, w, run, refs = make(cuda, quant, B)
    k = q - 1
    ver = M.LlamaVerifier(run, draft_len=k)
    plain = M.LlamaRunner(w, batch=B, max_ctx=64)   # plain decode teacher-forced through the same rows
    anchors = [17, 900][:B]
    ctx = [0] * B
    run.set_tokens(anchors)
    ver.sync_from_runner()
    # per step and sequence: None = the oracle's greedy continuation, j = wrong from draft j on, "all" = all wrong
    patterns = [[None, None], [k // 2, 0], ["all", None], [None, k - 1], [0, "all"], [None, None]]
    worst = 0.0
    for step, pat in enumerate(patterns):
        drafts, fed = [], []
        for b in range(B):
            ref = refs[b]
            tok, greedy = anchors[b], []
            for i in range(k):                       # the oracle's greedy continuation, then roll back
                tok = int(np.argmax(ref.step([tok], ctx[b] + i)[0])); greedy.append(tok)
            truncate(ref, ctx[b])
            p = pat[b % 2]
            d = list(greedy)
            if p == "all":
                d = [(t + 1) % cfg.vocab for t in greedy]
            elif p is not None:
                d[p] = (greedy[p] + 1) % cfg.vocab
            drafts.append(d)
            fed.append([anchors[b]] + d)
        ver.set_drafts(drafts)
        ver.step()
        torch.cuda.synchronize()
        got = ver.logits().float().cpu().numpy().reshape(B, q, -1)
        acc, em = ver.fetch()
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
            plain_errs = np.abs(ref_plain[b] - want).max(axis=1) / scale
            worst = max(worst, errs.max())
            # every row within the decode parity bound, or (the synthetic Q8_0 model drifts past it on longer
            # trajectories, plain decode included) no worse than plain decode of the same row plus 4 ulp
            assert ((errs <= TOL) | (errs <= plain_errs + 4 * 2.0 ** -8)).all(), (step, b, errs, plain_errs)
            assert np.abs(got[b] - ref_plain[b]).max() / scale <= TOL, (step, b)
            # the greedy rule on the oracle's choices, unless a row up to the decision is a near-tie
            want_a = 0
            while want_a < k and fed[b][want_a + 1] == int(np.argmax(want[want_a])):
                want_a += 1
            if not any(near_tie(want[i], scale, errs[i]) for i in range(min(want_a + 1, q))):
                assert acc[b] == want_a, (step, b, acc[b], want_a)
                assert em[b][acc[b]] == int(np.argmax(want[acc[b]])), (step, b)
            a = acc[b]
            assert em[b][:a + 1] == [int(t) for t in got[b][:a + 1].argmax(axis=1)]
            assert all(t == -1 for t in em[b][a + 1:])
            if pat[b % 2] is None:
                assert a == k or any(near_tie(want[i], scale, errs[i]) for i in range(q)), (step, b, a)
            ctx[b] += 1 + a
            truncate(refs[b], ctx[b])                # the rejected rows leave the oracle too
            anchors[b] = em[b][a]
        assert run.context_lens.cpu().tolist() == ctx
        assert run.error_flag.item() == 0
        if step % 2 == 1:                            # mix in a plain decode step on the same sequences
            ver.sync_to_runner()
            run.step()
            torch.cuda.synchronize()
            got1 = run.logits().float().cpu().numpy()
            plain.context_lens.copy_(torch.tensor(ctx, dtype=torch.int32))
            plain.set_tokens(anchors)
            plain.advance(); plain.forward()        # the reference runner's cache takes the same row
            d1 = (plain.logits().float() - run.logits().float()).abs().max().item()
            assert d1 <= TOL * run.logits().float().abs().max().item(), (step, d1)
            for b in range(B):
                want1 = refs[b].step([anchors[b]], ctx[b])[0]
                if quant == "q4_k_m":
                    assert np.abs(got1[b] - want1).max() <= TOL * np.abs(want1).max(), (step, b)
                ctx[b] += 1
            anchors = run.meta["token_ids"].cpu().tolist()
            ver.sync_from_runner()
    print(f"{quant} B={B} q={q}: worst logit error {worst / 2.0 ** -8:.2f} ulp of the logit scale")


def _plain_greedy(cuda, w, B, first, n):
    run = M.LlamaRunner(w, batch=B, max_ctx=96)
    run.set_tokens(first)
    toks, margins = [[] for _ in range(B)], [[] for _ in range(B)]
    for _ in range(n):
        run.step()
        lg = run.logits().float().cpu().numpy()
        for b, t in enumerate(run.meta["token_ids"].cpu().tolist()):
            toks[b].append(t)
            top2 = np.sort(lg[b])[-2:]
            margins[b].append((top2[1] - top2[0]) / np.abs(lg[b]).max())
    return toks, margins


@pytest.mark.parametrize("quant,B,k", [("q4_k_m", 2, 3), ("q8_0", 1, 7), ("q4_k_m", 1, 1)])
def test_speculative_generate_matches_plain_greedy(cuda, quant, B, k):
    cfg = M.LlamaConfig.tiny_test(quant=quant)
    w = M.LlamaWeights(cfg, cuda)
    first, n = [17, 900][:B], 48
    plain, margins = _plain_greedy(cuda, w, B, first, n)

    def propose(history):
        # drafts from the plain trajectory: correct, wrong from a seeded position, or all wrong; the two sequences
        # start from different tokens and so see different corruption, hence different accept counts
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

    run = M.LlamaRunner(w, batch=B, max_ctx=512)     # a sequence that accepts more runs ahead of the other
    ver = M.LlamaVerifier(run, draft_len=k)
    streams, steps = M.speculative_generate(ver, first, n, propose)
    assert len(steps) < n                            # drafts were accepted
    counts = np.array(steps)
    assert (counts >= 0).all() and (counts <= k).all()
    if B == 2:
        assert (counts[:, 0] != counts[:, 1]).any()
    for b in range(B):
        for i, (x, y) in enumerate(zip(streams[b], plain[b])):
            if x != y:    # only a bf16 near-tie of the plain step may flip a token (then the trajectories part)
                assert margins[b][i] <= TIE, (b, i, x, y)
                break


def test_graph_replay_matches_eager(cuda):
    cfg = M.LlamaConfig.tiny_test(quant="q4_k_m")
    w = M.LlamaWeights(cfg, cuda)
    B, k = 2, 3
    eager_r, graph_r = M.LlamaRunner(w, batch=B, max_ctx=64), M.LlamaRunner(w, batch=B, max_ctx=64)
    eager, graph = M.LlamaVerifier(eager_r, k), M.LlamaVerifier(graph_r, k)
    for r, v in ((eager_r, eager), (graph_r, graph)):
        r.set_tokens([5, 77]); v.sync_from_runner()
    graph.capture()
    rng = np.random.default_rng(0)
    for step in range(6):
        acc = eager.fetch()[1] if step else None
        drafts = rng.integers(0, cfg.vocab, size=(B, k)).tolist()
        if step % 2 == 0 and step:               # sometimes propose what the last step emitted (partial accepts)
            drafts = [[t if t >= 0 else 0 for t in e[1:]] for e in acc]
        eager.set_drafts(drafts); graph.set_drafts(drafts)
        eager.step(); graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(eager.logits(), graph.logits())
        assert torch.equal(eager.results, graph.results)
        assert torch.equal(eager_r.context_lens, graph_r.context_lens)
        assert torch.equal(eager.meta["token_ids"], graph.meta["token_ids"])


def test_overflow_freezes_the_sequence(cuda):
    cfg = M.LlamaConfig.tiny_test(quant="q8_0", n_layers=1)
    w = M.LlamaWeights(cfg, cuda)
    run = M.LlamaRunner(w, batch=2, max_ctx=32)
    ver = M.LlamaVerifier(run, draft_len=3)
    run.set_tokens([3, 4]); ver.sync_from_runner()
    run.context_lens.copy_(torch.tensor([29, 10], dtype=torch.int32))     # 29 + 4 rows > 32: sequence 0 is frozen
    caches = [c.clone() for c in run.k_cache + run.v_cache]
    ver.set_drafts([[1, 2, 3], [1, 2, 3]])
    ver.step()
    torch.cuda.synchronize()
    acc, em = ver.fetch()
    assert acc[0] == -1 and em[0] == [-1] * 4 and acc[1] >= 0
    assert run.context_lens.cpu().tolist()[0] == 29 and run.error_flag.item() & 1
    assert ver.meta["token_ids"][0].item() == 3                            # the frozen sequence keeps its anchor
    # sequence 0 wrote nothing; sequence 1 wrote only its own rows 10..13
    bs = cfg.block_size
    own = {run.tables[1][p // bs] * bs + p % bs for p in range(10, 14)}
    for before, after in zip(caches, run.k_cache + run.v_cache):
        changed = (before != after).reshape(before.shape[0], before.shape[1], bs, -1).any(dim=-1).any(dim=1)
        slots = {int(b) * bs + int(o) for b, o in torch.nonzero(changed).tolist()}
        assert slots <= own, sorted(slots - own)


def test_spec_accept_matches_restatement(cuda):
    rng = np.random.default_rng(7)
    for B, q in ((1, 2), (3, 4), (8, 8), (5, 3)):
        am = rng.integers(0, 6, size=B * q).astype(np.int32)
        rows = rng.integers(0, 6, size=B * q).astype(np.int32)
        rows[:q] = np.concatenate([[9], am[:q - 1]])                     # sequence 0 accepts everything
        slots = rng.integers(0, 100, size=B * q).astype(np.int64)
        if B > 2:
            slots[2 * q] = -1                                            # sequence 2 was frozen
        ctx = rng.integers(q, 200, size=B).astype(np.int32)
        want = accept_np(am, rows, slots[::q], ctx, q)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
        d_am, d_rows, d_slots, d_ctx = t(am), t(rows), t(slots), t(ctx)
        d_acc, d_em = torch.zeros(B, dtype=torch.int32, device=cuda), torch.zeros(B * q, dtype=torch.int32, device=cuda)
        P = lambda x: ctypes.c_void_p(x.data_ptr())
        rc = lib().mrs_spec_accept(P(d_am), P(d_rows), P(d_slots), P(d_ctx), P(d_acc), P(d_em), B, q, 0,
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0
        torch.cuda.synchronize()
        for got, w in zip((d_acc, d_em, d_ctx, d_rows), want):
            assert got.cpu().tolist() == list(map(int, w)), (B, q)
