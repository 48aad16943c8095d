"""Speculative decoding on the host side (no GPU): the greedy acceptance rule restated in numpy and checked against
hand-built cases of the reference's verifier (mistralrs-core/src/speculative/verifier.rs:198-291), and the argument
checks of LlamaVerifier, which must raise before anything is launched."""
import types

import numpy as np
import pytest
import torch

from mistralrs_b200 import model as M


def accept_np(argmax, rows, slot0, ctx_after_advance, q):
    """Restatement of mrs_spec_accept.  argmax / rows: [B*q] (rows = [anchor, drafts] per sequence), slot0: [B] slot of
    each sequence's first row (< 0: frozen by the advance), ctx_after_advance: [B] context_lens as the advance left
    them.  Returns (accepted [B], emitted [B*q], context_lens [B], rows with the next anchors)."""
    argmax, rows = np.asarray(argmax).reshape(-1, q), np.array(rows).reshape(-1, q)
    B = argmax.shape[0]
    acc, em, ctx = np.full(B, -1), np.full((B, q), -1), np.array(ctx_after_advance).copy()
    for b in range(B):
        if slot0[b] < 0:
            continue
        a = 0
        while a < q - 1 and rows[b, a + 1] == argmax[b, a]:
            a += 1
        acc[b] = a
        em[b, :a + 1] = argmax[b, :a + 1]
        ctx[b] += 1 + a - q
        rows[b, 0] = argmax[b, a]
    return acc, em.reshape(-1), ctx, rows.reshape(-1)


def test_all_drafts_accepted():
    # k = 3 drafts that are exactly the target's greedy choices: all accepted, k + 1 tokens out (the bonus token)
    acc, em, ctx, rows = accept_np([11, 12, 13, 14], [10, 11, 12, 13], [5], [24], 4)
    assert acc.tolist() == [3] and em.tolist() == [11, 12, 13, 14] and ctx.tolist() == [24] and rows[0] == 14


def test_first_draft_rejected():
    # the first draft disagrees: only the target's own token is emitted and the context keeps the anchor alone
    acc, em, ctx, rows = accept_np([7, 12, 13], [10, 8, 12], [5], [23], 3)
    assert acc.tolist() == [0] and em.tolist() == [7, -1, -1] and ctx.tolist() == [21] and rows[0] == 7


def test_rejection_in_the_middle_and_per_sequence_counts():
    argmax = [1, 2, 9, 4, 5, 6]
    rows = [0, 1, 2, 3, 4, 5]          # sequence 0: drafts 1, 2 -> a = 2; sequence 1: drafts 4, 5 vs argmax 4, 5 -> a = 2
    acc, em, ctx, rows2 = accept_np(argmax, rows, [0, 16], [10, 40], 3)
    assert acc.tolist() == [2, 2] and em.tolist() == [1, 2, 9, 4, 5, 6] and ctx.tolist() == [10, 40]
    acc, em, ctx, rows2 = accept_np([1, 7, 9, 4, 5, 6], [0, 1, 2, 3, 9, 5], [0, 16], [10, 40], 3)
    assert acc.tolist() == [1, 0] and em.tolist() == [1, 7, -1, 4, -1, -1] and ctx.tolist() == [9, 38]
    assert rows2[0] == 7 and rows2[3] == 4


def test_frozen_sequence_emits_nothing():
    acc, em, ctx, rows = accept_np([1, 2, 3, 4], [0, 1, 3, 4], [-1, 8], [30, 12], 2)
    assert acc.tolist() == [-1, 0] and em.tolist() == [-1, -1, 3, -1] and ctx.tolist() == [30, 11]
    assert rows.tolist() == [0, 1, 3, 4]


def _runner(B=1, head_dim=64, dt=torch.bfloat16, tp=1, fused=1, max_ctx=64, peer=None, ar=None):
    cfg = M.LlamaConfig.tiny_test(head_dim=head_dim)
    return types.SimpleNamespace(B=B, cfg=cfg, dt=dt, w=types.SimpleNamespace(tp_size=tp), _peer=peer, _ar_cb=ar,
                                 step_struct=types.SimpleNamespace(fused_attention=fused), max_ctx=max_ctx)


@pytest.mark.parametrize("kw,k,msg", [
    (dict(B=2), 4, "exceeds the 8 rows"), (dict(B=1), 8, "draft_len must be 1..7"), (dict(B=1), 0, "draft_len"),
    (dict(tp=2), 1, "single-GPU"), (dict(peer=object()), 1, "single-GPU"), (dict(ar=object()), 1, "single-GPU"),
    (dict(head_dim=96), 1, "head_dim"), (dict(dt=torch.float32), 1, "f16 / bf16"), (dict(fused=0), 1, "fused attention"),
    (dict(max_ctx=3), 3, "shorter than one verify step")])
def test_verifier_rejects_bad_arguments_before_any_launch(kw, k, msg):
    # the stub runner has no device state at all: reaching an allocation or a launch would fail differently
    with pytest.raises(ValueError, match=msg):
        M.LlamaVerifier(_runner(**kw), draft_len=k)
    assert M.check_verifier_args(_runner(B=2), 3) == 3


def test_drafts_are_checked():
    assert M.check_drafts([[1, 2], [3, 4]], 2, 2, 10).dtype == torch.int32
    for bad in ([[1, 2]], [[1, 2, 3], [4, 5, 6]], [[1, 2], [3, 10]], [[-1, 2], [3, 4]]):
        with pytest.raises(ValueError):
            M.check_drafts(bad, 2, 2, 10)
    with pytest.raises(ValueError):
        M.check_drafts(torch.zeros(2, 2, dtype=torch.float32), 2, 2, 10)
