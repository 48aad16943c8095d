"""The prompt chunk plan (host/prompt_chunks.hpp through kv_index) and LlamaPrefill.forward_batch's argument checks:
no GPU needed."""
import types

import numpy as np
import pytest
import torch

from mistralrs_b200 import kv_index as K
from mistralrs_b200 import model as M


# ---------------------------------------------------------------- the reference's text-only unit tests, case by case
def test_block_align_splits_the_prompt_tail():
    assert K.build_prompt_chunk_plan(65, 0, 4096, 32) == [(0, 64), (64, 65)]
    assert K.build_prompt_chunk_plan(64, 0, 4096, 32) == [(0, 64)]          # already aligned: no extra chunk
    assert K.build_prompt_chunk_plan(20, 0, 4096, 32) == [(0, 20)]          # shorter than one block: no split
    assert K.build_prompt_chunk_plan(6712, 0, 4096, 32) == [(0, 4096), (4096, 6688), (6688, 6712)]
    assert K.build_prompt_chunk_plan(65, 0, 4096, None) == [(0, 65)]


def test_chunk_groups_do_not_mix_final_and_nonfinal_sequences():
    plans = [[(0, 4)], [(0, 2), (2, 4)]]
    assert K.next_prompt_chunk_group([0, 0], plans) == ([0], True)
    assert K.next_prompt_chunk_group([1, 0], plans) == ([1], False)


def test_uniform_chunk_group_separates_unequal_final_tails():
    plans = [[(0, 4), (4, 5)], [(0, 4), (4, 7)]]
    assert K.next_prompt_chunk_group([1, 1], plans, False) == ([0, 1], True)
    assert K.next_prompt_chunk_group([1, 1], plans, True) == ([0], True)


def test_chunk_size_and_exhausted_plans():
    assert K.prompt_chunk_size(5, 32) == 6 and K.prompt_chunk_size(64, 4096) == 64
    assert K.prompt_chunk_size(8192, 4096) == 1 and K.prompt_chunk_size(0, 4096) == 4096
    assert K.next_prompt_chunk_group([1, 2], [[(0, 4)], [(0, 2), (2, 4)]]) is None
    assert K.next_prompt_chunk_group([], []) is None
    assert K.build_prompt_chunk_plan(10, 10, 4) == [] and K.build_prompt_chunk_plan(10, 12, 4) == []


# ---------------------------------------------------------------- properties of random plans
@pytest.mark.parametrize("seed", range(8))
def test_random_plans(seed):
    rng = np.random.default_rng(seed)
    for _ in range(200):
        total = int(rng.integers(0, 3000))
        prefix = int(rng.integers(0, total + 2))
        size = int(rng.integers(1, 600))
        align = [None, 8, 16, 32][int(rng.integers(0, 4))]
        plan = K.build_prompt_chunk_plan(total, prefix, size, align)
        pos = min(prefix, total)
        for s, e in plan:                       # chunks tile [prefix, total) in order, without gaps
            assert s == pos and pos < e <= pos + size
            unaligned = min(pos + size, total)
            if align and e != unaligned:        # shortened only to the block start inside the chunk
                a = unaligned // align * align
                assert e == a and pos < a < unaligned
            pos = e
        assert pos == max(min(prefix, total), total)
    for _ in range(100):
        n = int(rng.integers(1, 9))
        plans = [K.build_prompt_chunk_plan(int(rng.integers(1, 200)), 0, int(rng.integers(1, 50)), 16) for _ in range(n)]
        idx = [int(rng.integers(0, len(p) + 1)) for p in plans]
        uniform = bool(rng.integers(0, 2))
        g = K.next_prompt_chunk_group(idx, plans, uniform)
        left = [i for i in range(n) if idx[i] < len(plans[i])]
        if not left:
            assert g is None
            continue
        members, final = g
        assert members and members[0] == left[0] and members == sorted(members)
        q0 = plans[left[0]][idx[left[0]]]
        for i in left:                          # homogeneous in finality (and length when asked); nobody left out
            same = (idx[i] + 1 == len(plans[i])) == final
            if uniform:
                c = plans[i][idx[i]]
                same = same and c[1] - c[0] == q0[1] - q0[0]
            assert (i in members) == same, (i, members)


# ---------------------------------------------------------------- forward_batch's argument checks
def _prefill(max_tokens=64, runner=None):
    """A LlamaPrefill with its host-side state only (no weights, no device cache): enough to reach the checks."""
    pre = M.LlamaPrefill.__new__(M.LlamaPrefill)
    pre.cfg = M.LlamaConfig.tiny_test()
    pre.w, pre.dev, pre.dt = None, torch.device("cpu"), torch.bfloat16
    pre.max_tokens = max_tokens
    pre.table = list(range(1, -(-max_tokens // pre.cfg.block_size) + 1))
    if runner is not None:
        pre.runner = runner
    return pre


def _runner(B=4, blocks=4):
    return types.SimpleNamespace(B=B, max_blocks=blocks, tables=[list(range(1 + blocks * b, 1 + blocks * (b + 1)))
                                                                  for b in range(B)])


T2 = [[1, 2, 3], [4, 5]]
TAB2 = [[1, 2], [3, 4]]


@pytest.mark.parametrize("args,kw,match", [
    ([], {}, "1..256"),
    ([[1, 2]] * 257, {}, "1..256"),
    ([list(range(40)), list(range(40))], dict(tables=[[1, 2, 3], [4, 5, 6]]), "max_tokens"),
    ([[1, 2], []], dict(tables=TAB2), "sequence 1"),
    ([[1, 2], [3]], dict(tables=TAB2), "sequence 1"),
    ([[1, 2], [3]], dict(tables=TAB2, cached=[0, -1]), "sequence 1"),
    ([[1, 2, 3], list(range(30))], dict(tables=TAB2, cached=[0, 5]), "exceeds"),
    ([[1, 2], [3, 4]], dict(tables=[[1], [2, 3]], cached=[510, 0]), "exceeds"),
    (T2, dict(tables=TAB2, cached=[0]), "cached lengths"),
    (T2, dict(tables=[[1, 2]]), "tables for 2"),
    (T2, {}, "own tables"),
    (T2, dict(tables=[[1, 2], [2, 3]], cached=[16, 0]), "same cache slot"),
    (T2, dict(tables=[[1, 2], [1, 2]]), "same cache slot"),
    ([[1, 2, 1024], [4, 5]], dict(tables=TAB2), "token ids"),
    ([[1, 2, -1], [4, 5]], dict(tables=TAB2), "token ids"),
    ([[1.5, 2.0], [4, 5]], dict(tables=TAB2), "token ids"),
    (T2, dict(tables=TAB2, slots=[0, 1]), "runner"),
])
def test_forward_batch_rejects(args, kw, match):
    with pytest.raises(ValueError, match=match):
        _prefill().forward_batch(args, **kw)


@pytest.mark.parametrize("kw,match", [
    (dict(slots=[0]), "1 slots for 2"),
    (dict(slots=[1, 1]), "distinct"),
    (dict(slots=[0, 4]), "distinct"),
    (dict(slots=[-1, 0]), "distinct"),
    (dict(slots=[0, 1], final=False), "non-final"),
    (dict(slots=[0, 1], tables=[[1], [5, 6]]), "exceeds"),
])
def test_forward_batch_rejects_bad_slots(kw, match):
    with pytest.raises(ValueError, match=match):
        _prefill(runner=_runner()).forward_batch([[1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17], [4, 5]], **kw)


def test_forward_batch_accepts_good_arguments():
    """the checks pass through valid calls (the launch itself needs a GPU)"""
    pre = _prefill(runner=_runner())
    ids, cached, tables, slots = pre.check_batch_args(T2, tables=TAB2, cached=[16, 0])
    assert [a.tolist() for a in ids] == T2 and cached == [16, 0] and tables == TAB2 and slots is None
    _, _, tables, slots = pre.check_batch_args(T2, slots=(3, 1))
    assert slots == [3, 1] and tables == [_runner().tables[3], _runner().tables[1]]
    _, _, tables, _ = pre.check_batch_args([[1, 2]])
    assert tables == [pre.table]
