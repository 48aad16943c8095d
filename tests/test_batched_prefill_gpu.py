"""Batched prompt prefill: `LlamaPrefill.forward_batch` runs the prompts of up to 256 sequences through one
`mrs_llama_prefill_step`, and can hand them to a decode runner's rows on the device."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from mistralrs_b200 import GGML, kv_index, lib
from mistralrs_b200 import model as M
from oracle.model import OracleLlama

TDT = {"bf16": torch.bfloat16, "f16": torch.float16}
ULP = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11}
LOGIT_TOL = 2e-2     # test_prefill_composition_matches_oracle: the prefill GEMM chain vs the exact-GEMM oracle
# The synthetic Q8_0 model amplifies small perturbations: its exact-GEMM and Q8_1 oracles differ by 4-6 % of the logit
# scale over a few steps.  Against the rounded-weight oracle below, f32-vs-f64 accumulation alone reaches ~2.4 % over
# the longer ragged trajectories, so that model gets the wider bound (still below its own oracles' spread).
Q8_0_LOGIT_TOL = 3e-2


def _cfg(quant_, dt, **kw):
    if (quant_, dt) == ("q4_k_m", "f16"):        # the default synthetic block scales overflow f16 in this model
        kw["synth_scale_exp"] = (-15, -13)
    return M.LlamaConfig.tiny_test(quant=quant_, n_layers=2, **kw)


class RoundedWeightOracle(OracleLlama):
    """OracleLlama(exact_gemm=True) whose linears take the weights rounded once to the activation format, as the
    dequant GEMM's MMA operands are (see test_batched_decode_gpu.py)."""

    def _gemv(self, layer, name, x, rows, cols):
        cache = self.__dict__.setdefault("_w16", {})
        key = (layer, name)
        if key not in cache:
            ty = self.tt(self.cfg, name, layer)
            w = oracle.dequantize(ty, self.hw[key]).reshape(rows, cols).astype(np.float32)
            cache[key] = oracle.round_dtype(w, self.dt).astype(np.float64)
        y = np.asarray(x, dtype=np.float64) @ cache[key].T
        return oracle.round_dtype(y.astype(np.float32), self.dt)


def _oracle(w, dt):
    cos, sin = M.rope_tables(w.cfg)
    cls = RoundedWeightOracle if w.cfg.quant == "q8_0" else OracleLlama
    return cls(w.cfg, w.host, M.tensor_type, cos, sin, dt, exact_gemm=True)


def _near_tie(want_row, err, dt):
    top2 = np.sort(want_row)[-2:]
    return top2[1] - top2[0] <= max(8 * ULP[dt] * np.abs(want_row).max(), 2 * err)


def _prompts(vocab, n, lo, hi, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, vocab, size=int(rng.integers(lo, hi + 1))).tolist() for _ in range(n)]


def _own_tables(n, blocks):
    """disjoint tables of `blocks` blocks in a prefill's own cache (block 0 is the null block)"""
    return [list(range(1 + blocks * i, 1 + blocks * (i + 1))) for i in range(n)]


# ---------------------------------------------------------------- one pass == one sequence at a time
@pytest.mark.gpu
@pytest.mark.parametrize("quant_", ["q4_k_m", "q8_0"])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("n,lo,hi", [(1, 2, 40), (3, 2, 40), (8, 2, 40), (9, 2, 40), (33, 2, 40), (64, 33, 64)])
def test_batch_matches_one_at_a_time(cuda, quant_, dt, n, lo, hi):
    """Each GEMM row and each sequence's attention are computed on their own, so every sequence's K/V rows in every
    layer are bit-identical to n separate `forward` calls into identical tables, and so are the last-row logits where
    the lm_head takes the same route (n <= 8).  The 64-sequence case has more than 2048 rows: separate QKV and gate / up
    GEMMs there, grouped launches in the one-sequence calls."""
    w = M.LlamaWeights(_cfg(quant_, dt), cuda, dtype=TDT[dt])
    prompts = _prompts(w.cfg.vocab, n, lo, hi, seed=100 + n)
    tables = _own_tables(n, 4)
    a, b = (M.LlamaPrefill(w, max_tokens=64 * max(n, 2)) for _ in range(2))
    logits, first = a.forward_batch(prompts, tables=tables)
    singles = torch.stack([b.forward(p, table=t) for p, t in zip(prompts, tables)])
    torch.cuda.synchronize()
    for l in range(w.cfg.n_layers):
        assert torch.equal(a.k_cache[l], b.k_cache[l]) and torch.equal(a.v_cache[l], b.v_cache[l]), l
    assert torch.equal(first, torch.argmax(logits.float(), dim=-1).to(torch.int32).cpu())
    assert torch.isfinite(logits.float()).all()
    if n <= M.MMVQ_MAX_BATCH:
        assert torch.equal(logits, singles)
    else:   # the dequant-GEMM lm_head against the MMVQ one: same hidden rows, different lm_head numerics
        scale = singles.float().abs().max()
        assert float((logits.float() - singles.float()).abs().max() / scale) < LOGIT_TOL


# ---------------------------------------------------------------- against the oracle, with cached prefixes
@pytest.mark.gpu
@pytest.mark.parametrize("quant_", ["q4_k_m", "q8_0"])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("n", [9, 33, 64])
def test_ragged_batch_with_prefixes_matches_oracle(cuda, quant_, dt, n):
    """Ragged prompts; every third sequence has its first rows in the cache from an earlier, non-final call, so the
    second call runs the paged prompt attention.  Last-row logits against the oracle teacher-forced through each prompt;
    first tokens equal its argmax except at near-ties."""
    w = M.LlamaWeights(_cfg(quant_, dt), cuda, dtype=TDT[dt], keep_host=True)
    rng = np.random.default_rng(200 + n)
    lens = [(4, 9, 14, 20)[i % 4] for i in rng.permutation(n)]      # four lengths: one batched oracle per length
    prompts = [rng.integers(0, w.cfg.vocab, size=L).tolist() for L in lens]
    tables = _own_tables(n, 2)
    pre = M.LlamaPrefill(w, max_tokens=32 * n)
    pref = {i: len(p) // 2 for i, p in enumerate(prompts) if i % 3 == 0 and len(p) // 2 >= 2}
    assert pre.forward_batch([prompts[i][:c] for i, c in pref.items()], tables=[tables[i] for i in pref], final=False) is None
    cached = [pref.get(i, 0) for i in range(n)]
    logits, first = pre.forward_batch([p[c:] for p, c in zip(prompts, cached)], cached=cached, tables=tables)
    got = logits.float().cpu().numpy()
    tol = Q8_0_LOGIT_TOL if quant_ == "q8_0" else LOGIT_TOL
    for L in sorted(set(lens)):
        group = [i for i in range(n) if lens[i] == L]
        r = _oracle(w, dt)
        for pos in range(L):
            wants = r.step([prompts[i][pos] for i in group], pos)
        for i, want in zip(group, wants):
            scale = np.abs(want).max()
            err = np.abs(got[i] - want).max() / scale
            assert err <= tol, (i, cached[i], L, err)
            if int(first[i]) != int(np.argmax(want)):
                assert _near_tie(want, err * scale, dt), (i, int(first[i]), int(np.argmax(want)))


# ---------------------------------------------------------------- hand-off to a decode runner
def _runner_pair(w, B):
    runs = [M.LlamaRunner(w, batch=B, max_ctx=512, pdl=True) for _ in range(2)]
    for r in runs:
        r.capture()
    return runs


@pytest.mark.gpu
@pytest.mark.parametrize("B", [16, 4])
def test_hand_off_to_runner_matches_old_path(cuda, B):
    """forward_batch(slots=range(B)) fills a captured runner on the device; 8 replays give logits bit-identical to the
    old path: per-sequence forward into the runner's tables, reset(lengths), set_tokens(first tokens)."""
    w = M.LlamaWeights(_cfg("q4_k_m", "bf16"), cuda, dtype=torch.bfloat16)
    new, old = _runner_pair(w, B)
    prompts = _prompts(w.cfg.vocab, B, 2, 30, seed=300 + B)
    _, first = M.LlamaPrefill(w, max_tokens=512, runner=new).forward_batch(prompts, slots=range(B))
    assert new.steps_taken == max(len(p) for p in prompts)
    pre_old = M.LlamaPrefill(w, max_tokens=512, runner=old)
    for b, p in enumerate(prompts):
        pre_old.forward(p, table=old.tables[b])
    old.reset([len(p) for p in prompts])
    old.set_tokens(first.tolist())
    assert torch.equal(new.context_lens, old.context_lens) and torch.equal(new.meta["token_ids"], old.meta["token_ids"])
    for step in range(8):
        new.replay()
        old.replay()
        torch.cuda.synchronize()
        assert torch.equal(new.logits(), old.logits()), step
    assert int(new.error_flag.item()) == 0


@pytest.mark.gpu
def test_refill_two_slots_between_replays(cuda):
    """After 4 replays at batch 16, two new prompts are admitted into slots 3 and 7, then 4 more replays.  The other 14
    rows' logits are bit-identical to a run without the admission; rows 3 and 7 match a fresh run of the new prompts."""
    w = M.LlamaWeights(_cfg("q4_k_m", "bf16"), cuda, dtype=torch.bfloat16)
    B, slots = 16, [3, 7]
    prompts = _prompts(w.cfg.vocab, B, 2, 20, seed=400)
    fresh = _prompts(w.cfg.vocab, 2, 2, 20, seed=401)
    runs = [M.LlamaRunner(w, batch=B, max_ctx=512, pdl=True) for _ in range(3)]
    pres = [M.LlamaPrefill(w, max_tokens=512, runner=r) for r in runs]
    for r in runs:
        r.capture()
    for pre in pres:
        pre.forward_batch(prompts, slots=range(B))
    pres[2].forward_batch(fresh, slots=slots)          # the fresh run: the new prompts admitted before any replay
    keep = [b for b in range(B) if b not in slots]

    def replay(r):
        r.replay()
        torch.cuda.synchronize()
        return r.logits().clone()
    for _ in range(4):
        replay(runs[0]), replay(runs[1])
    pres[0].forward_batch(fresh, slots=slots)
    for step in range(4):
        got, plain, ref = replay(runs[0]), replay(runs[1]), replay(runs[2])
        assert torch.equal(got[keep], plain[keep]), step
        assert torch.equal(got[slots], ref[slots]), step


# ---------------------------------------------------------------- chunked prompts under a token budget
@pytest.mark.gpu
def test_chunked_under_budget_matches_one_shot(cuda):
    """Five prompts of 20..100 tokens through the prompt chunk plan at a 32-token budget, one forward_batch per chunk
    group: the final chunks' logits and the caches match a one-shot prefill within the oracle bound, and the decode
    that follows gives the same greedy tokens except at near-ties."""
    w = M.LlamaWeights(_cfg("q4_k_m", "bf16"), cuda, dtype=torch.bfloat16)
    B, budget, bs = 5, 32, w.cfg.block_size
    prompts = _prompts(w.cfg.vocab, B, 20, 100, seed=500)
    chunked, one = (M.LlamaRunner(w, batch=B, max_ctx=512, pdl=True) for _ in range(2))
    pre_c, pre_o = M.LlamaPrefill(w, max_tokens=512, runner=chunked), M.LlamaPrefill(w, max_tokens=512, runner=one)
    size = kv_index.prompt_chunk_size(B, budget)
    plans = [kv_index.build_prompt_chunk_plan(len(p), 0, size, bs) for p in prompts]
    idx, last, first_c, groups = [0] * B, [None] * B, [None] * B, 0
    while (g := kv_index.next_prompt_chunk_group(idx, plans)) is not None:
        members, final = g
        chunks = [plans[i][idx[i]] for i in members]
        out = pre_c.forward_batch([prompts[i][s:e] for i, (s, e) in zip(members, chunks)], cached=[s for s, _ in chunks],
                                  tables=[chunked.tables[i] for i in members], final=final)
        assert sum(e - s for s, e in chunks) <= budget
        if final:
            for j, i in enumerate(members):
                last[i], first_c[i] = out[0][j].float(), int(out[1][j])
        for i in members:
            idx[i] += 1
        groups += 1
    assert groups > max(len(p) for p in prompts) // size and all(x is not None for x in last)
    logits_o, first_o = pre_o.forward_batch(prompts, slots=range(B))
    scale = logits_o.float().abs().max()
    assert float((torch.stack(last) - logits_o.float()).abs().max() / scale) <= LOGIT_TOL
    for l in range(w.cfg.n_layers):
        for kc, ko in ((chunked.k_cache[l], one.k_cache[l]), (chunked.v_cache[l], one.v_cache[l])):
            assert float((kc.float() - ko.float()).abs().max()) <= 4 * ULP["bf16"] * float(ko.float().abs().max()), l
    chunked.reset([len(p) for p in prompts])
    chunked.set_tokens(first_c)
    for b in range(B):
        if first_c[b] != int(first_o[b]):
            assert _near_tie(logits_o[b].float().cpu().numpy(), LOGIT_TOL * float(scale), "bf16"), b
    one.set_tokens(first_c)             # continue both from the same tokens, so a near-tie flip above does not fork them
    for step in range(4):
        chunked.step()
        one.step()
        want = one.logits().float().cpu().numpy()
        got_ids, want_ids = chunked.meta["token_ids"].cpu().tolist(), one.meta["token_ids"].cpu().tolist()
        err = float(np.abs(chunked.logits().float().cpu().numpy() - want).max())
        for b in range(B):
            if got_ids[b] != want_ids[b]:
                assert _near_tie(want[b], err, "bf16"), (step, b)
        chunked.set_tokens(want_ids)


# ---------------------------------------------------------------- real size
@pytest.mark.gpu
def test_llama3_8b_shapes_batched_prefill(cuda):
    """Two Llama-3-8B Q4_K_M layers (layer 1 keeps attn_v / ffn_down in Q6_K) plus the Q6_K lm_head: 16 prompts of 16
    tokens in one step, against the exact-GEMM oracle (which dequantises every weight again at each of its steps, so
    the prompts are kept short)."""
    cfg = M.LlamaConfig.llama3_8b(n_layers=2, max_pos=128)
    w = M.LlamaWeights(cfg, cuda, dtype=torch.bfloat16, keep_host=True)
    B, L = 16, 16
    rng = np.random.default_rng(600)
    prompts = [rng.integers(0, cfg.vocab, size=L).tolist() for _ in range(B)]
    pre = M.LlamaPrefill(w, max_tokens=B * L)
    logits, first = pre.forward_batch(prompts, tables=_own_tables(B, L // cfg.block_size))
    got = logits.float().cpu().numpy()
    cos, sin = M.rope_tables(cfg)
    ref = OracleLlama(cfg, w.host, M.tensor_type, cos, sin, "bf16", exact_gemm=True)
    for pos in range(L):
        want = ref.step([p[pos] for p in prompts], pos)
    assert np.isfinite(got).all() and np.isfinite(want).all()
    scale = np.abs(want).max()
    assert scale > 1e-3 and np.unique(want).size > 1000, "degenerate logits"
    assert np.abs(got - want).max() / scale <= LOGIT_TOL
    for b in range(B):
        if int(first[b]) != int(np.argmax(want[b])):
            assert _near_tie(want[b], np.abs(got[b] - want[b]).max(), "bf16"), b


# ---------------------------------------------------------------- the C entry's rejections
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["n0", "n257", "t_lt_n", "null_x", "null_tables", "dtype", "tp", "lm_rows", "dest_rows",
                                  "null_q8", "paged2", "gate_up_type", "lm_head_type"])
def test_prefill_step_rejects(cuda, case):
    """Each bad field alone gives cudaErrorInvalidValue (1) before anything is launched: the caches stay untouched."""
    w = M.LlamaWeights(_cfg("q8_0", "bf16"), cuda, dtype=torch.bfloat16)
    pre = M.LlamaPrefill(w, max_tokens=64)
    prompts, tables = [[1, 2, 3], [4, 5]], _own_tables(2, 1)
    p, _, keep = pre.make_plan(prompts, [1, 0], tables, lm_rows=1)
    s = M._Step.from_buffer_copy(pre.step_struct)
    dummy = torch.zeros(64, dtype=torch.int32, device=cuda)
    if case == "n0":
        p.n_seqs = 0
    elif case == "n257":
        p.n_seqs = 257
    elif case == "t_lt_n":
        p.total_tokens = 1
    elif case == "null_x":
        p.x = None
    elif case == "null_tables":
        p.block_tables = None
    elif case == "dtype":
        s.act_dtype = 2
    elif case == "tp":
        s.tp = dummy.data_ptr()
    elif case == "lm_rows":
        p.lm_rows = 3
    elif case == "dest_rows":
        p.lm_rows, p.dest_rows = 2, dummy.data_ptr()
    elif case == "null_q8":
        p.q8_scratch = None
    elif case == "paged2":
        p.paged = 2
    elif case == "gate_up_type":      # only the last layer is wrong: the earlier layers must not run either
        layers = (M._Layer * len(pre._layers)).from_buffer_copy(pre._layers)
        layers[-1].w_up.ggml_type = GGML["q4_0"]
        s.layers = ctypes.cast(layers, ctypes.POINTER(M._Layer))
    elif case == "lm_head_type":      # no MMVQ launcher for the n <= 8 lm_head
        s.lm_head.ggml_type = GGML["q8_1"]
    torch.cuda.synchronize()
    rc = lib().mrs_llama_prefill_step(ctypes.byref(s), ctypes.byref(p), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert rc == 1, rc
    assert all(int(c.abs().sum()) == 0 for c in pre.k_cache)
