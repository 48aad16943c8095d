"""GGUF decode for 9..256 sequences: the layer chain on the wgmma dequant GEMM (mrs_mmq_gguf_grouped: grouped
q|k|v and the gate|up GLU epilogue).  Above 8 rows the step has the prefill GEMM's numerics, so the oracle is
OracleLlama(exact_gemm=True).  The argument checks at the end run without a GPU."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from mistralrs_b200 import GGML, lib, mmq, ops, quant
from mistralrs_b200 import model as M
from oracle.model import OracleLlama
from util import make_acts, make_weight, to_dev

TDT = {"bf16": torch.bfloat16, "f16": torch.float16}
ULP = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11}
LOGIT_TOL = 2e-2     # test_prefill_composition_matches_oracle: the prefill GEMM chain vs the exact-GEMM oracle
# The synthetic Q8_0 model amplifies small perturbations: its exact-GEMM and Q8_1 oracles differ by 4-6 % of the logit
# scale over a few steps.  Against the rounded-weight oracle below, f32-vs-f64 accumulation alone reaches ~2.4 % over
# the longer ragged trajectories, so that model gets the wider bound (still below its own oracles' spread).
Q8_0_LOGIT_TOL = 3e-2


def _gemm_tol(dtype, wb, x, ref, n, k, dt):
    # the bound test_mmq_gpu.py uses for mrs_mmq_gguf: output rounding + operand rounding of the weights
    mag = np.abs(oracle.dequantize(dtype, wb).reshape(n, k)).astype(np.float64) @ np.abs(x).astype(np.float64).T
    return ULP[dt] * np.abs(ref) * 1.01 + ULP[dt] * mag.T + 1e-6


# ---------------------------------------------------------------- the grouped GEMM op
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["q4_k", "q6_k", "q8_0", "q5_0"])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("M_", [9, 32, 33, 64, 200])
def test_grouped_gemm_and_glu(cuda, dtype, dt, M_):
    K = 512
    widths = (200, 72, 136)        # tiles straddle matrices at rows 200 and 272
    wbs = [make_weight(dtype, n, K, 10 + i) for i, n in enumerate(widths)]
    ws = [quant.QTensor(to_dev(wb.reshape(-1), cuda), dtype, (n, K)) for wb, n in zip(wbs, widths)]
    x = make_acts(M_, K, 3, dt)
    xd = to_dev(x, cuda, dt)
    outs = mmq.grouped(ws, xd)
    refs = [oracle.matmul_exact(dtype, wb, x, K, n) for wb, n in zip(wbs, widths)]
    for y, ref, wb, n in zip(outs, refs, wbs, widths):
        err = np.abs(y.float().cpu().numpy() - ref)
        tol = _gemm_tol(dtype, wb, x, ref, n, K, dt)
        assert (err <= tol).all(), (n, float((err / tol).max()))
    again = mmq.grouped(ws, xd)
    assert all(torch.equal(a, b) for a, b in zip(outs, again))
    two = mmq.grouped(ws[:2], xd)                     # q|k only, and a single matrix
    assert torch.equal(two[0], outs[0]) and torch.equal(two[1], outs[1])

    # GLU: gate | up of width 200 (tile 3 holds gate rows 192..199 and up rows 192..199 only)
    gate, up = ws[0], quant.QTensor(to_dev(make_weight(dtype, 200, K, 20).reshape(-1), cuda), dtype, (200, K))
    act = mmq.grouped([gate, up], xd, glu=True)
    g_, u_ = mmq.grouped([gate, up], xd)
    assert torch.equal(act, ops.fused_glu(g_, u_, 0)), "epilogue differs from fused_glu over the same GEMM"
    assert torch.equal(act, mmq.grouped([gate, up], xd, glu=True))
    ub = make_weight(dtype, 200, K, 20)
    gr, ur = refs[0], oracle.matmul_exact(dtype, ub, x, K, 200)
    want = oracle.fused_glu(oracle.round_dtype(gr.astype(np.float32), dt), oracle.round_dtype(ur.astype(np.float32), dt), 0, dt)
    tg, tu = _gemm_tol(dtype, wbs[0], x, gr, 200, K, dt), _gemm_tol(dtype, ub, x, ur, 200, K, dt)
    # |d silu| <= 1.1: gate error through the activation, up error times the activation, two roundings in T
    tol = 1.1 * tg * np.abs(ur) + tu * (np.abs(want / np.where(ur == 0, 1, ur)) + 1) + 3 * ULP[dt] * np.abs(want) + 1e-6
    got = act.float().cpu().numpy()
    fin = np.isfinite(want)          # f16: the product of two large synthetic outputs can overflow, on both sides
    assert np.array_equal(got[~fin], want[~fin])
    err = np.abs(got[fin] - want[fin])
    assert (err <= tol[fin]).all(), float((err / tol[fin]).max())


@pytest.mark.gpu
def test_grouped_gemm_rejects(cuda):
    w = quant.QTensor(to_dev(make_weight("q4_k", 64, 256, 1).reshape(-1), cuda), "q4_k", (64, 256))
    x = torch.zeros(16, 256, dtype=torch.bfloat16, device=cuda)
    L = lib()
    call = lambda n, rows, glu=0, K=256, xp=x.data_ptr(): L.mrs_mmq_gguf_grouped(
        GGML["q4_k"], n, (ctypes.c_void_p * 3)(w.data.data_ptr(), w.data.data_ptr(), w.data.data_ptr()), (ctypes.c_int32 * 3)(*rows),
        (ctypes.c_void_p * 3)(x.data_ptr(), x.data_ptr(), x.data_ptr()), ctypes.c_void_p(xp), 16, K, 1, glu, 0, None)
    assert call(4, (64, 64, 64)) == 1 and call(0, (64, 64, 64)) == 1
    assert call(2, (64, 32, 0), glu=1) == 1 and call(3, (64, 64, 64), glu=1) == 1
    assert call(1, (64, 0, 0), K=128) == 1                    # k-quants need K % 256
    assert call(2, (64, 0, 0)) == 1                           # a matrix with no rows
    assert call(1, (64, 0, 0), xp=x.data_ptr() + 2) == 716    # cudaErrorMisalignedAddress


# ---------------------------------------------------------------- the decode chain
def _cfg(quant_, dt, **kw):
    if (quant_, dt) == ("q4_k_m", "f16"):        # the default synthetic block scales overflow f16 in this model
        kw["synth_scale_exp"] = (-15, -13)
    return M.LlamaConfig.tiny_test(quant=quant_, n_layers=2, **kw)


class RoundedWeightOracle(OracleLlama):
    """OracleLlama(exact_gemm=True) whose linears take the weights rounded once to the activation format, as the
    dequant GEMM's MMA operands are: the exact f64 product of those weights with the activations.  The synthetic Q8_0
    model amplifies per-weight perturbations of that size past the logit bound (its own exact-GEMM and Q8_1 oracles
    differ by 4-6 % of the logit scale), so it is compared against the GEMM's operands rather than the raw blocks."""

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


def _prefill_ragged(w, run, B, seed):
    """prompts of different lengths; all but the last token of each are prefilled into the sequence's own table (the
    last one is the first decode input).  Returns the prompts."""
    cfg = w.cfg
    rng = np.random.default_rng(seed)
    lens = [int(3 + (7 * b + seed) % 11) for b in range(B)]
    prompts = [rng.integers(0, cfg.vocab, size=n).tolist() for n in lens]
    pre = M.LlamaPrefill(w, max_tokens=run.max_ctx, runner=run)
    for b in range(B):
        pre.forward(prompts[b][:-1], table=run.tables[b])
    run.reset([n - 1 for n in lens])
    return prompts


def _oracles(w, prompts, dt):
    refs = []
    for p in prompts:
        r = _oracle(w, dt)
        for pos, t in enumerate(p[:-1]):
            r.step([t], pos)
        refs.append(r)
    return refs


@pytest.mark.gpu
@pytest.mark.parametrize("quant_", ["q4_k_m", "q8_0"])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("B", [9, 16, 33, 64])
def test_ragged_batch_matches_oracle(cuda, quant_, dt, B):
    """Sequences at different positions (their own prompts, prefilled into their own tables), then decode steps of the
    whole batch: each sequence's logits against its own exact-GEMM oracle stepped through the same tokens.  q4_k_m
    takes the q|k + v launches (attn_v in Q6_K), q8_0 one grouped QKV launch."""
    cfg = _cfg(quant_, dt)
    w = M.LlamaWeights(cfg, cuda, dtype=TDT[dt], keep_host=True)
    run = M.LlamaRunner(w, batch=B, max_ctx=64, pdl=True)
    prompts = _prefill_ragged(w, run, B, seed=B)
    refs = _oracles(w, prompts, dt)
    toks = [p[-1] for p in prompts]
    pos = [len(p) - 1 for p in prompts]
    run.set_tokens(toks)
    tol = Q8_0_LOGIT_TOL if quant_ == "q8_0" else LOGIT_TOL
    worst = 0.0
    for step in range(4):
        run.step()
        torch.cuda.synchronize()
        got = run.logits().float().cpu().numpy()
        ids = run.meta["token_ids"].cpu().tolist()
        assert np.isfinite(got).all()
        for b in range(B):
            want = refs[b].step([toks[b]], pos[b])[0]
            scale = np.abs(want).max()
            err = np.abs(got[b] - want).max() / scale
            worst = max(worst, err)
            assert err <= tol, (step, b, err)
            if ids[b] != int(np.argmax(want)):
                assert _near_tie(want, err * scale, dt), (step, b, ids[b], int(np.argmax(want)))
        toks = ids
        pos = [p + 1 for p in pos]
    assert int(run.error_flag.item()) == 0
    print(f"B={B} {quant_} {dt}: worst logit error {worst:.3e} of the scale")


@pytest.mark.gpu
@pytest.mark.parametrize("B", [16, 64])
def test_llama3_8b_shapes_batched(cuda, B):
    """Config-2 shapes (two real-size Q4_K_M layers: layer 1 keeps attn_v / ffn_down in Q6_K; Q6_K lm_head) through the
    GEMM route, against the exact-GEMM oracle."""
    cfg = M.LlamaConfig.llama3_8b(n_layers=2, max_pos=64)
    w = M.LlamaWeights(cfg, cuda, dtype=torch.bfloat16, keep_host=True)
    run = M.LlamaRunner(w, batch=B, max_ctx=32, pdl=True)
    cos, sin = M.rope_tables(cfg)
    ref = OracleLlama(cfg, w.host, M.tensor_type, cos, sin, "bf16", exact_gemm=True)
    toks = [(1000 + 977 * b) % cfg.vocab for b in range(B)]
    run.set_tokens(toks)
    for pos in range(2):
        run.step()
        torch.cuda.synchronize()
        got = run.logits().float().cpu().numpy()
        want = ref.step(toks, pos)
        assert np.isfinite(got).all() and np.isfinite(want).all()
        scale = np.abs(want).max()
        assert scale > 1e-3 and np.unique(want).size > 1000, "degenerate logits"
        err = np.abs(got - want).max() / scale
        assert err <= LOGIT_TOL, (pos, err)
        ids = run.meta["token_ids"].cpu().tolist()
        for b in range(B):
            if ids[b] != int(np.argmax(want[b])):
                assert _near_tie(want[b], np.abs(got[b] - want[b]).max(), "bf16"), (pos, b)
        toks = ids


@pytest.mark.gpu
def test_graph_and_pdl_bit_identical(cuda):
    cfg = _cfg("q4_k_m", "bf16")
    w = M.LlamaWeights(cfg, cuda)
    B = 32
    toks = [(37 * b + 5) % cfg.vocab for b in range(B)]

    def eager(pdl):
        r = M.LlamaRunner(w, batch=B, max_ctx=64, pdl=pdl)
        r.set_tokens(toks)
        out = []
        for _ in range(4):
            r.step()
            out.append(r.logits().clone())
        return out, r

    plain, _ = eager(False)
    chained, r = eager(True)
    assert all(torch.equal(a, b) for a, b in zip(plain, chained))
    r.capture()
    r.set_tokens(toks)
    for want in chained:
        r.replay()
        torch.cuda.synchronize()
        assert torch.equal(r.logits(), want)


@pytest.mark.gpu
def test_fused_and_unfused_attention(cuda):
    cfg = _cfg("q4_k_m", "bf16")
    w = M.LlamaWeights(cfg, cuda)
    B = 16
    a = M.LlamaRunner(w, batch=B, max_ctx=512, fused_attention=True)
    b = M.LlamaRunner(w, batch=B, max_ctx=512, fused_attention=False)
    assert a.padded_tiles > B, "expected a split-KV plan"
    gen = torch.Generator(device=cuda).manual_seed(3)
    for l in range(cfg.n_layers):     # the same history in both caches
        for ca, cb in ((a.k_cache[l], b.k_cache[l]), (a.v_cache[l], b.v_cache[l])):
            ca.copy_(torch.randn(ca.shape, generator=gen, device=cuda).to(ca.dtype))
            cb.copy_(ca)
    lens = [100 + 23 * i for i in range(B)]
    a.reset(lens); b.reset(lens)
    toks = [(11 * i + 3) % cfg.vocab for i in range(B)]
    a.set_tokens(toks); b.set_tokens(toks)
    for _ in range(4):
        a.step(); b.step()
        torch.cuda.synchronize()
        la, lb = a.logits().float(), b.logits().float()
        assert (la - lb).abs().max().item() <= 2.0 ** -7 * lb.abs().max().item()
        b.set_tokens(a.meta["token_ids"].cpu().tolist())
    for l in range(cfg.n_layers):
        assert torch.equal(a.k_cache[l], b.k_cache[l]) and torch.equal(a.v_cache[l], b.v_cache[l])
    assert int(a.buf["attn_counters"].abs().sum()) == 0


@pytest.mark.gpu
def test_context_overflow_freezes_one_sequence(cuda):
    cfg = _cfg("q8_0", "bf16")
    w = M.LlamaWeights(cfg, cuda, keep_host=True)
    B = 12
    run = M.LlamaRunner(w, batch=B, max_ctx=64)
    prompts = _prefill_ragged(w, run, B, seed=5)
    refs = _oracles(w, prompts, "bf16")
    lens = [len(p) - 1 for p in prompts]
    lens[4] = run.max_ctx                                  # sequence 4 sits at its table's end
    run.reset(lens[:4] + [0] + lens[5:])
    run.context_lens[4] = run.max_ctx                      # (past the host-side bound, which step() would enforce)
    blocks = torch.tensor(run.tables[4], device=cuda)
    before = [(k[blocks].clone(), v[blocks].clone()) for k, v in zip(run.k_cache, run.v_cache)]
    toks = [p[-1] for p in prompts]
    run.set_tokens(toks)
    run.step()
    torch.cuda.synchronize()
    assert int(run.meta["slot_mapping"][4]) == -1 and int(run.error_flag.item()) & 1
    assert int(run.context_lens[4]) == run.max_ctx
    for (k0, v0), k, v in zip(before, run.k_cache, run.v_cache):
        assert torch.equal(k[blocks], k0) and torch.equal(v[blocks], v0)
    got = run.logits().float().cpu().numpy()
    for b in range(B):
        if b == 4:
            continue
        want = refs[b].step([toks[b]], len(prompts[b]) - 1)[0]
        assert int(run.context_lens[b]) == len(prompts[b])
        assert np.abs(got[b] - want).max() / np.abs(want).max() <= Q8_0_LOGIT_TOL, b


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 16])
def test_decode_step_rejects_mismatched_gate_up(cuda, B):
    """A last layer whose w_up has another ggml type than its w_gate gives cudaErrorInvalidValue before any launch, on
    the GEMV route (B = 1) and the GEMM route (B = 16): no cache row and no logit is written."""
    w = M.LlamaWeights(M.LlamaConfig.tiny_test(quant="q8_0", n_layers=2), cuda, dtype=torch.bfloat16)
    run = M.LlamaRunner(w, batch=B, max_ctx=64)
    run.set_tokens(list(range(1, B + 1)))
    run.advance()
    layers = (M._Layer * len(run._layers)).from_buffer_copy(run._layers)
    layers[-1].w_up.ggml_type = GGML["q4_0"]
    s = M._Step.from_buffer_copy(run.step_struct)
    s.layers = ctypes.cast(layers, ctypes.POINTER(M._Layer))
    torch.cuda.synchronize()
    rc = lib().mrs_llama_decode_step(ctypes.byref(s), run._stream())
    torch.cuda.synchronize()
    assert rc == 1, rc
    assert all(int(c.abs().sum()) == 0 for c in run.k_cache + run.v_cache)
    assert int(run.logits().abs().sum()) == 0


# ---------------------------------------------------------------- argument checks (no GPU)
def test_decode_step_rejects_bad_batch():
    L = lib()
    s = M._Step()
    for batch in (0, 257):
        s.batch = batch
        assert L.mrs_llama_decode_step(ctypes.byref(s), None) == 1
    s.batch = 9
    ctx = M._TpCtx()
    s.tp = ctypes.addressof(ctx)
    assert L.mrs_llama_decode_step(ctypes.byref(s), None) == 1
    s.tp = None
    s.all_reduce = M._AR_FN(lambda *a: None)
    assert L.mrs_llama_decode_step(ctypes.byref(s), None) == 1


def test_runner_rejects_bad_batch():
    for batch in (0, 257, -1, 2.0, True):
        with pytest.raises(ValueError, match="batch must be"):
            M.LlamaRunner(None, batch=batch)
    with pytest.raises(ValueError, match="tensor parallelism"):
        M.LlamaRunner(None, batch=9, comm=lambda *a: None)
    with pytest.raises(ValueError, match="tensor parallelism"):
        M.LlamaRunner(None, batch=256, peer_allreduce=object())
    M.check_runner_args(8, comm=lambda *a: None)
    M.check_runner_args(256)
