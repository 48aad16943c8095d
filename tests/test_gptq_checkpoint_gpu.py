"""GPTQ / AWQ checkpoint directories through GptqWeights.from_checkpoint on the int4 layer stack: the natural-order round
trip from a synthetic model (bit-identical), an identity act order (bit-identical), the permuted RMSNorm and the column
gather against their plain forms, decode of act-order GPTQ and AWQ checkpoints against the CPU oracle's checkpoint
product in both cache layouts and both activation dtypes, prompt prefill, speculative verify and graph replay on an
act-order checkpoint, and one Mistral-7B-shaped act-order checkpoint through every step."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import gptq as og
from oracle.gptq_model import OracleGptq
from mistralrs_b200 import gptq_model as G
from mistralrs_b200 import lib
from mistralrs_b200 import model as M
from mistralrs_b200.model import rope_tables
from test_gptq_checkpoint_host import gptq_quant, hf_config, make_checkpoint, synth_tensors, write_checkpoint

pytestmark = pytest.mark.gpu

TDT = {"f16": torch.float16, "bf16": torch.bfloat16}
# test_gptq_model_gpu.py's bound in f16; bf16 carries 8 significant bits against f16's 11, so every rounding of an
# activation weighs 2^3 times more: the same bound times 8 (test_gptq_prefill_gpu.py's bf16 bound)
LOGIT_TOL = {"f16": 3e-3, "bf16": 2.4e-2}
TIE = 1e-2          # a greedy token is checked where the top two logits differ by more than this fraction of the scale


class CheckpointOracle(OracleGptq):
    """OracleGptq over a checkpoint's linears as stored (the dict entries GptqWeights.from_checkpoint(keep_host=True)
    keeps): GPTQ W[k] = (q[k] - 8) * s[g_idx[k]], the act-order product, through og.dequant_gptq with g_idx; AWQ
    W = (q - z) * s through og.dequant_awq.  The dequantised weights go into the base class's cache, so its layer
    stack runs unchanged; never the stack's permuted tensors."""

    def __init__(self, cfg, host, rope_cos, rope_sin, dt="f16"):
        super().__init__(cfg, host, rope_cos, rope_sin, dt)
        for key, e in host.items():
            if isinstance(e, dict):
                self._deq[key] = (og.dequant_awq(e["qweight"], e["scales"], e["qzeros"], cfg.group_size) if "qzeros" in e
                                  else og.dequant_gptq(e["qweight"], e["scales"], e["g_idx"], cfg.group_size))


def _P(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _bits(t):
    return t.contiguous().view(torch.int16)


@pytest.fixture(scope="module")
def act_order_dir(tmp_path_factory):
    return make_checkpoint(str(tmp_path_factory.mktemp("gptq_act")), G.GptqConfig.tiny_test(), act_order=True, seed=21,
                           shards=2)


@pytest.fixture(scope="module")
def awq_dir(tmp_path_factory):
    return make_checkpoint(str(tmp_path_factory.mktemp("awq")), G.GptqConfig.tiny_test(), method="awq", seed=22)


def _decode(run, toks, steps):
    """greedy decode from `toks`: logits of every step (host f32)"""
    run.set_tokens(toks)
    out = []
    for _ in range(steps):
        run.step()
        torch.cuda.synchronize()
        out.append(run.logits().float().cpu().numpy())
    return out


# ---------------------------------------------------------------- bit-identical paths
@pytest.mark.parametrize("layout", ["hnd", "vllm"])
def test_round_trip_of_synthetic_model_is_bit_identical(cuda, tmp_path, layout):
    cfg = G.GptqConfig.tiny_test()
    syn = G.GptqWeights(cfg, cuda, keep_host=True)
    d = make_checkpoint(str(tmp_path / "rt"), cfg, host=syn.host)
    w = G.GptqWeights.from_checkpoint(d, cuda)
    assert w.cfg.max_pos == cfg.max_pos and not w.act_order_o
    a, b = G.GptqRunner(syn, batch=3, max_ctx=64, cache_layout=layout), G.GptqRunner(w, batch=3, max_ctx=64, cache_layout=layout)
    for x, y in zip(_decode(a, [5, 77, 300], 6), _decode(b, [5, 77, 300], 6)):
        assert np.array_equal(x, y)
    assert torch.equal(a.meta["token_ids"], b.meta["token_ids"])


def test_identity_act_order_is_bit_identical(cuda, tmp_path):
    cfg = G.GptqConfig.tiny_test()
    t = synth_tensors(cfg, seed=31)                          # g_idx = k // group
    plain = {k: v for k, v in t.items() if not k.endswith(".g_idx")}
    da = write_checkpoint(str(tmp_path / "desc"), hf_config(cfg, gptq_quant(64, desc_act=True)), t)
    db = write_checkpoint(str(tmp_path / "plain"), hf_config(cfg, gptq_quant(64)), plain)
    wa, wb = G.GptqWeights.from_checkpoint(da, cuda), G.GptqWeights.from_checkpoint(db, cuda)
    ra, rb = G.GptqRunner(wa, batch=2, max_ctx=64), G.GptqRunner(wb, batch=2, max_ctx=64)
    for x, y in zip(_decode(ra, [3, 9], 5), _decode(rb, [3, 9], 5)):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("H", [256, 4096])
def test_permuted_norm_and_gather_are_the_permuted_plain_kernels(cuda, dt, H):
    L, R, eps, code = lib(), 7, 1e-5, {"f16": 0, "bf16": 1}[dt]
    g = torch.Generator(device="cpu").manual_seed(H)
    r = lambda: torch.randn(R, H, generator=g).to(cuda).to(TDT[dt])
    x, res = r(), r()
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(cuda).to(TDT[dt])
    perm = torch.randperm(H, generator=g).to(torch.int32).to(cuda)
    e = lambda: torch.empty(R, H, dtype=TDT[dt], device=cuda)
    plain, sum_a, out_a = e(), e(), e()
    (L.mrs_rms_norm_f16 if dt == "f16" else L.mrs_rms_norm_bf16)(_P(x), _P(w), _P(plain), R, H, ctypes.c_float(eps),
                                                                 ctypes.c_int64(torch.cuda.current_stream().cuda_stream))
    L.mrs_add_rms_norm_pdl(_P(x), _P(res), _P(w), _P(sum_a), _P(out_a), R, H, ctypes.c_float(eps), code, 0, _st())
    for pdl in (0, 1):
        got, sum_b, out_b = e(), e(), e()
        assert L.mrs_rms_norm_perm_pdl(_P(x), _P(w), _P(perm), _P(got), R, H, ctypes.c_float(eps), code, pdl, _st()) == 0
        assert L.mrs_add_rms_norm_perm_pdl(_P(x), _P(res), _P(w), _P(perm), _P(sum_b), _P(out_b), R, H, ctypes.c_float(eps),
                                           code, pdl, _st()) == 0
        xa, ha, sum_c = x.clone(), x.clone(), e()            # x == norm_dst, as the prompt step normalises h in place
        assert L.mrs_rms_norm_perm_pdl(_P(xa), _P(w), _P(perm), _P(xa), R, H, ctypes.c_float(eps), code, pdl, _st()) == 0
        assert L.mrs_add_rms_norm_perm_pdl(_P(ha), _P(res), _P(w), _P(perm), _P(sum_c), _P(ha), R, H, ctypes.c_float(eps),
                                           code, pdl, _st()) == 0
        y = e()
        assert L.mrs_gather_cols_pdl(_P(x), _P(perm), _P(y), R, H, pdl, _st()) == 0
        torch.cuda.synchronize()
        p = perm.long()
        assert torch.equal(_bits(got), _bits(plain[:, p])) and torch.equal(_bits(xa), _bits(plain[:, p]))
        assert torch.equal(_bits(out_b), _bits(out_a[:, p])) and torch.equal(_bits(ha), _bits(out_a[:, p]))
        assert torch.equal(_bits(sum_b), _bits(sum_a)) and torch.equal(_bits(sum_c), _bits(sum_a))   # natural order
        assert torch.equal(_bits(y), _bits(x[:, p]))


# ---------------------------------------------------------------- against the checkpoint's product
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("layout", ["hnd", "vllm"])
@pytest.mark.parametrize("method", ["gptq_act_order", "awq"])
def test_decode_matches_oracle(cuda, act_order_dir, awq_dir, method, layout, dt):
    d = act_order_dir if method == "gptq_act_order" else awq_dir
    w = G.GptqWeights.from_checkpoint(d, cuda, dtype=TDT[dt], keep_host=True)
    assert w.quant_method == method[:4] and w.act_order_o == (method != "awq")
    run = G.GptqRunner(w, batch=3, max_ctx=64, cache_layout=layout)
    cos, sin = rope_tables(w.cfg)
    ref = CheckpointOracle(w.cfg, w.host, cos, sin, dt)
    toks, worst = [5, 77, 300], 0.0
    run.set_tokens(toks)
    for pos in range(5):
        run.step()
        torch.cuda.synchronize()
        got, want = run.logits().float().cpu().numpy(), ref.step(toks, pos)
        assert np.isfinite(got).all()
        scale = np.abs(want).max()
        err = np.abs(got - want).max() / scale
        worst = max(worst, err)
        assert err <= LOGIT_TOL[dt], (method, layout, dt, pos, err)
        nxt = run.meta["token_ids"].cpu().tolist()
        for b in range(len(toks)):
            top2 = np.sort(want[b])[-2:]
            if top2[1] - top2[0] > TIE * scale:
                assert nxt[b] == int(np.argmax(want[b])), (pos, b)
        toks = np.argmax(want, axis=1).tolist()
        run.set_tokens(toks)
    print(f"{method} checkpoint decode ({layout}, {dt}): worst logit error {worst:.2e} of the logit scale")


def test_prefill_hands_off_the_oracle_greedy_stream(cuda, act_order_dir):
    w = G.GptqWeights.from_checkpoint(act_order_dir, cuda, keep_host=True)
    run = G.GptqRunner(w, batch=3, max_ctx=64)
    pre = G.GptqPrefill(w, max_tokens=64, runner=run)
    rng = np.random.default_rng(7)
    prompts = [rng.integers(0, w.cfg.vocab, size=6).tolist() for _ in range(3)]
    cos, sin = rope_tables(w.cfg)
    ref = CheckpointOracle(w.cfg, w.host, cos, sin, "f16")
    for pos in range(6):
        want = ref.step([p[pos] for p in prompts], pos)
    _, first = pre.forward_batch(prompts, slots=[0, 1, 2])
    toks, checked = first.tolist(), 0
    assert run.context_lens.cpu().tolist() == [6, 6, 6]
    for pos in range(6, 12):
        scale = np.abs(want).max()
        for b in range(3):
            top2 = np.sort(want[b])[-2:]
            if top2[1] - top2[0] > TIE * scale:
                assert toks[b] == int(np.argmax(want[b])), (pos, b)
                checked += 1
        want = ref.step(toks, pos)               # the oracle follows the device's stream
        run.step()
        torch.cuda.synchronize()
        toks = run.meta["token_ids"].cpu().tolist()
    assert checked >= 6


def test_speculative_verify_returns_the_plain_greedy_stream(cuda, act_order_dir):
    w = G.GptqWeights.from_checkpoint(act_order_dir, cuda)
    B, k, n = 4, 3, 16
    rng = np.random.default_rng(9)
    prompts = [rng.integers(0, w.cfg.vocab, size=int(rng.integers(3, 10))).tolist() for _ in range(B)]

    def prefilled():
        run = G.GptqRunner(w, batch=B, max_ctx=128)
        _, first = G.GptqPrefill(w, max_tokens=64, runner=run).forward_batch(prompts, slots=list(range(B)))
        return run, first.tolist()
    plain, first = prefilled()
    streams, margins = [[t] for t in first], [[] for _ in range(B)]
    plain.set_tokens(first)
    for _ in range(n):
        plain.step()
        torch.cuda.synchronize()
        lg = plain.logits().float().cpu().numpy()
        for b, t in enumerate(plain.meta["token_ids"].cpu().tolist()):
            top2 = np.sort(lg[b])[-2:]
            margins[b].append((top2[1] - top2[0]) / np.abs(lg).max())
            streams[b].append(t)
    run, first2 = prefilled()
    assert first2 == first
    calls = [0]

    def propose(history):                        # right drafts, with a wrong one every few steps
        b, at = calls[0] % B, len(history) - 1
        calls[0] += 1
        d = [streams[b][at + 1 + i] if at + 1 + i <= n else 0 for i in range(k)]
        if (at + b) % 3 == 0:
            d[1] = (d[1] + 1) % w.cfg.vocab
        return d
    got, steps = M.speculative_generate(G.GptqVerifier(run, draft_len=k), first, n, propose)
    assert len(steps) < n
    for b in range(B):                           # streams[b][0] is the prefill's first token, which got[b] starts after
        for i, (x, y) in enumerate(zip(got[b], streams[b][1:])):
            if x != y:                           # only a near-tie of the plain step may part the two streams
                assert margins[b][i] <= TIE, (b, i, x, y)
                break


def test_graph_replay_matches_eager(cuda, act_order_dir):
    w = G.GptqWeights.from_checkpoint(act_order_dir, cuda)
    eager, graph = G.GptqRunner(w, batch=4, max_ctx=64), G.GptqRunner(w, batch=4, max_ctx=64)
    graph.capture()
    eager.set_tokens([1, 2, 3, 4]); graph.set_tokens([1, 2, 3, 4])
    for _ in range(8):
        eager.step(); graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.meta["token_ids"], graph.meta["token_ids"])
    assert torch.equal(eager.logits(), graph.logits())


def test_mistral_7b_shaped_act_order_runs_every_step(cuda, tmp_path):
    """Mistral-7B's dimensions (hidden 4096, 32 / 8 heads of 128, intermediate 14336, vocab 32000, g128), one layer:
    prefill, decode and verify once each.  One layer because seeded int4 weights at these sizes grow the f16 residual
    stream past its range within a few layers (the synthetic GptqWeights model does the same), and finite logits are
    what is checked here."""
    cfg = G.GptqConfig.mistral_7b(n_layers=1)
    d = make_checkpoint(str(tmp_path / "m7"), cfg, act_order=True, seed=41, shards=2, sliding_window=4096)
    w = G.GptqWeights.from_checkpoint(d, cuda)
    assert w.cfg.max_pos == 4096 and w.act_order_o
    run = G.GptqRunner(w, batch=2, max_ctx=256)
    logits, first = G.GptqPrefill(w, max_tokens=256, runner=run).forward_batch([list(range(1, 65)), list(range(7, 40))],
                                                                               slots=[0, 1])
    assert torch.isfinite(logits).all()
    run.set_tokens(first.tolist())
    run.step()
    torch.cuda.synchronize()
    assert torch.isfinite(run.logits()).all()
    nxt = run.meta["token_ids"].cpu().tolist()
    got, _ = M.speculative_generate(G.GptqVerifier(run, draft_len=2), nxt, 3, lambda h: [h[-1]] * 2)
    assert all(len(s) == 3 and all(0 <= t < cfg.vocab for t in s) for s in got)
