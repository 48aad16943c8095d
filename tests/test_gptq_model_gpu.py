"""GPTQ int4 decode stack (mrs_gptq_decode_step: fused QKV / gate||up W4A16 GEMMs on the swap-AB
wgmma kernel, fused RoPE + KV write + paged attention, dense lm_head) vs the CPU oracle stack, in
both KV-cache layouts of BASELINE config 4 (HND / FlashInfer and vLLM)."""
import numpy as np
import pytest
import torch

from oracle.gptq_model import OracleGptq
from mistralrs_b200 import gptq_model as G
from mistralrs_b200.model import rope_tables

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("layout", ["hnd", "vllm"])
def test_gptq_decode_matches_oracle(cuda, layout):
    cfg = G.GptqConfig.tiny_test()
    w = G.GptqWeights(cfg, cuda, keep_host=True)
    run = G.GptqRunner(w, batch=3, max_ctx=64, cache_layout=layout)
    cos, sin = rope_tables(cfg)
    ref = OracleGptq(cfg, w.host, cos, sin, "f16")
    toks = [5, 77, 300]
    run.set_tokens(toks)
    worst = 0.0
    for pos in range(5):
        run.step()
        torch.cuda.synchronize()
        got = run.logits().float().cpu().numpy()
        want = ref.step(toks, pos)
        assert np.isfinite(got).all() and np.isfinite(want).all()
        scale = np.abs(want).max()
        err = np.abs(got - want).max() / scale
        worst = max(worst, err)
        assert err <= 3e-3, (layout, pos, err)    # f16 tensors on both sides; f32 (tensor core) vs f64 accumulation
        nxt = run.meta["token_ids"].cpu().tolist()
        for b in range(len(toks)):
            top2 = np.sort(want[b])[-2:]
            if top2[1] - top2[0] > 1e-2 * scale:
                assert nxt[b] == int(np.argmax(want[b])), (pos, b)
        toks = np.argmax(want, axis=1).tolist()
        run.set_tokens(toks)
    print(f"gptq decode stack ({layout}): worst logit error {worst:.2e} of the logit scale")


@pytest.mark.parametrize("layout", ["hnd", "vllm"])
def test_gptq_context_guard_and_per_sequence_reset(cuda, layout):
    w = G.GptqWeights(G.GptqConfig.tiny_test(), cuda)
    run = G.GptqRunner(w, batch=2, max_ctx=32, cache_layout=layout)
    assert run.max_ctx == 32
    with pytest.raises(ValueError):
        run.reset([1, 2, 3])
    run.set_tokens([1, 2])
    run.reset([30, 31])                      # sequences at different positions; the bound follows the longer one
    assert run.steps_taken == 31
    run.step()                               # the longer sequence writes the last row of its table
    torch.cuda.synchronize()
    assert run.meta["positions"].tolist() == [30, 31]
    assert run.context_lens.tolist() == [31, 32]
    run.check_overflow()
    with pytest.raises(RuntimeError, match="context exhausted"):
        run.step()                           # raised on the host, before anything is enqueued
    assert run.context_lens.tolist() == [31, 32]


def test_gptq_graph_replay_matches_eager(cuda):
    cfg = G.GptqConfig.tiny_test()
    w = G.GptqWeights(cfg, cuda)
    eager, graph = G.GptqRunner(w, batch=4, max_ctx=64), G.GptqRunner(w, batch=4, max_ctx=64)
    graph.capture()
    eager.set_tokens([1, 2, 3, 4]); graph.set_tokens([1, 2, 3, 4])
    for _ in range(8):
        eager.step(); graph.graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.meta["token_ids"], graph.meta["token_ids"])
    assert torch.equal(eager.logits(), graph.logits())
