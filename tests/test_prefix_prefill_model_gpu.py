"""LlamaPrefill.forward(cached=n): prompts continued over K/V already in the paged cache — chunked prefill, a
prefix-cache hit admitted through KVCacheManager, and decode after a chunked prefill — against the CPU oracle."""
import numpy as np
import pytest
import torch

from oracle.model import OracleLlama
from mistralrs_b200 import model as M
from mistralrs_b200.kv_index import KVCacheManager, compute_block_hashes

pytestmark = pytest.mark.gpu


def _model(cuda):
    cfg = M.LlamaConfig.tiny_test(quant="q4_k_m", n_layers=2)
    w = M.LlamaWeights(cfg, cuda, keep_host=True)        # bf16 (f16 overflows on the synthetic 2-layer model)
    cos, sin = M.rope_tables(cfg)
    return cfg, w, cos, sin


def _prompt(cfg, n, seed=7):
    return [(131 * i + seed) % cfg.vocab for i in range(n)]


def test_chunked_prefill_matches_oracle(cuda):
    cfg, w, cos, sin = _model(cuda)
    pre = M.LlamaPrefill(w, max_tokens=64)
    toks = _prompt(cfg, 37)
    got, done = [], 0
    for n in (20, 1, 16):
        got.append(pre.forward(toks[done:done + n], all_logits=True, cached=done).float().cpu().numpy())
        done += n
    got = np.concatenate(got)
    ref = OracleLlama(cfg, w.host, M.tensor_type, cos, sin, "bf16", exact_gemm=True)
    want = np.stack([ref.step([t], pos)[0] for pos, t in enumerate(toks)])
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err <= 2e-2, err            # the bound of test_prefill_composition_matches_oracle


def test_prefix_cache_hit_end_to_end(cuda):
    cfg, w, cos, sin = _model(cuda)
    bs = cfg.block_size
    nblocks = 16
    mgr = KVCacheManager(nblocks, bs, True)
    pre = M.LlamaPrefill(w, max_tokens=(nblocks - 1) * bs)      # its cache has nblocks blocks; block 0 is the null block
    a = _prompt(cfg, 2 * bs + 5, seed=3)
    b = a[:2 * bs] + _prompt(cfg, 9, seed=11)                   # shares A's two full blocks
    assert mgr.allocate_slots(1, len(a)) is not None
    pre.forward(a, table=mgr.get_block_ids(1))
    mgr.cache_blocks(1, compute_block_hashes(a, bs), len(a))
    a_blocks = mgr.get_block_ids(1)
    torch.cuda.synchronize()
    a_rows = [(kc[a_blocks].clone(), vc[a_blocks].clone()) for kc, vc in zip(pre.k_cache, pre.v_cache)]

    hit = mgr.get_computed_blocks(compute_block_hashes(b, bs), len(b))
    assert hit.num_computed_tokens == 2 * bs and hit.block_ids == a_blocks[:2]
    assert mgr.allocate_slots(2, len(b), hit.block_ids) is not None
    b_blocks = mgr.get_block_ids(2)
    assert b_blocks[:2] == a_blocks[:2] and not set(b_blocks[2:]) & set(a_blocks)
    got = pre.forward(b[2 * bs:], cached=hit.num_computed_tokens, table=b_blocks).float().cpu().numpy()
    torch.cuda.synchronize()
    for (kc, vc), (ka, va) in zip(zip(pre.k_cache, pre.v_cache), a_rows):   # B wrote only its own blocks
        assert torch.equal(kc[a_blocks], ka) and torch.equal(vc[a_blocks], va)

    fresh = M.LlamaPrefill(w, max_tokens=64).forward(b).float().cpu().numpy()
    scale = np.abs(fresh).max()
    assert np.abs(got - fresh).max() / scale <= 2e-2
    ref = OracleLlama(cfg, w.host, M.tensor_type, cos, sin, "bf16", exact_gemm=True)
    want = [ref.step([t], pos)[0] for pos, t in enumerate(b)][-1]
    # the bound test_prefill_composition_matches_oracle puts on the last row (its lm_head is the decode GEMV)
    assert np.abs(got - want).max() / np.abs(want).max() <= 3e-2


def test_decode_after_chunked_prefill(cuda):
    cfg, w, cos, sin = _model(cuda)
    run = M.LlamaRunner(w, batch=1, max_ctx=64)
    pre = M.LlamaPrefill(w, max_tokens=64, runner=run)
    toks = _prompt(cfg, 29, seed=5)
    pre.forward(toks[:13])
    pre.forward(toks[13:], cached=13)
    ref = OracleLlama(cfg, w.host, M.tensor_type, cos, sin, "bf16", exact_gemm=True)   # the prompt: exact linears
    want = [ref.step([t], pos) for pos, t in enumerate(toks)][-1]
    ref.exact_gemm = False                                       # decode steps: Q8_1 GEMVs, as on the GPU
    run.reset(len(toks))
    nxt = [int(np.argmax(want[0]))]
    for i in range(4):
        run.set_tokens(nxt)
        run.step()
        torch.cuda.synchronize()
        got = run.logits().float().cpu().numpy()
        want = ref.step(nxt, len(toks) + i)
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 4.1 * 2.0 ** -7, (i, err)                 # the bound of test_model_gpu
        nxt = [int(np.argmax(want[0]))]
