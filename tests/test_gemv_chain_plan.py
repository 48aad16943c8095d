"""scripts/bench_gemv_chain.py attributes the batch-1 GEMV chain launch by launch: its plan of one token's launches must
be the decoder's (129 on Llama-3-8B Q4_K_M: q∥k∥v fused where attn_v shares q's type, q∥k and a Q6_K v as one grid)
and its bytes the ones bench.py's roofline divides by, in either form of the q∥k + v launch."""
import importlib.util
import os

from mistralrs_b200 import model as M

import bench

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script():
    spec = importlib.util.spec_from_file_location("bench_gemv_chain", os.path.join(ROOT, "scripts", "bench_gemv_chain.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_plan_matches_decoder_and_bench_bytes():
    cfg = M.LlamaConfig.llama3_8b()
    script = _script()
    plan, split = script.chain_plan(cfg, M), script.chain_plan(cfg, M, one_grid_v=False)
    roles, split_roles = [p[0] for p in plan], [p[0] for p in split]
    assert len(plan) == 129 and len(split) == 145
    assert roles.count("qk_v") == roles.count("qkv") == 16
    assert split_roles.count("qk") == split_roles.count("v") == 16 and split_roles.count("qkv") == 16
    assert roles.count("o_proj") == roles.count("gate_up") == roles.count("down") == 32 and roles[-1] == "lm_head"
    for r, t, K, vrows, _, l in split:
        if r == "v":
            assert t == M.tensor_type(cfg, "attn_v", l) == "q6_k" and (K, vrows) == (4096, 1024)
        if r == "down":
            assert (K, vrows) == (cfg.inter, cfg.hidden)
    _, weight_bytes = bench.algorithmic_bytes_per_token(cfg, M)
    assert sum(p[4] for p in plan) == sum(p[4] for p in split) == weight_bytes == 4_616_331_264


def test_attribute_phases_from_stamps():
    """two launches, two CTAs each, stamps in ns: the phases are the CTA medians, span runs from exit to exit"""
    import numpy as np
    script = _script()
    plan = [("o_proj", "q4_k", 4096, 4096, 1000, 0), ("down", "q4_k", 14336, 4096, 3000, 0)]
    tok = np.zeros((2, 320, 16), dtype=np.int64)
    #                entry init issue1 waited pass0 pass1 pass2 full0 loopend exit
    tok[0, 0, :10] = [0, 0, 0, 1000, 0, 0, 2000, 2000, 5000, 6000]
    tok[0, 1, :10] = [0, 0, 0, 1000, 0, 0, 2000, 2000, 5000, 7000]
    tok[1, 0, :10] = [6500, 0, 0, 8000, 0, 0, 9000, 9500, 12000, 13000]
    tok[1, 1, :10] = [6500, 0, 0, 8000, 0, 0, 9000, 9500, 12000, 12500]
    tok[:, 0, 15] = 2
    tok[0, 0, 14], tok[1, 0, 14] = (4096 << 32) | 4096, (4096 << 32) | 14336
    rates = {"o_proj/q4_k": {"gbs": 1.0}, "down/q4_k": {"gbs": 2.0}}
    per, roles, total = script.attribute(plan, [tok], rates)
    d = per[1]
    assert (d["gap"], d["span"], d["entry_wait"], d["prologue"], d["first_seg"], d["consume"], d["tail"]) == \
        (-0.5, 6.0, 1.5, 1.0, 0.5, 2.5, 1.0)
    assert d["ideal"] == 1.5 and per[0]["ideal"] == 1.0 and np.isnan(per[0]["span"])
    assert roles["down"]["launches"] == 1 and total["span"] == 6.0 and total["ideal"] == 2.5
