"""Batched prompt prefill on the headline model: Llama-3-8B Q4_K_M (synthetic seeded weights, 32 layers).
What does one `LlamaPrefill.forward_batch` over B prompts cost against B sequential `forward` calls?

Parts (--parts, comma-separated; default all):
  gemm     grouped QKV and gate|up with the GLU epilogue (one `mrs_mmq_gguf_grouped` launch each) against the separate
           GEMMs + `fused_glu`, at --gemm-rows rows (default 4096) on the config-3 (Q8_0) and config-2 (Q4_K) shapes of
           one layer, alternating in one run; median ms of CUDA-event timings
  batch    B = 1, 8, 16, 64 prompts of 128 tokens: one forward_batch against B forward calls, alternating; median ms,
           prompt tokens/s and the ratio.  16 x 128 rows take the grouped QKV / GLU launches, 64 x 128 the separate
           ones (the step's 2048-row threshold)
  ragged   the same for 32 prompts of 32..512 tokens (seeded)
  chunked  64 prompts of 512 tokens driven through the prompt chunk plan at a 4096-token budget (the reference's
           max_num_batched_tokens: 64-row chunks, one forward_batch per chunk group), against one forward_batch per 8
           whole 512-token prompts (the same 4096 rows per step)
The first line gives the GPU name, power limit and max SM clock from nvidia-smi, read in the same run.
Usage: python scripts/bench_batched_prefill.py [--parts gemm,batch,ragged,chunked] [--reps 5] [--layers 32]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in out[0].split(",")] if out else ("unknown", "unknown", "unknown")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn, reps):
    """median ms of `reps` CUDA-event timings of fn()"""
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def alternate(fns, reps):
    """{name: median ms}, the callables interleaved rep by rep so drift hits every one alike"""
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            ts[k].append(timed(fn, 1))
    return {k: float(np.median(v)) for k, v in ts.items()}


def part_gemm(M, dev, rows, reps):
    from mistralrs_b200 import mmq, ops, quant
    out = []
    for quant_name, cfg_name in (("q8_0", "config 3 (Q8_0)"), ("q4_k_m", "config 2 (Q4_K_M)")):
        cfg = M.LlamaConfig.llama3_8b(quant=quant_name, n_layers=1)
        w = M.LlamaWeights(cfg, dev, fast_synth=True)
        L = w.layers[0]
        qt = lambda e: quant.QTensor(e[0], e[1], (e[2], e[3]))
        q, k, v, g, u = (qt(L[n]) for n in ("attn_q", "attn_k", "attn_v", "ffn_gate", "ffn_up"))
        x = (torch.randn(rows, cfg.hidden, device=dev) * 0.5).to(torch.bfloat16)
        qkv_same = q.dtype == k.dtype == v.dtype
        fns = {
            "qkv_separate": lambda: (mmq.forward(q, x), mmq.forward(k, x), mmq.forward(v, x)),
            "qkv_grouped": (lambda: mmq.grouped([q, k, v], x)) if qkv_same else
                           (lambda: (mmq.grouped([q, k], x), mmq.forward(v, x))),
            "glu_separate": lambda: ops.fused_glu(mmq.forward(g, x), mmq.forward(u, x), 0),
            "glu_grouped": lambda: mmq.grouped([g, u], x, glu=True),
        }
        for fn in fns.values():      # warm-up every shape
            fn()
        torch.cuda.synchronize()
        r = alternate(fns, reps)
        r.update({"part": "gemm", "model": cfg_name, "rows": rows, "qkv_types": [q.dtype, k.dtype, v.dtype],
                  "qkv_grouped_over_separate": r["qkv_grouped"] / r["qkv_separate"],
                  "glu_grouped_over_separate": r["glu_grouped"] / r["glu_separate"]})
        out.append(r)
        del w
        torch.cuda.empty_cache()
    return out


def _tables(n, blocks):
    return [list(range(1 + blocks * i, 1 + blocks * (i + 1))) for i in range(n)]


def _compare(pre, prompts, reps, chunk_budget=None):
    """one forward_batch over `prompts` against one forward per prompt (or, with chunk_budget, the chunk plan's
    forward_batch calls against whole-prompt forward_batch calls of the same number of sequences per step),
    alternating; the same tables every time (the caches are overwritten)"""
    from mistralrs_b200 import kv_index
    bs = pre.cfg.block_size
    blocks = -(-max(len(p) for p in prompts) // bs)
    tables = _tables(len(prompts), blocks)
    tokens = sum(len(p) for p in prompts)

    def batched():
        return pre.forward_batch(prompts, tables=tables)[0]

    def sequential():
        return [pre.forward(p, table=t) for p, t in zip(prompts, tables)]

    def chunked():
        size = kv_index.prompt_chunk_size(len(prompts), chunk_budget)
        plans = [kv_index.build_prompt_chunk_plan(len(p), 0, size, bs) for p in prompts]
        idx = [0] * len(prompts)
        while (g := kv_index.next_prompt_chunk_group(idx, plans)) is not None:
            members, final = g
            ch = [plans[i][idx[i]] for i in members]
            pre.forward_batch([prompts[i][s:e] for i, (s, e) in zip(members, ch)], cached=[s for s, _ in ch],
                              tables=[tables[i] for i in members], final=final)
            for i in members:
                idx[i] += 1

    def whole_steps():    # the same sequences, whole prompts, as many per step as the budget holds
        per = max(1, chunk_budget // max(len(p) for p in prompts))
        for i in range(0, len(prompts), per):
            pre.forward_batch(prompts[i:i + per], tables=tables[i:i + per])

    fns = {"chunk_plan": chunked, "whole_prompt_steps": whole_steps} if chunk_budget else \
          {"forward_batch": batched, "sequential_forward": sequential}
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    r = alternate(fns, reps)
    a, b = list(fns)
    r.update({"prompts": len(prompts), "tokens": tokens, f"{a}_tok_s": tokens / r[a] * 1e3,
              f"{b}_tok_s": tokens / r[b] * 1e3, f"{b}_over_{a}": r[b] / r[a]})
    return r


def part_prefill(M, dev, parts, reps, layers):
    cfg = M.LlamaConfig.llama3_8b(n_layers=layers)
    w = M.LlamaWeights(cfg, dev, fast_synth=True)
    pre = M.LlamaPrefill(w, max_tokens=64 * 512)      # its own cache holds the 64 x 512-token chunked workload
    vocab = cfg.vocab
    rng = np.random.default_rng(0xB200)
    ids = lambda n: rng.integers(0, vocab, size=n).tolist()
    if "batch" in parts:
        for B in (1, 8, 16, 64):
            r = _compare(pre, [ids(128) for _ in range(B)], reps)
            r.update({"part": "batch", "workload": f"{B} prompts x 128 tokens, Llama-3-8B Q4_K_M, {layers} layers"})
            print(json.dumps(r), flush=True)
    if "ragged" in parts:
        lens = rng.integers(32, 513, size=32).tolist()
        r = _compare(pre, [ids(n) for n in lens], reps)
        r.update({"part": "ragged", "workload": f"32 prompts of 32..512 tokens ({sum(lens)} in all), {layers} layers"})
        print(json.dumps(r), flush=True)
    if "chunked" in parts:
        r = _compare(pre, [ids(512) for _ in range(64)], max(2, reps // 2), chunk_budget=4096)
        r.update({"part": "chunked", "workload": f"64 prompts x 512 tokens, chunk plan at a 4096-token budget "
                                                  f"(64-row chunks), against 8 whole prompts per step, {layers} layers"})
        print(json.dumps(r), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="gemm,batch,ragged,chunked")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--gemm-rows", default="4096", help="comma-separated row counts")
    ap.add_argument("--layers", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batched_prefill: needs a GPU")
    graft.load_package()
    from mistralrs_b200 import model as M
    dev = torch.device("cuda:0")
    print(json.dumps(gpu_info()), flush=True)
    parts = args.parts.split(",")
    if "gemm" in parts:
        for rows in (int(r) for r in args.gemm_rows.split(",")):
            for r in part_gemm(M, dev, rows, max(args.reps, 10)):
                print(json.dumps(r), flush=True)
    if {"batch", "ragged", "chunked"} & set(parts):
        part_prefill(M, dev, parts, args.reps, args.layers)


if __name__ == "__main__":
    main()
