"""GPTQ prompt prefill on BASELINE config 4's model: Mistral-7B GPTQ int4 g128 (synthetic seeded weights, 32 layers).
What does one `GptqPrefill.forward_batch` cost against feeding the prompts through the decode graph one token a step?

Parts (--parts, comma-separated; default all):
  gemm     one layer's whole-K W4A16 GEMMs at --gemm-rows rows (default 512,2048,4096): q||k||v, o, down, and gate||up
           with the GLU epilogue (`pdl` bit 2) against the gate||up GEMM + fused_split_glu, alternating; median ms of
           CUDA-event timings and TFLOP/s, also as a share of the H100 SXM data-sheet dense FP16 figure (989 TFLOP/s)
  config4  32 prompts of 128 tokens into a captured batch-32 GptqRunner: one forward_batch(slots=...) against 128
           decode-graph replays (set_tokens + replay per prompt position, as bench.py's config 4 does), alternating;
           median ms, prompt tokens/s, the ratio; then both continue 16 decode tokens, which must agree except where the
           runner's logits have a near-tie
  ttft     one 4096-token prompt through GptqPrefill.forward: median ms and TFLOP/s (linears + causal attention)
The first line gives the GPU name, power limit and max SM clock from nvidia-smi, read in the same run.
Usage: python scripts/bench_gptq_prefill.py [--parts gemm,config4,ttft] [--reps 5] [--layers 32]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402

DENSE_FP16_PEAK = 989.0   # TFLOP/s, H100 SXM data sheet (dense), a card allowed 700 W


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


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def part_gemm(G, dev, rows_list, reps):
    from mistralrs_b200 import lib
    cfg = G.GptqConfig.mistral_7b(n_layers=1)
    w = G.GptqWeights(cfg, dev)
    L = w.layers[0]
    H, I = cfg.hidden, cfg.inter
    out = []
    for rows in rows_list:
        x = (torch.randn(rows, I, device=dev) * 0.5).to(torch.float16)     # wide enough for every GEMM's K
        y = torch.empty(rows, 2 * I, dtype=torch.float16, device=dev)
        act = torch.empty(rows, I, dtype=torch.float16, device=dev)

        def gemm(name, flags, dst, n_launch=5):
            tiles, scales, K, N = L[name]
            xk = x[:, :K].contiguous() if K != I else x
            def fn():
                for _ in range(n_launch):
                    rc = lib().mrs_w4a16_gemm_pdl(ctypes.c_void_p(xk.data_ptr()), ctypes.c_void_p(tiles.data_ptr()),
                                                  ctypes.c_void_p(scales.data_ptr()), None, ctypes.c_void_p(dst.data_ptr()),
                                                  rows, K, N, cfg.group_size, 0, 0, 2 | flags, _stream())
                    assert rc == 0, rc
            return fn, 2.0 * rows * K * N * n_launch

        def split_form(n_launch=5):
            plain, flop = gemm("w_gate_up", 0, y, 1)
            def fn():
                for _ in range(n_launch):
                    plain()
                    lib().mrs_split_glu_pdl(ctypes.c_void_p(y.data_ptr()), ctypes.c_void_p(act.data_ptr()), ctypes.c_uint32(rows),
                                            ctypes.c_uint32(I), 0, 0, 0, _stream())
            return fn, flop * n_launch

        fns = {"qkv": gemm("wqkv", 0, y), "o": gemm("wo", 0, y), "down": gemm("w_down", 0, y),
               "gate_up_glu_epilogue": gemm("w_gate_up", 4, act), "gate_up_then_split_glu": split_form()}
        for fn, _ in fns.values():
            fn()
        torch.cuda.synchronize()
        # bit-identity of the two gate||up forms at this size
        fns["gate_up_glu_epilogue"][0]()
        glu = act.clone()
        fns["gate_up_then_split_glu"][0]()
        torch.cuda.synchronize()
        same = bool(torch.equal(glu, act))
        ms = alternate({k: f for k, (f, _) in fns.items()}, reps)
        r = {"part": "gemm", "rows": rows, "glu_forms_bit_identical": same}
        for k, (_, flop) in fns.items():
            per = ms[k] / 5
            r[k] = {"ms": per, "tflops": flop / 5 / per / 1e9, "share_of_fp16_peak": flop / 5 / per / 1e9 / DENSE_FP16_PEAK}
        r["glu_epilogue_over_split"] = ms["gate_up_glu_epilogue"] / ms["gate_up_then_split_glu"]
        out.append(r)
        del x, y, act
    del w
    torch.cuda.empty_cache()
    return out


def _linear_flop(cfg, tokens):
    nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
    per_tok = cfg.hidden * (nq + 2 * nkv) + nq * cfg.hidden + cfg.hidden * 2 * cfg.inter + cfg.inter * cfg.hidden
    return 2.0 * tokens * per_tok * cfg.n_layers


def part_config4(G, w, dev, reps, batch=32, prompt_len=128, gen=16):
    cfg = w.cfg
    run = G.GptqRunner(w, batch=batch, max_ctx=4096)
    run.capture()
    pre = G.GptqPrefill(w, max_tokens=batch * prompt_len, runner=run)
    rng = np.random.default_rng(0xC4)
    prompts = [rng.integers(0, cfg.vocab, size=prompt_len).tolist() for _ in range(batch)]

    def prefill():
        return pre.forward_batch(prompts, slots=range(batch))[0]

    def replays():
        run.reset()
        for i in range(prompt_len):
            run.set_tokens([p[i] for p in prompts])
            run.replay()
        return run.logits()

    ms = alternate({"forward_batch": prefill, "decode_replays": replays}, reps)
    tokens = batch * prompt_len

    def gap():
        lg = run.logits().float()
        top2 = torch.topk(lg, 2, dim=-1).values
        return ((top2[:, 0] - top2[:, 1]) / lg.abs().amax(dim=-1)).cpu().tolist()

    def continue_(start):
        """tokens [gen + 1, batch] from the first sampled one on, and the top-2 gap of the logits behind each (as a
        share of the row's logit scale; meaningful on the replay side, whose runner computed every one of them)"""
        first_logits = start().float().clone()
        ids, gaps = [run.meta["token_ids"].cpu().tolist()], [gap()]
        for _ in range(gen):
            run.replay()
            ids.append(run.meta["token_ids"].cpu().tolist())
            gaps.append(gap())
        return np.array(ids), np.array(gaps), first_logits

    a_ids, _, a_logits = continue_(prefill)
    b_ids, b_gaps, b_logits = continue_(replays)
    logit_err = float((a_logits - b_logits).abs().max() / b_logits.abs().max())
    first_diff = [int(np.argmax(a_ids[:, r] != b_ids[:, r])) if (a_ids[:, r] != b_ids[:, r]).any() else -1
                  for r in range(batch)]
    # a fork is explained when the replay side's logits behind the first differing token have a near-tie: the two
    # sides' hidden states differ by f32 summation order, and 1 % of the logit scale covers that
    unexplained = [r for r, d in enumerate(first_diff) if d >= 0 and b_gaps[d, r] > 1e-2]
    r = {"part": "config4", "workload": f"{batch} prompts x {prompt_len} tokens, Mistral-7B GPTQ g128, {cfg.n_layers} layers",
         **ms, "forward_batch_tok_s": tokens / ms["forward_batch"] * 1e3, "decode_replays_tok_s": tokens / ms["decode_replays"] * 1e3,
         "replays_over_forward_batch": ms["decode_replays"] / ms["forward_batch"],
         "forward_batch_linear_tflops": _linear_flop(cfg, tokens) / ms["forward_batch"] / 1e9,
         "continuation_tokens": gen, "rows_forked": sum(d >= 0 for d in first_diff), "first_token_equal": bool((a_ids[0] == b_ids[0]).all()),
         "forks_without_near_tie": unexplained,
         "first_logits_max_err_of_scale": logit_err}
    del pre, run
    torch.cuda.empty_cache()
    return r


def part_ttft(G, w, dev, reps, T=4096):
    cfg = w.cfg
    pre = G.GptqPrefill(w, max_tokens=T)
    prompt = np.random.default_rng(0x77).integers(0, cfg.vocab, size=T).tolist()
    pre.forward(prompt)
    torch.cuda.synchronize()
    ms = timed(lambda: pre.forward(prompt), reps)
    nq = cfg.n_heads * cfg.head_dim
    attn = 2.0 * T * T * nq * cfg.n_layers                  # causal QK^T and PV: 2 x 2 x T^2 / 2 x nq per layer
    flop = _linear_flop(cfg, T) + attn + 2.0 * cfg.hidden * cfg.vocab
    r = {"part": "ttft", "workload": f"one {T}-token prompt, Mistral-7B GPTQ g128, {cfg.n_layers} layers", "ms": ms,
         "tflops": flop / ms / 1e9, "share_of_fp16_peak": flop / ms / 1e9 / DENSE_FP16_PEAK}
    del pre
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="gemm,config4,ttft")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--gemm-rows", default="512,2048,4096", help="comma-separated row counts")
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gptq_prefill: needs a GPU")
    graft.load_package()
    from mistralrs_b200 import gptq_model as G
    dev = torch.device("cuda:0")
    lines = []

    def emit(r):
        print(json.dumps(r), flush=True)
        lines.append(r)
    emit(gpu_info())
    parts = args.parts.split(",")
    if "gemm" in parts:
        for r in part_gemm(G, dev, [int(x) for x in args.gemm_rows.split(",")], max(args.reps, 10)):
            emit(r)
    if {"config4", "ttft"} & set(parts):
        # scales of 2^U(-10, -8): with the default 2^U(-8, -6) the synthetic residual stream passes the f16 range within
        # four layers, and the continuation check would compare argmaxes of NaN logits.  Timings do not depend on it.
        w = G.GptqWeights(G.GptqConfig.mistral_7b(n_layers=args.layers, scale_exp=(-10, -8)), dev)
        if "config4" in parts:
            emit(part_config4(G, w, dev, args.reps))
        if "ttft" in parts:
            emit(part_ttft(G, w, dev, args.reps))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
