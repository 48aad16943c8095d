"""Speculative decoding on the headline workload: Llama-3-8B Q4_K_M (synthetic weights), batch 1, a 128-token prompt
through LlamaPrefill(runner=...), then greedy generation.  What does a verify step of q = k + 1 rows cost next to a
plain decode step, and what does that buy in tokens per second at a given draft acceptance?

Prints one JSON line:
  gpu / power_limit         read with nvidia-smi in the same run
  steps[q]                  median ms per graph replay (CUDA events, >= --replays replays, context fixed at 256) of
                            the plain decode step (q = 1) and of the verify step at q = 2, 4, 8, with the GEMV-only
                            (attention skipped, skip_mask 1) and attention-only (GEMVs skipped, skip_mask 2) splits
  plain                     256 greedy tokens through the decode graph: device-only tok/s, and tok/s with one host
                            round trip per token (H2D of the input id, D2H of the sampled id), the way a serving loop
                            that looks at every token runs it
  generation[k][target]     256 tokens by speculative_generate with drafts from the plain greedy trajectory, every draft
                            position corrupted with a seeded probability chosen for a mean acceptance of `target`:
                            tok/s (host clock around work that ends in a device synchronise), mean accepted drafts per
                            step, measured acceptance, and whether the stream equals the plain greedy one
--batch B > 1 runs B sequences, each with its own 128-token prompt prefilled into its own block table.  Batches of 9
and more take the dequant-GEMM route for plain and verify steps alike, so the step splits are named linear_ms there.
Step costs are measured at q = 2, 4, 8 (those that fit the 8 rows of the GEMV route when B <= 8); the plain and
generation rates count the tokens of all B sequences, and generation reports how many of the B streams equal their
plain greedy stream (with the first differing position of each that does not).
Usage: python scripts/bench_speculative.py [--batch 1] [--replays 200] [--layers N] [--out FILE]"""
import argparse
import itertools
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402

PROMPT_LEN, GEN_LEN = 128, 256


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in out[0].split(",")] if out else ("unknown", "unknown", "unknown")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def median_replay_ms(graph, runner, ctx, n):
    """median of n single-replay CUDA-event timings; the context is reset before each replay so every one does the
    same work (the reset is outside the timed window)"""
    for _ in range(5):
        runner.context_lens.fill_(ctx); graph.replay()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for e0, e1 in ev:
        runner.context_lens.fill_(ctx)
        e0.record(); graph.replay(); e1.record()
    torch.cuda.synchronize()
    return float(np.median([e0.elapsed_time(e1) for e0, e1 in ev]))


def capture_forward(fwd):
    fwd(); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fwd()
    return g


def corruption_for(target, k):
    """per-position corruption probability e with E[accepted] / k = target when every draft is wrong with prob. e"""
    if target >= 1.0:
        return 0.0
    lo, hi = 0.0, 1.0
    for _ in range(60):
        e = (lo + hi) / 2
        rate = sum((1 - e) ** i for i in range(1, k + 1)) / k
        lo, hi = (e, hi) if rate > target else (lo, e)
    return (lo + hi) / 2


def step_costs(runner, vers, linear, replays, ctx=PROMPT_LEN + GEN_LEN // 2):
    """step cost: plain decode and verify at q = k + 1 for every verifier, whole and split (`linear`: the name of the
    linear-only split), every step at context `ctx`"""
    steps = {}
    for q in (1,) + tuple(k + 1 for k in vers):
        s = runner.step_struct if q == 1 else vers[q - 1].step_struct
        fwd = runner.forward if q == 1 else vers[q - 1].forward
        row = {}
        for name, mask in (("total_ms", 0), (linear, 1), ("attention_ms", 2)):
            s.skip_mask = mask
            runner.context_lens.fill_(ctx)
            (runner.advance if q == 1 else vers[q - 1].advance)()      # metadata of a context-`ctx` step
            row[name] = median_replay_ms(capture_forward(fwd), runner, ctx + q, replays)
        s.skip_mask = 0
        row["ms_per_row"] = row["total_ms"] / q
        steps[q] = row
    return steps


def emit(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1, help="sequences per step (1..256)")
    ap.add_argument("--replays", type=int, default=200)
    ap.add_argument("--layers", type=int, default=0, help="truncate the model (rehearsal only)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not 1 <= args.batch <= 256:
        raise SystemExit(f"--batch must be 1..256, got {args.batch}")
    if not torch.cuda.is_available():
        raise SystemExit("bench_speculative.py needs a CUDA device")
    graft.load_package()
    from mistralrs_b200 import model as M
    dev = torch.device("cuda:0")
    info = gpu_info()
    cfg = M.LlamaConfig.llama3_8b()
    if args.layers:
        cfg.n_layers = args.layers
    w = M.LlamaWeights(cfg, dev)
    if args.batch > 1:
        emit(run_batched(M, w, cfg, dev, info, args), args.out)
        return
    ks = (1, 3, 7)
    runner = M.LlamaRunner(w, batch=1, max_ctx=PROMPT_LEN + GEN_LEN + 32, pdl=True)
    vers = {k: M.LlamaVerifier(runner, draft_len=k) for k in ks}
    steps = step_costs(runner, vers, "gemv_ms", args.replays)

    # ---- plain greedy generation (the reference stream)
    runner.reset()
    runner.capture()
    for v in vers.values():
        v.capture()
    pre = M.LlamaPrefill(w, max_tokens=PROMPT_LEN, runner=runner)
    prompt = [1000 + ((131 + i) % 2048) for i in range(PROMPT_LEN)]

    def prefill():
        logits = pre.forward(prompt)
        runner.reset(PROMPT_LEN)
        return int(torch.argmax(logits))

    first = prefill()
    runner.set_tokens([first])
    ids = torch.zeros(GEN_LEN, dtype=torch.int32, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(GEN_LEN):
        runner.graph.replay()
        ids[i].copy_(runner.meta["token_ids"][0])
    e1.record()
    torch.cuda.synchronize()
    plain_ids = ids.cpu().tolist()
    plain = {"tok_s_device": GEN_LEN / (e0.elapsed_time(e1) / 1e3)}
    first = prefill()
    tok_h = torch.zeros(1, dtype=torch.int32).pin_memory()
    tok_h[0] = first
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(GEN_LEN):
        runner.meta["token_ids"].copy_(tok_h, non_blocking=True)
        runner.graph.replay()
        tok_h.copy_(runner.meta["token_ids"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
    plain["tok_s_host_loop"] = GEN_LEN / (time.perf_counter() - t0)

    # ---- speculative generation with drafts from the plain trajectory
    gen = {}
    for k in ks:
        gen[k] = {}
        for target in (1.0, 0.8, 0.5):
            e = corruption_for(target, k)
            rng = np.random.default_rng(int(1000 * target) + k)

            def propose(history, k=k, e=e, rng=rng):
                at = len(history) - 1
                d = [plain_ids[at + i] if at + i < GEN_LEN else 0 for i in range(k)]
                return [(t + 1) % cfg.vocab if rng.random() < e else t for t in d]
            first = prefill()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            streams, acc = M.speculative_generate(vers[k], [first], GEN_LEN, propose)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            a = np.array(acc)[:, 0]
            match = streams[0] == plain_ids
            gen[k][str(target)] = {"tok_s": GEN_LEN / dt, "steps": len(acc), "mean_accepted": float(a.mean()),
                                   "acceptance": float(a.mean() / k), "tokens_per_step": float(GEN_LEN / len(acc)),
                                   "equals_plain_greedy": bool(match),
                                   "first_mismatch": None if match else next(i for i, (x, y) in enumerate(zip(streams[0], plain_ids)) if x != y)}
    res = {"metric": "speculative_decode", "model": f"llama-3-8b q4_k_m synthetic, {cfg.n_layers} layers", "batch": 1,
           "prompt": PROMPT_LEN, "generated": GEN_LEN, "replays": args.replays, **info,
           "steps": {str(q): v for q, v in steps.items()}, "plain": plain, "generation": {str(k): v for k, v in gen.items()}}
    emit(res, args.out)


def run_batched(M, w, cfg, dev, info, args):
    """--batch B > 1: the same measurements over B sequences with their own prompts and tables"""
    B = args.batch
    ks = tuple(k for k in (1, 3, 7) if B > M.MMVQ_MAX_BATCH or B * (k + 1) <= M.MMVQ_MAX_BATCH)
    linear = "gemv_ms" if B <= M.MMVQ_MAX_BATCH else "linear_ms"
    # room for a sequence that accepts more than the others to run ahead of the slowest one
    runner = M.LlamaRunner(w, batch=B, max_ctx=PROMPT_LEN + 2 * GEN_LEN + 32, pdl=True)
    vers = {k: M.LlamaVerifier(runner, draft_len=k) for k in ks}
    steps = step_costs(runner, vers, linear, args.replays)
    for row in steps.values():
        row["vs_plain"] = row["total_ms"] / steps[1]["total_ms"]

    # every sequence its own prompt in its own table; generation only writes positions >= PROMPT_LEN, so the prompts
    # stay in the cache across the runs below
    runner.reset()
    runner.capture()
    for v in vers.values():
        v.capture()
    pre = M.LlamaPrefill(w, max_tokens=PROMPT_LEN, runner=runner)
    firsts = []
    for b in range(B):
        prompt = [1000 + ((131 + 17 * b + i) % 2048) for i in range(PROMPT_LEN)]
        firsts.append(int(torch.argmax(pre.forward(prompt, table=runner.tables[b]))))

    def start():
        runner.reset(PROMPT_LEN)
        runner.set_tokens(firsts)
        torch.cuda.synchronize()

    start()
    ids = torch.zeros(GEN_LEN, B, dtype=torch.int32, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(GEN_LEN):
        runner.graph.replay()
        ids[i].copy_(runner.meta["token_ids"])
    e1.record()
    torch.cuda.synchronize()
    plain_ids = ids.t().cpu().tolist()
    plain = {"tok_s_device": B * GEN_LEN / (e0.elapsed_time(e1) / 1e3)}
    start()
    tok_h = torch.tensor(firsts, dtype=torch.int32).pin_memory()
    t0 = time.perf_counter()
    for _ in range(GEN_LEN):
        runner.meta["token_ids"].copy_(tok_h, non_blocking=True)
        runner.graph.replay()
        tok_h.copy_(runner.meta["token_ids"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
    plain["tok_s_host_loop"] = B * GEN_LEN / (time.perf_counter() - t0)

    gen = {}
    for k in ks:
        gen[k] = {}
        for target in (1.0, 0.8, 0.5):
            e = corruption_for(target, k)
            rng = np.random.default_rng(int(1000 * target) + k)
            calls = itertools.count()

            def propose(history, k=k, e=e, rng=rng, calls=calls):
                # speculative_generate asks for the drafts of sequences 0 .. B-1 in order, once per step (two
                # sequences may share a first token, so that cannot tell them apart)
                b = next(calls) % B
                assert history[0] == firsts[b]
                at = len(history) - 1
                d = [plain_ids[b][at + i] if at + i < GEN_LEN else 0 for i in range(k)]
                return [(t + 1) % cfg.vocab if rng.random() < e else t for t in d]
            start()
            t0 = time.perf_counter()
            streams, acc = M.speculative_generate(vers[k], firsts, GEN_LEN, propose)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            a = np.array(acc)
            mism = {b: next(i for i, (x, y) in enumerate(zip(streams[b], plain_ids[b])) if x != y)
                    for b in range(B) if streams[b] != plain_ids[b]}
            gen[k][str(target)] = {"tok_s": B * GEN_LEN / dt, "steps": len(acc), "mean_accepted": float(a.mean()),
                                   "acceptance": float(a.mean() / k),
                                   "tokens_per_step": float(1 + a.mean()),
                                   "streams_equal_plain_greedy": B - len(mism),
                                   "first_mismatch": {str(b): i for b, i in mism.items()}}
    return {"metric": "speculative_decode", "model": f"llama-3-8b q4_k_m synthetic, {cfg.n_layers} layers", "batch": B,
            "route": "gemv" if B <= M.MMVQ_MAX_BATCH else "gemm", "prompt": PROMPT_LEN, "generated": GEN_LEN,
            "replays": args.replays, **info, "steps": {str(q): v for q, v in steps.items()}, "plain": plain,
            "generation": {str(k): v for k, v in gen.items()}}


if __name__ == "__main__":
    main()
