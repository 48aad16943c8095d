"""Speculative decoding of a GPTQ model: Mistral-7B GPTQ int4 g128 (synthetic seeded weights, 32 layers, f16, HND
cache), every sequence with its own 128-token prompt.  The synthetic group scales are 2^U(-10, -8) instead of
GptqConfig's 2^U(-8, -6): with those, the 32-layer residual stream leaves the f16 range and most rows' logits are NaN,
which makes every greedy stream a string of token 0.  The scales change no kernel's work, only the values.  What does a verify step of B * (k + 1) rows cost next to a plain
decode step of B rows, and at which draft acceptance does verification start to pay?

Prints one JSON line:
  gpu / power_limit           read with nvidia-smi in the same run
  batches[B].steps[q]         median ms per graph replay (CUDA events, --replays replays, every sequence at a 128-token
                              context) of the plain decode step (q = 1) and of the verify step at q = 2, 4, 8, with the
                              linear-only (attention skipped, skip_mask 1) and attention-only (linears skipped,
                              skip_mask 2) splits, and the ratio to the plain step
  batches[B].break_even[k]    the acceptance a at which a verify step's 1 + a*k tokens per sequence cost what 1 + a*k
                              plain steps cost: (verify_ms(k + 1) / plain_ms - 1) / k, from the measured step times;
                              above 1 verification does not pay at any acceptance
  batches[B].plain            --gen greedy tokens per sequence through the decode graph: device-only tok/s, and tok/s
                              with one host round trip per step (H2D of the input ids, D2H of the sampled ids)
  batches[B].generation[k][a] --gen tokens per sequence by speculative_generate with drafts from the plain greedy
                              trajectory, every draft position corrupted with a seeded probability chosen for a mean
                              acceptance of a: tok/s (host clock around work that ends in a device synchronise), steps,
                              measured acceptance, how many streams equal their plain greedy stream, and for those
                              that do not, the median position of the first differing token and the largest top-2
                              margin (share of the row's largest |logit|) of the plain step that chose it there
Token rates count the tokens of all B sequences.
Usage: python scripts/bench_gptq_speculative.py [--batches 1,8,32,64,128] [--replays 50] [--gen 128] [--layers N]
       [--out FILE]"""
import argparse
import itertools
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402
from bench_speculative import corruption_for, emit, gpu_info, step_costs  # noqa: E402

PROMPT_LEN = 128
SCALE_EXP = (-10, -8)
KS = (1, 3, 7)
TARGETS = (1.0, 0.8, 0.5)


def max_ctx(n):
    return PROMPT_LEN + (max(KS) + 1) * n + 32


def run_batch(G, M, w, B, args):
    cfg, dev, n = w.cfg, w.device, args.gen
    # room for a sequence that accepts every draft at every step to run ahead of one that accepts none
    runner = G.GptqRunner(w, batch=B, max_ctx=max_ctx(n))
    vers = {k: G.GptqVerifier(runner, draft_len=k) for k in KS}
    steps = step_costs(runner, vers, "linear_ms", args.replays, ctx=PROMPT_LEN)
    for row in steps.values():
        row["vs_plain"] = row["total_ms"] / steps[1]["total_ms"]
    break_even = {str(k): (steps[k + 1]["total_ms"] / steps[1]["total_ms"] - 1) / k for k in KS}

    # every sequence its own prompt in its own table; generation only writes positions >= PROMPT_LEN, so the prompts
    # stay in the cache across the runs below
    runner.reset()
    runner.capture()
    for v in vers.values():
        v.capture()
    per_call = max(1, runner.max_ctx // PROMPT_LEN)
    pre = G.GptqPrefill(w, max_tokens=per_call * PROMPT_LEN, runner=runner)
    prompts = [[1000 + ((131 + 17 * b + i) % 2048) for i in range(PROMPT_LEN)] for b in range(B)]
    firsts = []
    for i in range(0, B, per_call):
        _, f = pre.forward_batch(prompts[i:i + per_call], tables=[runner.tables[b] for b in range(i, min(i + per_call, B))])
        firsts += f.tolist()

    def start():
        runner.reset(PROMPT_LEN)
        runner.set_tokens(firsts)
        torch.cuda.synchronize()

    start()
    ids = torch.zeros(n, B, dtype=torch.int32, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        runner.replay()
        ids[i].copy_(runner.meta["token_ids"])
    e1.record()
    torch.cuda.synchronize()
    plain_ids = ids.t().cpu().tolist()
    plain = {"tok_s_device": B * n / (e0.elapsed_time(e1) / 1e3)}
    start()
    tok_h = torch.tensor(firsts, dtype=torch.int32).pin_memory()
    t0 = time.perf_counter()
    for _ in range(n):
        runner.meta["token_ids"].copy_(tok_h, non_blocking=True)
        runner.replay()
        tok_h.copy_(runner.meta["token_ids"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
    plain["tok_s_host_loop"] = B * n / (time.perf_counter() - t0)
    # untimed: the top-2 margin of every plain step, to tell near-ties from real disagreements below
    start()
    margins = torch.zeros(n, B, device=dev)
    for i in range(n):
        runner.replay()
        ids[i].copy_(runner.meta["token_ids"])
        top2 = torch.topk(runner.logits().float(), 2, dim=1).values
        margins[i] = (top2[:, 0] - top2[:, 1]) / runner.logits().float().abs().amax(dim=1)
    plain["repeatable"] = ids.t().cpu().tolist() == plain_ids
    margins = margins.t().cpu().tolist()

    gen = {}
    for k in KS:
        gen[str(k)] = {}
        for target in TARGETS:
            e = corruption_for(target, k)
            rng = np.random.default_rng(int(1000 * target) + k)
            calls = itertools.count()

            def propose(history, k=k, e=e, rng=rng, calls=calls):
                # speculative_generate asks for the drafts of sequences 0 .. B-1 in order, once per step
                b = next(calls) % B
                at = len(history) - 1
                d = [plain_ids[b][at + i] if at + i < n else 0 for i in range(k)]
                return [(t + 1) % cfg.vocab if rng.random() < e else t for t in d]
            start()
            t0 = time.perf_counter()
            streams, acc = M.speculative_generate(vers[k], firsts, n, propose)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            a = np.array(acc)
            mism = {b: next(i for i, (x, y) in enumerate(zip(streams[b], plain_ids[b])) if x != y)
                    for b in range(B) if streams[b] != plain_ids[b]}
            gen[str(k)][str(target)] = {"tok_s": B * n / dt, "vs_plain_host_loop": B * n / dt / plain["tok_s_host_loop"],
                                        "steps": len(acc), "mean_accepted": float(a.mean()),
                                        "acceptance": float(a.mean() / k), "streams_equal_plain_greedy": B - len(mism),
                                        "first_mismatch_median": float(np.median(list(mism.values()))) if mism else None,
                                        "first_mismatch_max_margin": max((margins[b][i] for b, i in mism.items()),
                                                                         default=None)}
    del vers, runner, pre
    torch.cuda.empty_cache()
    return {"steps": {str(q): v for q, v in steps.items()}, "break_even": break_even, "plain": plain, "generation": gen}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32,64,128", help="comma-separated sequence counts (1..256)")
    ap.add_argument("--replays", type=int, default=50)
    ap.add_argument("--gen", type=int, default=128, help="tokens generated per sequence")
    ap.add_argument("--layers", type=int, default=0, help="truncate the model (rehearsal only)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    batches = [int(b) for b in args.batches.split(",")]
    if not all(1 <= b <= 256 for b in batches):
        raise SystemExit(f"--batches must lie in 1..256, got {batches}")
    if not torch.cuda.is_available():
        raise SystemExit("bench_gptq_speculative.py needs a CUDA device")
    graft.load_package()
    from mistralrs_b200 import gptq_model as G, model as M
    dev = torch.device("cuda:0")
    info = gpu_info()
    cfg = G.GptqConfig.mistral_7b(max_pos=max_ctx(args.gen), scale_exp=SCALE_EXP)
    if args.layers:
        cfg.n_layers = args.layers
    w = G.GptqWeights(cfg, dev)
    res = {"metric": "gptq_speculative_decode", "model": f"mistral-7b gptq g128 synthetic (scales 2^U{SCALE_EXP}), {cfg.n_layers} layers, f16, hnd",
           "prompt": PROMPT_LEN, "generated": args.gen, "replays": args.replays, **info, "batches": {}}
    for B in batches:
        res["batches"][str(B)] = run_batch(G, M, w, B, args)
        print(f"B={B}: " + json.dumps(res["batches"][str(B)]["steps"]), file=sys.stderr, flush=True)
        if args.out:                                  # the batches so far, should a later one not finish
            with open(args.out, "w") as f:
                f.write(json.dumps(res) + "\n")
    emit(res, args.out)


if __name__ == "__main__":
    main()
