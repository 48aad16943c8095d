"""GPTQ / AWQ checkpoints on the int4 stack: what does loading a Mistral-7B-shaped checkpoint cost, and what does act-order
(one column gather per layer before o_proj, permuted norms in front of q||k||v and gate||up) add to a decode step?

Three seeded Mistral-7B-shaped checkpoints (32 layers, g128) are written one at a time into a temporary directory under
--out, measured, and deleted: GPTQ without act-order, GPTQ with act-order, AWQ.  Per checkpoint:
  load_s            GptqWeights.from_checkpoint wall time (read, host transform, upload, repack)
  decode_ms[B]      graph-replayed decode step at batch 1, 32 and 64: median of --reps CUDA-event timings of --steps replays
  prefill_ms        one GptqPrefill.forward_batch of 32 prompts of 128 tokens (median of --reps, after one warm-up)
The act-order overhead is each act-order number against the natural-order GPTQ checkpoint's.  The first line gives
the GPU name and power limit from nvidia-smi, read in the same run; the last line is the JSON of everything.
Usage: python scripts/bench_gptq_checkpoint.py [--out DIR (default: the system temporary directory)] [--steps 32] [--reps 5]
       [--layers 32]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))      # the seeded checkpoint writer of the host tests

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402

CHECKPOINTS = (("gptq_g128", "gptq", False), ("gptq_g128_act_order", "gptq", True), ("awq_g128", "awq", False))


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power = [x.strip() for x in out[0].split(",")] if out else (torch.cuda.get_device_name(), "unknown")
    return {"gpu": name, "power_limit": power}


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def measure(G, path, dev, steps, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    w = G.GptqWeights.from_checkpoint(path, dev)
    torch.cuda.synchronize()
    res = {"load_s": time.perf_counter() - t0, "act_order_o": w.act_order_o, "decode_ms": {}}
    for B in (1, 32, 64):
        run = G.GptqRunner(w, batch=B, max_ctx=(steps + 2) * reps + 64)
        run.capture()
        run.set_tokens([(17 * b + 1) % w.cfg.vocab for b in range(B)])

        def replays():
            for _ in range(steps):
                run.replay()
        replays()                                   # warm-up
        res["decode_ms"][B] = timed(replays, reps - 1) / steps
        del run
    pre = G.GptqPrefill(w, max_tokens=32 * 128)
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, w.cfg.vocab, size=128).tolist() for _ in range(32)]
    per = 128 // w.cfg.block_size
    tables = [pre.table[i * per:(i + 1) * per] for i in range(32)]       # the prefill's own cache, 128 rows each
    pre.forward_batch(prompts, tables=tables)
    res["prefill_ms"] = timed(lambda: pre.forward_batch(prompts, tables=tables), reps)
    del pre, w
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=tempfile.gettempdir(), help="the checkpoints are written under (and removed from) it")
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--layers", type=int, default=32)
    args = ap.parse_args()
    graft.load_package()
    from mistralrs_b200 import gptq_model as G
    from test_gptq_checkpoint_host import make_checkpoint
    dev = torch.device("cuda:0")
    info = gpu_info()
    print(json.dumps(info), flush=True)
    os.makedirs(args.out, exist_ok=True)
    cfg = G.GptqConfig.mistral_7b(n_layers=args.layers)
    out = dict(info, model=f"Mistral-7B shape, {args.layers} layers, g128", results={})
    for i, (name, method, act) in enumerate(CHECKPOINTS):
        d = tempfile.mkdtemp(prefix=name + "-", dir=args.out)
        try:
            make_checkpoint(d, cfg, method=method, act_order=act, seed=0xC400 + i, shards=2)
            r = measure(G, d, dev, args.steps, args.reps)
        finally:
            shutil.rmtree(d, ignore_errors=True)
        out["results"][name] = r
        print(name, json.dumps(r), flush=True)
    base, act = out["results"]["gptq_g128"], out["results"]["gptq_g128_act_order"]
    out["act_order_overhead"] = {f"decode_b{B}": act["decode_ms"][B] / base["decode_ms"][B] - 1 for B in base["decode_ms"]}
    out["act_order_overhead"]["prefill_32x128"] = act["prefill_ms"] / base["prefill_ms"] - 1
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
