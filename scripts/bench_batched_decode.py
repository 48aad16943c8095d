"""Batched GGUF decode on the headline model: Llama-3-8B Q4_K_M (synthetic weights), context fixed at 256, PDL on.
Batches of 1..8 run the GEMV chain (MMVQ), 9..256 the dequant-GEMM chain (the reference's MMQ branch).  What does a
step cost per batch, and how much of the weight stream's bandwidth do the linears reach?

Prints one JSON line per batch B in {1, 8, 9, 16, 32, 64, 128, 256}:
  step_ms / linear_ms / attention_ms   median ms of >= --replays single-graph-replay CUDA-event timings of the whole
                                       step, the linear-only split (attention skipped, skip_mask 1) and the
                                       attention-only split (linears skipped, skip_mask 2)
  tok_s                                B / step
  linear_bw_share                      weight bytes per step / linear_ms as a share of the 3.35 TB/s data-sheet HBM3
                                       bandwidth of the H100 SXM
and, for B = 16, two_batch8_ms: two batch-8 steps back to back in one graph (what a caller of a GEMV-only decode chain
has to run for 16 sequences).  The first line gives the GPU name, power limit and max SM clock from nvidia-smi.
Usage: python scripts/bench_batched_decode.py [--replays 100] [--layers N] [--batches 1,8,9,...]"""
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

CTX = 256
WEIGHT_BYTES = 4_616_331_264     # Llama-3-8B Q4_K_M: every linear incl. the lm_head, read once per step
HBM_BPS = 3.35e12                # H100 SXM data sheet


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in out[0].split(",")] if out else ("unknown", "unknown", "unknown")
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def capture(fn):
    fn(); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def median_replay_ms(graph, runner, n):
    """median of n single-replay CUDA-event timings; every replay runs the step at context CTX (the step's metadata
    was advanced once before capture; the fused attention rewrites the same cache slot each time)"""
    for _ in range(5):
        graph.replay()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for e0, e1 in ev:
        e0.record(); graph.replay(); e1.record()
    torch.cuda.synchronize()
    return float(np.median([e0.elapsed_time(e1) for e0, e1 in ev]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=100)
    ap.add_argument("--layers", type=int, default=0, help="truncate the model (rehearsal only)")
    ap.add_argument("--batches", default="1,8,9,16,32,64,128,256")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batched_decode.py needs a CUDA device")
    graft.load_package()
    from mistralrs_b200 import model as M
    dev = torch.device("cuda:0")
    print(json.dumps(gpu_info()), flush=True)
    cfg = M.LlamaConfig.llama3_8b()
    if args.layers:
        cfg.n_layers = args.layers
    w = M.LlamaWeights(cfg, dev)
    for B in [int(b) for b in args.batches.split(",")]:
        run = M.LlamaRunner(w, batch=B, max_ctx=CTX + 32, pdl=True)
        run.set_tokens([(1000 + 31 * b) % cfg.vocab for b in range(B)])
        run.context_lens.fill_(CTX - 1)
        run.advance()                                # metadata of a step at context CTX
        row = {"batch": B, "route": "gemv" if B <= M.MMVQ_MAX_BATCH else "gemm", "context": CTX, "replays": args.replays}
        for name, mask in (("step_ms", 0), ("linear_ms", 1), ("attention_ms", 2)):
            run.step_struct.skip_mask = mask
            row[name] = round(median_replay_ms(capture(run.forward), run, args.replays), 4)
        run.step_struct.skip_mask = 0
        row["tok_s"] = round(B / row["step_ms"] * 1e3, 1)
        if not args.layers:
            row["linear_bw_share"] = round(WEIGHT_BYTES / (row["linear_ms"] * 1e-3) / HBM_BPS, 4)
        if B == 16:
            r8 = M.LlamaRunner(w, batch=8, max_ctx=CTX + 32, pdl=True)
            r8.set_tokens([(1000 + 31 * b) % cfg.vocab for b in range(8)])
            r8.context_lens.fill_(CTX - 1)
            r8.advance()
            row["two_batch8_ms"] = round(median_replay_ms(capture(lambda: (r8.forward(), r8.forward())), r8, args.replays), 4)
            del r8
        print(json.dumps(row), flush=True)
        del run
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
