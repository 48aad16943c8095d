"""Prefix-cache and chunked prefill on the config-3 model (Llama-3-8B shape, Q8_0 blocks everywhere, synthetic weights
generated on the device as bench.py's config 3 does, 4096-token prompt), timed with CUDA events after warm-up:

  (a) full prefill of the 4096-token prompt
  (b) 3584 tokens already cached, the 512-token suffix prefilled (`LlamaPrefill.forward(cached=3584)`)
  (c) the same prompt in 4 chunks of 1024 (sum of the four calls)
  (d) prompt attention alone, 32 heads / 8 KV heads / head 128, bf16: the paged kernel over a page-16 cache at
      cached = 0 against mrs_prefill_attention on the same q / k / v, and the paged kernel for (b)'s 512 x 4096 shape;
      TFLOP/s from the visible (query, key) pairs, 4 * head_dim FLOPs per pair and head.

Prints one JSON line with the GPU's name and power limit, read in the same run.  Writes nothing to disk.
usage: python scripts/bench_prefix_prefill.py [--steps 5] [--layers 0]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True)
    return out.stdout.strip() if out.returncode == 0 else "nvidia-smi unavailable"


def timed(torch, fn, steps):
    """median seconds of `steps` calls of fn, each between two CUDA events"""
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--layers", type=int, default=0, help="truncate the model (0: all 32 layers)")
    args = ap.parse_args()

    import torch
    import __graft_entry__ as graft
    graft.load_package()
    from mistralrs_b200 import model as M, paged_attn

    if not torch.cuda.is_available():
        raise SystemExit("bench_prefix_prefill.py needs a CUDA device")
    dev = torch.device("cuda:0")
    prompt, cached, chunk = 4096, 3584, 1024
    toks = [1000 + ((131 + i) % 2048) for i in range(prompt)]
    cfg = M.LlamaConfig.llama3_8b(quant="q8_0")
    if args.layers:
        cfg.n_layers = args.layers
    w = M.LlamaWeights(cfg, dev, fast_synth=True)
    pre = M.LlamaPrefill(w, max_tokens=prompt)

    def chunks():
        for c in range(0, prompt, chunk):
            pre.forward(toks[c:c + chunk], cached=c)

    pre.forward(toks)                                   # warm-up of every shape the timed windows use
    pre.forward(toks[cached:], cached=cached)
    chunks()
    torch.cuda.synchronize()
    full = timed(torch, lambda: pre.forward(toks), args.steps)
    suffix = timed(torch, lambda: pre.forward(toks[cached:], cached=cached), args.steps)   # rows < 3584 stay in the cache
    chunked = timed(torch, chunks, args.steps)

    H, KVH, D, page = cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, 16
    gen = torch.Generator(device=dev).manual_seed(0)
    q, k, v = (torch.randn(prompt, h, D, device=dev, generator=gen).to(torch.bfloat16) for h in (H, KVH, KVH))
    nb = prompt // page
    kc = k.view(nb, page, KVH, D).transpose(1, 2).contiguous()      # token t -> block t // page, row t % page
    vc = v.view(nb, page, KVH, D).transpose(1, 2).contiguous()
    bt = torch.arange(nb, dtype=torch.int32, device=dev)[None]
    cu = lambda n: torch.tensor([0, n], dtype=torch.int32, device=dev)
    scale = D ** -0.5
    reps = 20
    fresh_fn = lambda: [paged_attn.prefill_attention(q, k, v, scale) for _ in range(reps)]
    paged_fn = lambda: [paged_attn.prefill_attention_paged(q, kc, vc, bt, cu(prompt), cu(prompt), prompt, prompt, scale)
                        for _ in range(reps)]
    qs = q[cached:]
    cu_s, cu_k = cu(prompt - cached), cu(prompt)
    suffix_fn = lambda: [paged_attn.prefill_attention_paged(qs, kc, vc, bt, cu_s, cu_k, prompt - cached, prompt, scale)
                         for _ in range(reps)]
    same = torch.equal(paged_attn.prefill_attention(q, k, v, scale),
                       paged_attn.prefill_attention_paged(q, kc, vc, bt, cu(prompt), cu(prompt), prompt, prompt, scale))
    for fn in (fresh_fn, paged_fn, suffix_fn):
        fn()
    torch.cuda.synchronize()
    # alternate the two kernels so that a clock or neighbour change hits both
    t_fresh, t_paged = [], []
    for _ in range(3):
        t_fresh.append(timed(torch, fresh_fn, 1) / reps)
        t_paged.append(timed(torch, paged_fn, 1) / reps)
    t_fresh, t_paged = min(t_fresh), min(t_paged)
    t_suffix = timed(torch, suffix_fn, 3) / reps
    pairs_full = prompt * (prompt + 1) // 2
    pairs_suffix = sum(cached + i + 1 for i in range(prompt - cached))
    tflops = lambda pairs, t: 4.0 * D * H * pairs / t / 1e12

    print(json.dumps({
        "gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(dev), "layers": cfg.n_layers, "steps": args.steps,
        "workload": f"Llama-3-8B Q8_0, {prompt}-token prompt, page {cfg.block_size}",
        "a_full_prefill_ms": full * 1e3,
        "b_cached_%d_suffix_%d_ms" % (cached, prompt - cached): suffix * 1e3,
        "c_%d_chunks_of_%d_ms" % (prompt // chunk, chunk): chunked * 1e3,
        "d_attention": {
            "shape": f"{H} heads / {KVH} KV heads / D {D} / page {page}, bf16, causal, one layer",
            "fresh_ms": t_fresh * 1e3, "fresh_tflops": tflops(pairs_full, t_fresh),
            "paged_cached0_ms": t_paged * 1e3, "paged_cached0_tflops": tflops(pairs_full, t_paged),
            "paged_equals_fresh_bitwise": bool(same),
            "paged_suffix_ms": t_suffix * 1e3, "paged_suffix_tflops": tflops(pairs_suffix, t_suffix),
        },
    }))


if __name__ == "__main__":
    main()
