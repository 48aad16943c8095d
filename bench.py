#!/usr/bin/env python
"""bench.py — the quantized-linear + paged-attention hot path of mistral.rs on an H100 (sm_90a).

Headline (BASELINE.json configs[1], `--config 2`, the default): Llama-3-8B, GGUF Q4_K_M tensor types,
decode batch 1, 128-token prompt -> +256 generated tokens, synthetic weights / prompts (SURVEY §8(d)),
paged KV cache block_size 16 (FlashInfer HND layout).  Metric definitions follow the reference's
`mistralrs bench` (mistralrs-cli/src/commands/bench.rs:269-296): prefill tok/s = L / TTFT, decode
tok/s = (G - 1) / (t_last_token - t_first_token).

A "step" is one full generation; its timed region is the decode phase, bracketed by CUDA events on
the launching stream (max over ranks).  `value` replays the per-token CUDA graph with every input
resident in HBM; `e2e` drives the same graph the way a serving engine does (token id copied from
pinned host memory before every step, sampled id read back after it).  The same JSON line carries
`roofline` (dominant kernel, measured live), `cpu_baseline` (the reference's CPU arithmetic, whole
tokens on all host cores), `prefill` (BASELINE config 3: 4096-token prompt on Q8_0 weights, TTFT
including prompt attention) and `config4` (Mistral-7B GPTQ int4 decode at batch 32, both KV layouts).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config 2|3|4|5]
  torchrun --nnodes=1 --nproc-per-node N ... bench.py --gpus N      (tensor parallel)
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

PROMPT_LEN, GEN_LEN = 128, 256
GGML = {"q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8, "q2_k": 10, "q3_k": 11, "q4_k": 12, "q5_k": 13, "q6_k": 14}


def prompt_tokens(it, case=0, n=PROMPT_LEN):
    # REF bench.rs:52-55,427-430: 1000 + ((131*(it+1) + 719*case + i) mod 2048)
    return [1000 + ((131 * (it + 1) + 719 * case + i) % 2048) for i in range(n)]


def algorithmic_bytes_per_token(cfg, M, tp=1):
    """Quantized weight bytes touched once per token + KV bytes at the mean context."""
    from mistralrs_b200 import BLOCK_BYTES, BLOCK_ELEMS
    H, I = cfg.hidden, cfg.inter
    nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
    tot = 0
    for l in range(cfg.n_layers):
        for name, n in (("attn_q", nq * H), ("attn_k", nkv * H), ("attn_v", nkv * H), ("attn_output", H * nq),
                        ("ffn_gate", I * H), ("ffn_up", I * H), ("ffn_down", H * I)):
            t = M.tensor_type(cfg, name, l)
            tot += n // tp * BLOCK_BYTES[t] // BLOCK_ELEMS[t]
    t = M.tensor_type(cfg, "output", 0)
    head = cfg.vocab * H * BLOCK_BYTES[t] // BLOCK_ELEMS[t]
    mean_ctx = PROMPT_LEN + GEN_LEN // 2
    kv = 2 * (nkv // tp) * 2 * cfg.n_layers * mean_ctx
    return tot + head + kv, tot + head


class ClockSampler:
    """nvidia-smi clocks + throttle reasons during the timed region."""

    def __init__(self, gpu_index=0):
        self.proc, self.lines, self.gpu = None, [], gpu_index

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={q}", "--format=csv,noheader,nounits",
                                          "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, mx, reasons = [], 0, set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx = max(mx, float(f[1]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons),
                "samples": len(sm)}


# ------------------------------------------------------------------------------------------- CPU arm
def _cgroup_cpus():
    """CPU quota of this container (cgroup v2 cpu.max / v1 cfs quota), rounded up; 0 when unlimited or unknown"""
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        return 0 if q == "max" else max(1, -(-int(q) // int(per)))
    except Exception:
        pass
    try:
        q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
        per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
        return 0 if q <= 0 else max(1, -(-q // per))
    except Exception:
        return 0


def cpu_decode_samples(cfg, M, seconds=10.0, min_tokens=2, threads=0, nsamples=1):
    """The reference's CPU arithmetic (oracle/mrs_oracle.c: Q8_K / Q8_0 activations + integer block dots,
    the candle QMatMul algorithm) on WHOLE tokens of this model: all layers, every weight byte streamed
    from DRAM each token, attention / norms / GLU included, one pinned thread per usable host core
    (oracle/cpu_decode_bench.c).  Compiled here, on the box that runs it, with -O3 -march=native.
    `nsamples` timed samples of about `seconds` each share ONE model allocation (one short-lived child process).
    Returns ([tok/s per sample], threads, description)."""
    src = os.path.join(ROOT, "oracle", "cpu_decode_bench.c")
    out_dir = os.path.join(tempfile.gettempdir(), f"mrs_cpu_bench_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libcpu_decode_bench.so")
    subprocess.check_call(["gcc", "-O3", "-march=native", "-fPIC", "-shared", "-pthread", "-Wno-unused-function", "-I",
                           os.path.join(ROOT, "oracle"), "-o", so, src, "-lm"])
    # a short-lived child: the benchmark allocates the whole model (4.6 GB) and pins its threads
    code = (
        "import ctypes, json, sys\n"
        f"L = ctypes.CDLL({so!r}); L.mrs_cpu_decode_bench_samples.restype = ctypes.c_double\n"
        "a = json.loads(sys.argv[1])\n"
        "types = (ctypes.c_int * len(a['types']))(*a['types'])\n"
        "n = a['nsamples']\n"
        "ts, tk = (ctypes.c_double * n)(), (ctypes.c_int * n)()\n"
        "wb, tu = ctypes.c_double(), ctypes.c_int()\n"
        "r = L.mrs_cpu_decode_bench_samples(a['layers'], a['hidden'], a['inter'], a['heads'], a['kv_heads'], a['head_dim'], a['vocab'], types,\n"
        "                                   a['head_type'], a['ctx'], a['threads'], ctypes.c_double(a['seconds']), a['min_tokens'], n,\n"
        "                                   ts, tk, ctypes.byref(wb), ctypes.byref(tu))\n"
        "print(json.dumps({'tok_s': list(ts), 'tokens': list(tk), 'weight_bytes': wb.value, 'threads': tu.value}))\n")
    types = []
    for l in range(cfg.n_layers):
        types += [GGML[M.tensor_type(cfg, n, l)] for n in ("attn_q", "attn_k", "attn_v", "attn_output", "ffn_gate", "ffn_up", "ffn_down")]
    arg = dict(layers=cfg.n_layers, hidden=cfg.hidden, inter=cfg.inter, heads=cfg.n_heads, kv_heads=cfg.n_kv_heads,
               head_dim=cfg.head_dim, vocab=cfg.vocab, types=types, head_type=GGML[M.tensor_type(cfg, "output", 0)],
               ctx=PROMPT_LEN + GEN_LEN // 2, threads=threads, seconds=seconds, min_tokens=min_tokens, nsamples=nsamples)

    def run(a):
        return json.loads(subprocess.check_output([sys.executable, "-c", code, json.dumps(a)], text=True).strip().splitlines()[-1])
    if threads <= 0:
        # the container's CPU quota can be far below the number of CPUs in the affinity mask (128 visible, a
        # fraction schedulable): a pinned pool sized to the mask then crawls.  Probe a few pool sizes on a short
        # sample and keep the fastest — "all the host threads it can use".
        ncpu = len(os.sched_getaffinity(0))
        cands = sorted({max(1, ncpu >> s) for s in range(0, 5)} | ({_cgroup_cpus()} if _cgroup_cpus() else set()), reverse=True)
        cands = [c for c in cands if c <= ncpu]
        best = None
        for c in cands:
            pr = run(dict(arg, threads=c, seconds=min(1.5, seconds / 4), min_tokens=1, nsamples=1))
            if best is None or pr["tok_s"][0] > best[0]:
                best = (pr["tok_s"][0], c)
        arg["threads"] = best[1]
    r = run(arg)
    sample = (f"{r['tokens'][-1]} whole tokens (all {cfg.n_layers} layers + lm_head, {r['weight_bytes'] / 1e9:.2f} GB of weights streamed "
              f"from DRAM per token, attention over {arg['ctx']} cached tokens, norms and GLU included), decode batch 1, "
              f"-O3 -march=native, {r['threads']} pinned threads (pool size chosen by a short probe over {len(os.sched_getaffinity(0))} visible CPUs)")
    return r["tok_s"], r["threads"], sample


def cpu_decode_tokens_per_s(cfg, M, seconds=10.0, min_tokens=2, threads=0):
    vals, th, sample = cpu_decode_samples(cfg, M, seconds=seconds, min_tokens=min_tokens, threads=threads, nsamples=1)
    return vals[0], th, sample


def run_reference(args):
    """--impl reference: the reference's CPU implementation of the path (candle QMatMul cannot be built
    here: no Rust toolchain, candle un-vendored — the C restatement in oracle/, kind "port"), all host
    threads, same metric and workload; each step is one bounded sample of whole decode tokens."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import __graft_entry__ as g
    g.load_package()
    from mistralrs_b200 import model as M
    cfg = M.LlamaConfig.llama3_8b()
    if args.layers:
        cfg.n_layers = args.layers
    t0 = time.perf_counter()
    steps = max(1, args.steps)
    budget = args.cpu_seconds if args.cpu_seconds > 0 else max(4.0, min(20.0, 150.0 / (steps + max(args.warmup, 0))))
    # warm-up samples and timed samples share one model allocation and one pool-size probe: the run is
    # (warmup + steps) x budget seconds plus ~30 s of set-up, whatever --steps says
    nw = max(args.warmup, 0)
    allv, threads, sample = cpu_decode_samples(cfg, M, seconds=budget, nsamples=nw + steps)
    vals = allv[nw:]
    value = sum(vals) / len(vals)
    print(json.dumps({
        "impl": "reference", "metric": "decode_tok_s", "value": value, "unit": "tok/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 / value * (GEN_LEN - 1), "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "int8 (Q8_K / Q8_0) activations x ggml block dots, f32 accumulate", "data": "synthetic",
        "config": {"workload": "Llama-3-8B GGUF Q4_K_M decode batch=1 (CPU, whole tokens; each step a bounded sample)"},
        "cpu_baseline": {"value": value, "unit": "tok/s", "cores": threads, "kind": "port", "sample": sample},
        "e2e": {"value": value, "unit": "tok/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "wall_s": time.perf_counter() - t0}))


def run_config1(args):
    """BASELINE config 1: TinyLlama-1.1B GGUF Q4_K_M on the CPU, 128-token prompt + 64 decode tokens — plumbing
    only (no GPU): the CPU port of the reference's arithmetic through every layer (oracle/cpu_decode_bench.c),
    the prompt fed token by token like the decode steps."""
    if int(os.environ.get("RANK", "0")) != 0:
        return
    import __graft_entry__ as g
    g.load_package()
    from mistralrs_b200 import model as M
    cfg = M.LlamaConfig.tinyllama()
    t0 = time.perf_counter()
    v, threads, sample = cpu_decode_tokens_per_s(cfg, M, seconds=0.0, min_tokens=128 + 64)
    print(json.dumps({"metric": "decode_tok_s", "value": v, "unit": "tok/s", "n_gpus": 0, "steps": 1, "warmup": 1,
                      "ms_per_step": 1e3 * (128 + 64) / v, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
                      "dtype": "int8 (Q8_K / Q8_0) activations x ggml block dots, f32 accumulate", "data": "synthetic",
                      "config": {"workload": "TinyLlama-1.1B GGUF Q4_K_M on CPU, 128-token prompt + 64 decode tokens (192 token steps, plumbing)"},
                      "cpu_baseline": {"value": v, "unit": "tok/s", "cores": threads, "kind": "port", "sample": sample},
                      "e2e": {"value": v, "unit": "tok/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                      "gpu_launches": 0, "wall_s": time.perf_counter() - t0}))


# ------------------------------------------------------------------------------------------- helpers
def count_graph_kernels(graph):
    """kernel nodes of a captured CUDA graph (= our launches per replay), read back from the driver"""
    try:
        cu = ctypes.CDLL("libcuda.so.1")
        raw = ctypes.c_void_p(int(graph.raw_cuda_graph()))
        n = ctypes.c_size_t(0)
        if cu.cuGraphGetNodes(raw, None, ctypes.byref(n)) != 0:
            return None
        nodes = (ctypes.c_void_p * n.value)()
        if cu.cuGraphGetNodes(raw, nodes, ctypes.byref(n)) != 0:
            return None
        k = 0
        for i in range(n.value):
            ty = ctypes.c_int(-1)
            cu.cuGraphNodeGetType(ctypes.c_void_p(nodes[i]), ctypes.byref(ty))
            k += int(ty.value == 0)      # CU_GRAPH_NODE_TYPE_KERNEL
        return k
    except Exception:
        return None


def timed_graph(graph, reps, torch):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def validate_first_tokens(weights, M, torch, n_tokens=6):
    """The benchmarked 32-layer model against the CPU oracle (thread-pooled over rows): one prompt token,
    then greedy decoding; logits compared on every step, sampled ids must agree off ties."""
    import numpy as np
    from oracle.model import OracleLlama
    cfg = weights.cfg
    threads = max(1, min(32, len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 1))
    run = M.LlamaRunner(weights, batch=1, max_ctx=32, pdl=True)
    cos, sin = M.rope_tables(cfg)
    ref = OracleLlama(cfg, weights.host, M.tensor_type, cos, sin, "bf16", threads=threads)
    toks, worst, same = [prompt_tokens(0)[0]], 0.0, 0
    run.set_tokens(toks)
    t0 = time.perf_counter()
    for pos in range(n_tokens):
        run.step()
        torch.cuda.synchronize()
        got = run.logits().float().cpu().numpy()
        want = ref.step(toks, pos)
        scale = float(np.abs(want).max())
        if not (np.isfinite(want).all() and np.isfinite(got).all() and scale > 0):
            raise AssertionError("bench validation: non-finite or degenerate logits")
        worst = max(worst, float(np.abs(got - want).max()) / scale)
        top2 = np.sort(want[0])[-2:]
        tie = (top2[1] - top2[0]) <= 8 * 2.0 ** -8 * scale
        g_tok, w_tok = int(run.meta["token_ids"][0]), int(np.argmax(want[0]))
        if g_tok != w_tok and not tie:
            raise AssertionError(f"bench validation: sampled token {g_tok} != oracle {w_tok} at position {pos}")
        same += int(g_tok == w_tok)
        toks = [w_tok]
        run.set_tokens(toks)
    if not worst <= 4.1 * 2.0 ** -7:
        raise AssertionError(f"bench validation: logits differ from the oracle by {worst:.3e} of the logit scale")
    del run
    return {"tokens_checked": n_tokens, "tokens_equal": same, "worst_logit_err_ulp_bf16": worst / 2.0 ** -8,
            "oracle_threads": threads, "seconds": time.perf_counter() - t0,
            "what": f"all {cfg.n_layers} layers + lm_head of the benchmarked weights vs oracle/ (CPU), greedy from one prompt token"}


# ------------------------------------------------------------------------------------------- config 3
def bench_prefill_q8(M, torch, dev, peaks, prompt=4096, layers=0, steps=3, warmup=1, dump=None):
    """BASELINE config 3: Llama-3-8B with Q8_0 blocks everywhere (UQFF q8), one 4096-token prompt.
    TTFT = embedding -> 32 x (norm, wgmma dequant-GEMMs, RoPE, causal prompt attention, KV scatter, GLU) ->
    lm_head on the last row -> argmax; prefill tok/s = L / TTFT (bench.rs:269-271).  `steps` timed prompts (median),
    after `warmup` untimed ones; `dump` (a dict) receives the last timed prompt's logits and first token."""
    cfg = M.LlamaConfig.llama3_8b(quant="q8_0")
    if layers:
        cfg.n_layers = layers
    w = M.LlamaWeights(cfg, dev, fast_synth=True)
    pre = M.LlamaPrefill(w, max_tokens=prompt)
    for it in range(warmup):
        pre.forward(prompt_tokens(it, n=prompt))
    torch.cuda.synchronize()
    ts = []
    for it in range(steps):
        toks = prompt_tokens(warmup + it, n=prompt)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        logits = pre.forward(toks)
        first = torch.argmax(logits)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3)
    if dump is not None:
        import numpy as np
        dump["prefill_logits"] = logits.float().reshape(-1).cpu().numpy()
        dump["first_token"] = np.array([int(first)], dtype=np.float64)
    ttft = sorted(ts)[len(ts) // 2]
    # attention share, timed alone on the same shapes
    H, KVH, D = cfg.n_heads, cfg.n_kv_heads, cfg.head_dim
    from mistralrs_b200 import paged_attn
    q = torch.randn(prompt, H, D, device=dev).to(w.dtype)
    k = torch.randn(prompt, KVH, D, device=dev).to(w.dtype)
    v = torch.randn(prompt, KVH, D, device=dev).to(w.dtype)
    paged_attn.prefill_attention(q, k, v, D ** -0.5)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(cfg.n_layers):
        paged_attn.prefill_attention(q, k, v, D ** -0.5)
    e1.record()
    torch.cuda.synchronize()
    attn_s = e0.elapsed_time(e1) / 1e3
    lin_params = cfg.n_layers * (2 * cfg.hidden * H * D + 2 * cfg.hidden * KVH * D + 3 * cfg.hidden * cfg.inter)
    flop = 2.0 * prompt * lin_params + cfg.n_layers * 2.0 * prompt * prompt * H * D + 2.0 * cfg.vocab * cfg.hidden
    attn_flop = cfg.n_layers * 2.0 * prompt * prompt * H * D
    tpeak = peaks.get("bf16_tflops_sustained", 989.0)
    out = {"workload": "Llama-3-8B Q8_0 (UQFF q8) prefill, 1 x %d tokens, incl. prompt attention, lm_head on the last row" % prompt,
           "prompt_tokens": prompt, "layers": cfg.n_layers, "steps": steps, "warmup": warmup, "ttft_ms": ttft * 1e3, "prefill_tok_s": prompt / ttft,
           "tflops": flop / ttft / 1e12, "tensor_peak_tflops": tpeak, "tensor_frac": flop / ttft / 1e12 / tpeak,
           "attention_ms": attn_s * 1e3, "attention_tflops": attn_flop / attn_s / 1e12,
           "linears_ms_est": (ttft - attn_s) * 1e3, "linears_tflops_est": 2.0 * prompt * lin_params / max(ttft - attn_s, 1e-9) / 1e12,
           "weights": "synthetic Q8_0 blocks generated on the device", "first_token": int(first)}
    del pre, w
    torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------------------------------- config 4
def bench_gptq_batch32(torch, dev, peaks, steps=2, layers=0, batch=32, warmup=1, dump=None):
    """BASELINE config 4: Mistral-7B GPTQ int4 (g128, symmetric) decode at batch 32, paged KV block 16,
    128-token prompts -> +256 tokens, in the HND (FlashInfer) and vLLM cache layouts; `steps` timed generations per
    layout after `warmup` untimed ones.  `dump` (a dict) receives the last timed HND generation's final token ids and
    logits."""
    from mistralrs_b200 import gptq_model as G
    cfg = G.GptqConfig.mistral_7b()
    if layers:
        cfg.n_layers = layers
    w = G.GptqWeights(cfg, dev)
    peak = peaks.get("hbm_gbs", 3350.0)
    kv_mean = batch * 2 * cfg.n_kv_heads * cfg.head_dim * 2 * cfg.n_layers * (PROMPT_LEN + GEN_LEN // 2)
    res = {"workload": f"Mistral-7B GPTQ int4 g128 decode batch={batch}, 128-token prompts -> +256 tokens, paged KV block_size=16",
           "layers": cfg.n_layers, "steps": steps, "warmup": warmup, "weight_bytes_per_step": w.nbytes, "kv_bytes_per_step_mean": kv_mean}
    for layout in ("hnd", "vllm"):
        run = G.GptqRunner(w, batch=batch, max_ctx=PROMPT_LEN + GEN_LEN + 16, cache_layout=layout)
        graph = run.capture()
        vals = []
        for it in range(warmup + steps):
            run.reset()
            ptoks = [prompt_tokens(it, case=b) for b in range(batch)]
            for i in range(PROMPT_LEN):
                run.set_tokens([p[i] for p in ptoks])
                graph.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(GEN_LEN - 1):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            if it >= warmup:
                vals.append(e0.elapsed_time(e1) / 1e3)
        if dump is not None and layout == "hnd":
            import numpy as np
            dump["token_ids"] = run.meta["token_ids"].cpu().numpy().astype(np.float64)
            dump["last_logits"] = run.logits().float().reshape(-1).cpu().numpy()
        sec = sum(vals) / len(vals)
        step_s = sec / (GEN_LEN - 1)
        res[layout] = {"decode_tok_s": batch * (GEN_LEN - 1) / sec, "ms_per_decode_step": step_s * 1e3,
                       "hbm_frac": (w.nbytes + kv_mean) / step_s / 1e9 / peak, "launches_per_step": count_graph_kernels(graph)}
        # the W4A16 + dense linears alone (attention-side kernels skipped): roofline of the dominant kernel
        if layout == "hnd":
            run.step_struct.skip_mask = 1
            gg = torch.cuda.CUDAGraph()
            run.reset(PROMPT_LEN + GEN_LEN // 2); run.step(); torch.cuda.synchronize()
            with torch.cuda.graph(gg):
                run.step()
            lin_s = timed_graph(gg, 10, torch)
            run.step_struct.skip_mask = 0
            res["linears"] = {"ms_per_step": lin_s * 1e3, "achieved_gbs": w.nbytes / lin_s / 1e9, "hbm_frac": w.nbytes / lin_s / 1e9 / peak,
                              "kernel": "hg_kernel<Int4TileSrc, 32> (swap-AB wgmma) + dense lm_head"}
        del run, graph
    del w
    torch.cuda.empty_cache()
    return res


# ------------------------------------------------------------------------------------------- main
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", type=int, default=2, choices=[1, 2, 3, 4, 5],
                    help="headline workload: 1 = TinyLlama-1.1B Q4_K_M on the CPU (plumbing, no GPU), 2 = 8B Q4_K_M decode b=1 (default), "
                         "3 = 8B Q8_0 prefill 4096, 4 = Mistral-7B GPTQ b=32, 5 = Llama-3-70B Q4_K_M tensor parallel (needs --gpus 8)")
    ap.add_argument("--layers", type=int, default=0, help="debug: truncate the model")
    ap.add_argument("--pdl", type=int, default=int(os.environ.get("MRS_PDL", "1")))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip the config 3 / config 4 blocks of the default line")
    ap.add_argument("--no-validate", action="store_true")
    ap.add_argument("--cpu-seconds", type=float, default=0.0, help="bound of one CPU sample (tests); 0: derived from --steps")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write what the last timed step computed (generated token ids, last logits, "
                         "prompt logits) as DIR/<name>.npy in float32 / float64")
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be at least 1 and --warmup at least 0")
    if args.impl == "reference":
        return run_reference(args)
    if args.config == 1:
        return run_config1(args)

    import numpy as np
    import torch
    import torch.distributed as dist
    import __graft_entry__ as g
    g.load_package()
    from mistralrs_b200 import lib, model as M

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    lib()  # fail loudly if the CUDA extension is missing
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak, peak_src = (peaks["hbm_gbs"], "measured") if "hbm_gbs" in peaks else (3350.0, "fallback: H100 SXM data sheet")

    def write_dump(dump):
        if args.dump_outputs and rank == 0:
            os.makedirs(args.dump_outputs, exist_ok=True)
            for name, a in dump.items():
                np.save(os.path.join(args.dump_outputs, f"{name}.npy"), a)

    if args.config == 3 and world == 1:
        dump = {}
        pf = bench_prefill_q8(M, torch, dev, peaks, layers=args.layers, steps=args.steps, warmup=args.warmup, dump=dump)
        write_dump(dump)
        print(json.dumps({"metric": "prefill_tok_s", "value": pf["prefill_tok_s"], "unit": "tok/s", "n_gpus": 1, "steps": args.steps,
                          "warmup": args.warmup,
                          "ms_per_step": pf["ttft_ms"], "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
                          "dtype": "bf16 activations x Q8_0 blocks dequantised to bf16 (wgmma), f32 accumulate", "data": "synthetic",
                          "config": {"workload": pf["workload"]}, "prefill": pf,
                          "roofline": {"bound": "tensor", "achieved": pf["tflops"], "peak": pf["tensor_peak_tflops"], "unit": "TFLOP/s",
                                       "frac": pf["tensor_frac"], "traffic": None}}))
        return
    if args.config == 4 and world == 1:
        dump = {}
        c4 = bench_gptq_batch32(torch, dev, peaks, steps=args.steps, layers=args.layers, warmup=args.warmup, dump=dump)
        write_dump(dump)
        print(json.dumps({"metric": "decode_tok_s", "value": c4["hnd"]["decode_tok_s"], "unit": "tok/s", "n_gpus": 1, "steps": args.steps,
                          "warmup": args.warmup, "ms_per_step": c4["hnd"]["ms_per_decode_step"] * (GEN_LEN - 1), "higher_is_better": True,
                          "scaling": "strong", "vs_baseline": None, "dtype": "f16 activations x int4 (q-8)*s dequantised to f16 (wgmma), f32 accumulate",
                          "data": "synthetic", "config": {"workload": c4["workload"]}, "config4": c4,
                          "roofline": {"bound": "hbm", "achieved": c4["linears"]["achieved_gbs"], "peak": peak, "unit": "GB/s",
                                       "frac": c4["linears"]["hbm_frac"], "traffic": None, "peak_source": peak_src}}))
        return

    # ---------------------------------------------------------------- configs 2 / 5: decode batch 1 (TP = world)
    big = args.config == 5
    cfg = M.LlamaConfig.llama3_70b() if big else M.LlamaConfig.llama3_8b()
    if args.layers:
        cfg.n_layers = args.layers
    validate = (not args.no_validate) and world == 1 and not big
    weights = M.LlamaWeights(cfg, dev, tp_rank=rank, tp_size=world, keep_host=validate, fast_synth=big)
    peer, comm, bufs = None, None, {}
    def nccl_comm(buf, count, dtype, stream, user):                   # A/B and last resort: NCCL through torch.distributed
        dist.all_reduce(bufs[buf])
    if world > 1 and os.environ.get("MRS_TP_NCCL", "0") != "1":
        try:
            peer = M.PeerAllReduce(cfg.hidden, weights.dtype, dev)   # in-graph peer-memory sum (product path)
        except Exception as e:                                        # no symmetric memory on this box: keep the run alive
            print(f"[bench] rank {rank}: peer-memory all-reduce unavailable ({e!r}); using NCCL", file=sys.stderr, flush=True)
        ok = torch.tensor([1 if peer is not None else 0], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)                     # every rank must take the same path
        if int(ok.item()) == 0:
            peer = None
    if world > 1 and peer is None:
        comm = nccl_comm

    def make_runner():
        r = M.LlamaRunner(weights, batch=1, max_ctx=PROMPT_LEN + GEN_LEN + 16, pdl=bool(args.pdl), comm=comm, peer_allreduce=peer)
        if comm is not None:
            bufs[r.buf["x"].data_ptr()] = r.buf["x"]
            bufs[r.buf["x2"].data_ptr()] = r.buf["x2"]
        return r
    runner = make_runner()
    if peer is not None and peer.low_latency:
        # the low-latency protocol polls for its peers' words with a time-out: make sure a few eager steps go through on
        # every rank before anything is captured or timed; otherwise fall back to the flags + pull protocol
        for _ in range(2):
            runner.step()
        torch.cuda.synchronize()
        bad = torch.tensor([1 if peer.timed_out() else 0], device=dev)
        dist.all_reduce(bad, op=dist.ReduceOp.MAX)
        if int(bad.item()) != 0:
            print(f"[bench] rank {rank}: low-latency all-reduce timed out; falling back to flags + pull", file=sys.stderr, flush=True)
            dist.barrier()
            peer = M.PeerAllReduce(cfg.hidden, weights.dtype, dev, low_latency=False)
            runner = make_runner()
        else:
            runner.reset()
    validation = validate_first_tokens(weights, M, torch) if validate else None
    weights.host = None
    runner.capture()
    graph = runner.graph
    launches_per_token = count_graph_kernels(graph)
    tok_dev = runner.meta["token_ids"]
    pinned_in = torch.zeros(1, dtype=torch.int32).pin_memory()
    pinned_out = torch.zeros(1, dtype=torch.int32).pin_memory()
    prefill_runner = M.LlamaPrefill(weights, max_tokens=PROMPT_LEN, runner=runner) if world == 1 else None

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    ttfts = []
    dump = {}   # the last timed step's outputs (--dump-outputs)

    def generation(it, e2e, out=None, record=False):
        """one step: the prompt (one prefill pass on a single GPU; token by token through the decode graph
        under TP), then GEN_LEN tokens.  Returns device-timed seconds of the decode phase.  `out` (a dict) receives the
        prompt logits and the last logits, read after the timed windows; `record` also collects every generated token
        id, one device copy per token — only for an untimed step."""
        gen_ids = torch.zeros(GEN_LEN, dtype=torch.int32, device=dev) if record else None
        runner.reset()
        toks = prompt_tokens(it)
        if prefill_runner is not None:
            if e2e:
                hp = torch.tensor(toks, dtype=torch.int32).pin_memory()   # prompt ids cross PCIe inside the timed TTFT
            p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            p0.record()
            logits = prefill_runner.forward(hp if e2e else toks)
            tok_dev.copy_(torch.argmax(logits).to(torch.int32).reshape(1))
            runner.reset(PROMPT_LEN)
            p1.record()
            if out is not None:   # (after p1: outside the timed prompt window)
                out["prompt_logits"] = logits.float().reshape(-1).cpu().numpy()
        else:
            for t in toks:
                pinned_in[0] = t
                tok_dev.copy_(pinned_in, non_blocking=True)
                graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        if prefill_runner is not None:
            ttfts.append(p0.elapsed_time(p1) / 1e3)
        if record:
            gen_ids[0].copy_(tok_dev[0])
        e0.record()
        if not e2e:
            for i in range(GEN_LEN - 1):
                graph.replay()
                if record:
                    gen_ids[i + 1].copy_(tok_dev[0])
        else:
            pinned_in.copy_(tok_dev)
            for _ in range(GEN_LEN - 1):
                tok_dev.copy_(pinned_in, non_blocking=True)      # H2D: this step's input token
                graph.replay()
                pinned_out.copy_(tok_dev, non_blocking=True)     # D2H: the sampled token
                torch.cuda.current_stream().synchronize()
                pinned_in[0] = pinned_out[0]
        e1.record()
        barrier()
        if out is not None:
            out["last_logits"] = runner.logits().float().reshape(-1).cpu().numpy()
        if record:
            out["token_ids"] = gen_ids.cpu().numpy().astype(np.float64)
        return e0.elapsed_time(e1) / 1e3

    def max_over_ranks(x):
        if world == 1:
            return x
        t = torch.tensor([x], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0])

    for w_ in range(args.warmup):
        generation(w_, False)
    ttfts.clear()

    def timed_steps():
        sampler = ClockSampler(local)
        if rank == 0:
            sampler.start()
        ts = [max_over_ranks(generation(args.warmup + i, False, out=dump if args.dump_outputs and i == args.steps - 1 else None))
              for i in range(args.steps)]
        return ts, (sampler.stop() if rank == 0 else None)

    times, clocks = timed_steps()
    bad = {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    redo = torch.tensor([1 if (rank == 0 and bad & set(clocks.get("reasons", []))) else 0], device=dev)
    if world > 1:
        dist.broadcast(redo, src=0)
    if bool(redo.item()):
        first = clocks
        ttfts.clear()
        times, clocks = timed_steps()
        if rank == 0:
            clocks["remeasured_after"] = first.get("reasons", [])
    ttft_dev = sorted(ttfts)[len(ttfts) // 2] if ttfts else None
    if args.dump_outputs:
        # the generated ids: the same step again, untimed, collecting each token; the step is deterministic, and its
        # logits must equal the timed step's bit for bit, so these are the ids the timed step produced
        again = {}
        generation(args.warmup + args.steps - 1, False, out=again, record=True)
        for name in ("prompt_logits", "last_logits"):
            if name in dump and not np.array_equal(dump[name], again[name]):
                raise AssertionError(f"--dump-outputs: the untimed repeat of the last timed step differs in {name}")
        dump["token_ids"] = again["token_ids"]
        write_dump(dump)
    ttfts.clear()
    e2e_times = [max_over_ranks(generation(args.warmup + i, True)) for i in range(max(1, min(args.steps, 2)))]
    ttft_e2e = sorted(ttfts)[len(ttfts) // 2] if ttfts else None
    ntok = GEN_LEN - 1
    value = ntok * len(times) / sum(times)
    e2e_value = ntok * len(e2e_times) / sum(e2e_times)

    # ---- roofline of the dominant kernel (mmvq_stream_kernel: every quantized GEMV of a token), measured live:
    # a CUDA graph of ONE token's GEMV chain only (attention-side kernels skipped), CUDA events on the launching
    # stream; weights (4.6 GB) >> L2 so every launch streams from HBM.  Under TP the chain includes the all-reduces.
    runner.step_struct.skip_mask = 1
    gg = torch.cuda.CUDAGraph(keep_graph=True)
    runner.reset(PROMPT_LEN + GEN_LEN // 2)
    runner.forward(); torch.cuda.synchronize()
    with torch.cuda.graph(gg):
        runner.forward()
    barrier()
    gemv_s = max_over_ranks(timed_graph(gg, 20, torch))
    runner.step_struct.skip_mask = 2
    ga = torch.cuda.CUDAGraph()
    runner.forward(); torch.cuda.synchronize()
    with torch.cuda.graph(ga):
        runner.forward()
    barrier()
    attn_s = max_over_ranks(timed_graph(ga, 20, torch))
    runner.step_struct.skip_mask = 0
    total_bytes, weight_bytes = algorithmic_bytes_per_token(cfg, M, world)
    if world > 1:   # replicated lm_head: every rank streams all of it
        t = M.tensor_type(cfg, "output", 0)
        from mistralrs_b200 import BLOCK_BYTES, BLOCK_ELEMS
        head = cfg.vocab * cfg.hidden * BLOCK_BYTES[t] // BLOCK_ELEMS[t]
        weight_bytes = (weight_bytes - head) + head   # algorithmic_bytes_per_token already keeps the head whole per rank
    n_gemv = sum(4 if M.tensor_type(cfg, "attn_v", l) == M.tensor_type(cfg, "attn_q", l) else 5 for l in range(cfg.n_layers)) + 1
    achieved = weight_bytes / gemv_s / 1e9
    traffic = None

    # ---- GPU reference arm: the unmodified reference kernels (oracle/_ref) chained as mistral.rs chains them, one
    # CUDA graph per token, same weights, same box (scripts/gpu_reference_chain.py)
    gpu_ref = None
    if world == 1 and not big and not args.no_extras:
        try:
            sys.path.insert(0, os.path.join(ROOT, "scripts"))
            from gpu_reference_chain import RefChain
            rc_ = RefChain(weights, M, batch=1, max_ctx=PROMPT_LEN + GEN_LEN + 16)
            rg = rc_.capture()
            rc_.run.reset(PROMPT_LEN)
            for _ in range(5):
                rg.replay()
            rc_.run.reset(PROMPT_LEN)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(GEN_LEN - 1):
                rg.replay()
            e1.record()
            torch.cuda.synchronize()
            sec = e0.elapsed_time(e1) / 1e3
            gpu_ref = {"decode_tok_s": (GEN_LEN - 1) / sec, "launches_per_token": count_graph_kernels(rg),
                       "what": "unmodified reference kernels (mmvq_gguf, rotary, add_rms_norm, reshape_and_cache_flashinfer, flashinfer_decode; "
                               "built from the reference sources with its own flags) chained per layer as mistral.rs does, CUDA graph per token, "
                               "reference split-KV policy; same synthetic weights, same decode window"}
            del rc_, rg
        except Exception as e:
            gpu_ref = {"unavailable": repr(e)}

    prefill = c4 = None
    if world == 1 and not args.no_extras and not big and not args.layers:
        del prefill_runner
        try:
            prefill = bench_prefill_q8(M, torch, dev, peaks)
        except Exception as e:   # the extras must never take the headline line down
            prefill = {"error": repr(e)}
        try:
            c4 = bench_gptq_batch32(torch, dev, peaks, steps=1)
        except Exception as e:
            c4 = {"error": repr(e)}

    if rank == 0:
        cpu = None
        if not args.no_cpu_baseline and world == 1 and not big:
            try:
                v, threads, sample = cpu_decode_tokens_per_s(cfg, M, seconds=12.0)
                cpu = {"value": v, "unit": "tok/s", "cores": threads, "kind": "port", "sample": sample}
            except Exception as e:
                cpu = {"value": None, "unit": "tok/s", "cores": 0, "kind": "port", "sample": f"failed: {e!r}"}
        name = "Llama-3-70B" if big else "Llama-3-8B"
        out = {
            "metric": "decode_tok_s", "value": value, "unit": "tok/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": 1e3 * sum(times) / len(times), "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "int8 activations x 4/6-bit ggml blocks (dp4a), f32 accumulate, bf16 I/O",
            "data": "synthetic",
            "config": {"workload": f"{name} GGUF Q4_K_M decode batch=1, 128-token prompt -> +256 tokens, paged KV block_size=16 (HND)",
                       "parallelism": f"tp{world}", "l2": "inputs larger than L2 (weights streamed once per token)",
                       "layers": cfg.n_layers, "pdl": bool(args.pdl),
                       "all_reduce": None if world == 1 else (("peer-memory one-shot sum + residual, in-graph (mrs_tp_allreduce_residual; " + ("low-latency push of {data, sequence} words" if peer.low_latency else "flags + pull") + ")") if peer is not None else "NCCL via torch.distributed, captured"),
                       "kv_split": f"{runner.split_pages * cfg.block_size}-token chunks, {runner.padded_tiles} tiles (SM-filling plan)"},
            "e2e": {"value": e2e_value, "unit": "tok/s", "h2d_bytes_per_step": 4 * ntok + 4 * PROMPT_LEN, "d2h_bytes_per_step": 4 * ntok,
                    "ttft_ms": None if ttft_e2e is None else ttft_e2e * 1e3},
            "gpu_launches": None if launches_per_token is None else launches_per_token * ntok,
            "launches_per_token": launches_per_token,
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "traffic": traffic, "algorithmic_bytes_per_launch": weight_bytes / n_gemv, "peak_source": peak_src,
                         "kernel": "mmvq_stream_kernel (all quantized GEMVs of one token" + (", incl. the in-graph all-reduces)" if world > 1 else ")"),
                         "launches": n_gemv, "avg_launch_us": gemv_s / n_gemv * 1e6, "bytes_per_token": weight_bytes},
            "breakdown_us_per_token": {"gemv_chain": gemv_s * 1e6, "attention_chain": attn_s * 1e6, "whole_token": 1e6 / value},
            "step_hbm_frac": total_bytes * value / 1e9 / peak,
            "clocks": clocks,
        }
        if ttft_dev is not None:
            out["prompt"] = {"tokens": PROMPT_LEN, "ttft_ms": ttft_dev * 1e3, "prefill_tok_s": PROMPT_LEN / ttft_dev,
                             "note": "the 128-token prompt of this workload: one prefill pass (wgmma dequant-GEMMs + prompt attention + KV scatter) + first sample"}
        if gpu_ref:
            out["gpu_reference"] = gpu_ref
            if "decode_tok_s" in gpu_ref:
                out["gpu_reference"]["ours_over_reference_kernels"] = value / gpu_ref["decode_tok_s"]
        if validation:
            out["validation"] = validation
        if cpu:
            out["cpu_baseline"] = cpu
        if prefill:
            out["prefill"] = prefill
        if c4:
            out["config4"] = c4
        print(json.dumps(out))
    if world > 1:
        # NCCL teardown with captured collectives still alive can hang: synchronise and leave
        dist.barrier()
        torch.cuda.synchronize()
        sys.stdout.flush()
        os._exit(0)


if __name__ == "__main__":
    main()
