"""Where the batch-1 GEMV chain of one decode token spends its time, by launch role.

Builds the `-DMRS_TIMELINE` variant of mmvq.cu into a temporary directory (linked with the in-tree objects of the
other sources, which `build()` leaves in csrc/), captures one decode token of the config-2 model (Llama-3-8B,
Q4_K_M, batch 1, PDL on) with every GEMV launch stamping %globaltimer per CTA, and reports per role
(q∥k∥v; q∥k + v as one grid where attn_v is Q6_K; o_proj, gate∥up, down, lm_head) in µs per token:

  ideal    the role's weight bytes at the stream rate that shape reaches alone on this card: a CUDA graph of
           back-to-back launches of the shape rotating over enough distinct weight copies to exceed 2 x L2
  span     sum over the role's launches of (its last CTA exit - the previous launch's last CTA exit)
  entry_wait  median over CTAs of (PDL release - CTA entry)
  prologue    median over CTAs of (activation image ready - PDL release)
  first_seg   median over CTAs of (first full ring segment - activation image ready)
  consume     median over CTAs of (end of the dot loop - first full segment)
  tail        last CTA exit - median loop end

plus, per launch, the gap from the previous launch's last exit to this launch's first CTA entry and the medians and
maxima of every stamp.  Prints the card, its power limit and the median SM clock, and writes everything to
OUT/gemv_chain.json.

  python scripts/bench_gemv_chain.py [--out DIR] [--reps N] [--lib PATH]
"""
import argparse
import ctypes
import glob
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

CSRC = os.path.join(ROOT, "mistral.rs_b200", "csrc")
STAMPS = ["entry", "init", "issue1", "waited", "pass0", "pass1", "pass2", "full0", "loopend", "exit", "prodend"]
SLOTS = 320  # CTA records per launch in the timeline buffer (mmvq.cu)
GGML = {"q4_k": 12, "q6_k": 14}
DT_BF16 = 1


def build_timeline_lib(tmp):
    objs = [o for o in sorted(glob.glob(os.path.join(CSRC, "*.o"))) if os.path.basename(o) != "mmvq.o"]
    if not objs:
        raise RuntimeError("no in-tree objects under csrc/: run build() first")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    obj = os.path.join(tmp, "mmvq_timeline.o")
    subprocess.check_call([nvcc, "-std=c++17", "-O3", *arch, "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
                           "-DMRS_TIMELINE", "-I" + os.path.join(ROOT, "include"), "-c", os.path.join(CSRC, "mmvq.cu"),
                           "-o", obj])
    so = os.path.join(tmp, "libmrs_b200_timeline.so")
    subprocess.check_call([nvcc, *arch, "-shared", "-o", so, obj, *objs, "-lcudart"])
    return so


def gpu_facts():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                                      text=True).strip().splitlines()[0]
        name, pl, mx = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_max_mhz": float(mx)}
    except Exception as e:
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None, "error": repr(e)}


def chain_plan(cfg, M, one_grid_v=True):
    """The GEMV launches of one token in issue order: (role, ggml type, K, virtual rows, weight bytes, layer).
    Where attn_v has its own type, q∥k and v are one grid (role qk_v, the rows of its first program) or, with
    one_grid_v False, two launches (as the decoder issued them before it used mrs_mmvq_fused_qkv_mixed)."""
    from mistralrs_b200 import BLOCK_BYTES, BLOCK_ELEMS
    H, I = cfg.hidden, cfg.inter
    nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
    nbytes = lambda t, rows, k: rows * k * BLOCK_BYTES[t] // BLOCK_ELEMS[t]
    plan = []
    for l in range(cfg.n_layers):
        tq, tv = M.tensor_type(cfg, "attn_q", l), M.tensor_type(cfg, "attn_v", l)
        if tq == tv:
            plan.append(("qkv", tq, H, nq + 2 * nkv, nbytes(tq, nq + 2 * nkv, H), l))
        elif one_grid_v:
            plan.append(("qk_v", tq, H, nq + nkv, nbytes(tq, nq + nkv, H) + nbytes(tv, nkv, H), l))
        else:
            plan.append(("qk", tq, H, nq + nkv, nbytes(tq, nq + nkv, H), l))
            plan.append(("v", tv, H, nkv, nbytes(tv, nkv, H), l))
        to = M.tensor_type(cfg, "attn_output", l)
        plan.append(("o_proj", to, nq, H, nbytes(to, H, nq), l))
        tg = M.tensor_type(cfg, "ffn_gate", l)
        plan.append(("gate_up", tg, H, I, nbytes(tg, 2 * I, H), l))
        td = M.tensor_type(cfg, "ffn_down", l)
        plan.append(("down", td, I, H, nbytes(td, H, I), l))
    th = M.tensor_type(cfg, "output", 0)
    plan.append(("lm_head", th, H, cfg.vocab, nbytes(th, cfg.vocab, H), -1))
    return plan


class ShapeCall:
    """The decoder's mrs_mmvq_fused call for one launch role (PDL on), on weights chosen by the caller."""

    def __init__(self, lib, weights, cfg, dev):
        H, I = cfg.hidden, cfg.inter
        nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
        a = lambda n: (torch.randn(n, device=dev) * 0.5).to(torch.bfloat16)
        self.lib, self.dims, self.vocab = lib, (H, I, nq, nkv), cfg.vocab
        self.norm = weights.layers[0]["attn_norm"]
        self.b = {"x": a(H), "attn": a(nq), "act": a(I), "q": a(nq), "k": a(nkv), "v": a(nkv), "y": a(H),
                  "res": a(H), "logits": a(cfg.vocab)}

    def __call__(self, role, t, mats, stream):
        """mats: the role's weights as LlamaWeights holds them, (blocks, ggml type, rows, cols) each"""
        H, I, nq, nkv = self.dims
        b, nw = self.b, self.norm
        w = [m[0] for m in mats] + [None] * (3 - len(mats))
        ptr = lambda d: ctypes.c_void_p(d.data_ptr() if d is not None else 0)
        if role == "qk_v":
            rc = self.lib.mrs_mmvq_fused_qkv_mixed(ctypes.c_int(GGML[mats[0][1]]), ctypes.c_int(GGML[mats[2][1]]),
                                                   ctypes.c_int(DT_BF16), *[ptr(m) for m in w], ptr(b["x"]), ptr(nw),
                                                   ctypes.c_float(1e-5), ptr(b["q"]), ptr(b["k"]), ptr(b["v"]),
                                                   ctypes.c_int(H), ctypes.c_int(nq), ctypes.c_int(nkv), ctypes.c_int(nkv),
                                                   ctypes.c_int(1), ctypes.c_int(1), stream)
            if rc != 0:
                raise RuntimeError(f"mrs_mmvq_fused_qkv_mixed -> cudaError {rc}")
            return
        mode, x, norm, res, dst, K, n = {
            "qkv": (2, b["x"], nw, None, (b["q"], b["k"], b["v"]), H, (nq, nkv, nkv)),
            "qk": (2, b["x"], nw, None, (b["q"], b["k"], None), H, (nq, nkv, 0)),
            "v": (0, b["x"], nw, None, (b["v"], None, None), H, (nkv, 0, 0)),
            "o_proj": (0, b["attn"], None, b["res"], (b["y"], None, None), nq, (H, 0, 0)),
            # as the decoder chains them: gate∥up writes act in block_q8_1 form, down reads it
            "gate_up": (1 | 8, b["x"], nw, None, (b["act"], None, None), H, (I, I, 0)),
            "down": (4, b["act"], None, b["res"], (b["y"], None, None), I, (H, 0, 0)),
            "lm_head": (0, b["x"], nw, None, (b["logits"], None, None), H, (self.vocab, 0, 0)),
        }[role]
        rc = self.lib.mrs_mmvq_fused(ctypes.c_int(GGML[t]), ctypes.c_int(mode), ctypes.c_int(DT_BF16),
                                     *[ptr(m) for m in w], ptr(x), ptr(norm), ctypes.c_float(1e-5), ptr(res),
                                     *[ptr(d) for d in dst], ctypes.c_int(K), *[ctypes.c_int(v) for v in n],
                                     ctypes.c_int(1), ctypes.c_int(0), ctypes.c_int(1), stream)
        if rc != 0:
            raise RuntimeError(f"mrs_mmvq_fused({role}) -> cudaError {rc}")


def stream_rates(weights, cfg, M, lib, dev, plan):
    """GB/s each (role, type) shape reaches alone: a graph of back-to-back PDL launches rotating over distinct weights
    (the model's own layers of that shape, plus copies until they exceed 2 x L2)."""
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size
    names = {"qkv": ("attn_q", "attn_k", "attn_v"), "qk_v": ("attn_q", "attn_k", "attn_v"), "qk": ("attn_q", "attn_k"),
             "v": ("attn_v",),
             "o_proj": ("attn_output",), "gate_up": ("ffn_gate", "ffn_up"), "down": ("ffn_down",)}
    sr = ShapeCall(lib, weights, cfg, dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    out = {}
    for role, t in sorted({(r, t) for r, t, *_ in plan}):
        if role == "lm_head":
            sets = [(weights.output,)]
        else:
            sets = [tuple(weights.layers[l][n] for n in names[role]) for r, tt, _, _, _, l in plan if r == role and tt == t]
        nbytes = next(b for r, tt, _, _, b, _ in plan if r == role and tt == t)
        extra = []
        while nbytes * (len(sets) + len(extra)) < 2 * l2:
            src = sets[len(extra) % len(sets)]
            extra.append(tuple((m[0].clone(), *m[1:]) for m in src))
        sets = sets + extra
        launches = max(len(sets), 32)
        for _ in range(2):                              # module load, attributes
            sr(role, t, sets[0], stream)
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            for i in range(launches):
                sr(role, t, sets[i % len(sets)], stream)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        for _ in range(3):
            gr.replay()
        torch.cuda.synchronize()
        ts = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            gr.replay()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 1e3)
        sec = float(np.median(ts))
        out[f"{role}/{t}"] = {"gbs": nbytes * launches / sec / 1e9, "us_per_launch": sec / launches * 1e6,
                              "bytes": nbytes, "distinct_copies": len(sets)}
        del gr, extra, sets
        torch.cuda.empty_cache()
    return out


PHASES = ("ideal", "span", "gap", "entry_wait", "prologue", "first_seg", "consume", "tail")


def attribute(plan, tokens, rates):
    """Per-launch phases (µs) from the stamps of each recorded token ([launch][CTA][16] globaltimer ns; slot 15 of CTA 0
    holds the grid, slot 14 vrows << 32 | K), medians over tokens, then summed per role and over the whole chain."""
    per_launch = []
    for i, (role, t, K, vrows, nbytes, layer) in enumerate(plan):
        rec = {"role": role, "type": t, "K": K, "vrows": vrows, "bytes": nbytes, "layer": layer}
        vals = {k: [] for k in PHASES[1:] + ("grid",)}
        med_stamps, max_stamps = [], []
        for tok in tokens:
            grid = int(tok[i, 0, 15])
            kv = int(tok[i, 0, 14])
            if grid == 0 or (kv & 0xffffffff) != K or (kv >> 32) != vrows:
                raise RuntimeError(f"launch {i}: stamps say grid {grid} K {kv & 0xffffffff} vrows {kv >> 32}, plan {role} K {K} vrows {vrows}")
            a = tok[i, :grid, :11].astype(np.float64) / 1e3       # µs
            t0 = a[:, 0].min()
            prev_exit = tok[i - 1, :int(tok[i - 1, 0, 15]), 9].max() / 1e3 if i > 0 else np.nan
            exit_max = a[:, 9].max()
            med_stamps.append(np.median(a - t0, axis=0)); max_stamps.append((a - t0).max(axis=0))
            vals["grid"].append(grid)
            vals["gap"].append(t0 - prev_exit)
            vals["span"].append(exit_max - prev_exit)
            vals["entry_wait"].append(np.median(a[:, 3] - a[:, 0]))
            vals["prologue"].append(np.median(a[:, 6] - a[:, 3]))
            vals["first_seg"].append(np.median(a[:, 7] - a[:, 6]))
            vals["consume"].append(np.median(a[:, 8] - a[:, 7]))
            vals["tail"].append(exit_max - np.median(a[:, 8]))
        for k, v in vals.items():
            rec[k] = float(np.median(v))
        rec["stamp_median_us"] = dict(zip(STAMPS, np.median(med_stamps, axis=0).round(3).tolist()))
        rec["stamp_max_us"] = dict(zip(STAMPS, np.median(max_stamps, axis=0).round(3).tolist()))
        rate = rates[f"{role}/{t}"]["gbs"]
        rec["ideal"] = nbytes / rate / 1e3
        per_launch.append(rec)

    roles = {}
    for rec in per_launch:
        r = roles.setdefault(rec["role"], {"launches": 0, "bytes": 0, **{k: 0.0 for k in PHASES}})
        r["launches"] += 1
        r["bytes"] += rec["bytes"]
        for k in PHASES:
            if not np.isnan(rec[k]):
                r[k] += rec[k]
    total = {k: sum(r[k] for r in roles.values()) for k in ("launches", "bytes") + PHASES}
    return per_launch, roles, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gemv_chain_out")
    ap.add_argument("--reps", type=int, default=5, help="recorded tokens (the medians are over tokens too)")
    ap.add_argument("--lib", default=None, help="an already built -DMRS_TIMELINE library (else built into a temp dir)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gemv_chain needs a GPU"
    facts = gpu_facts()
    pkg = g.load_package()
    pkg.LIB_PATH = args.lib or build_timeline_lib(tempfile.mkdtemp(prefix="mrs_timeline_"))
    from mistralrs_b200 import lib, model as M
    sys.path.insert(0, ROOT)
    from bench import ClockSampler, PROMPT_LEN, GEN_LEN

    dev = torch.device("cuda:0")
    cfg = M.LlamaConfig.llama3_8b()
    weights = M.LlamaWeights(cfg, dev)
    plan = chain_plan(cfg, M)
    n = len(chain_plan(cfg, M, one_grid_v=False))   # room for either form
    L = lib()
    L.mrs_mmvq_timeline.argtypes = [ctypes.c_void_p, ctypes.c_int]
    L.mrs_mmvq_timeline.restype = ctypes.c_int

    run = M.LlamaRunner(weights, batch=1, max_ctx=PROMPT_LEN + GEN_LEN + 16, pdl=True)
    run.reset(PROMPT_LEN + GEN_LEN // 2)
    run.step(); torch.cuda.synchronize()
    buf = torch.zeros(n * SLOTS * 16, dtype=torch.int64, device=dev)
    L.mrs_mmvq_timeline(ctypes.c_void_p(buf.data_ptr()), n)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        run.step()
    got = L.mrs_mmvq_timeline(ctypes.c_void_p(0), 0)      # launches recorded at capture; stop recording new ones
    if got != len(plan):
        plan = chain_plan(cfg, M, one_grid_v=False)       # a library that launches v on its own
    if got != len(plan):
        raise RuntimeError(f"recorded {got} GEMV launches, the plan has {len(plan)}")
    sampler = ClockSampler(0)
    sampler.start()
    tokens = []
    for r in range(args.reps + 3):
        run.reset(PROMPT_LEN + GEN_LEN // 2)
        gr.replay()
        torch.cuda.synchronize()
        if r >= 3:
            tokens.append(buf.cpu().numpy().reshape(n, SLOTS, 16)[:got].copy())
    rates = stream_rates(weights, cfg, M, L, dev, plan)
    clocks = sampler.stop()

    per_launch, roles, total = attribute(plan, tokens, rates)
    result = {"gpu": facts, "clocks": clocks, "stream_rates": rates, "roles": roles, "total": total,
              "launches": per_launch, "tokens_recorded": len(tokens)}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gemv_chain.json"), "w") as f:
        json.dump(result, f, indent=1)

    print(f"{facts['name']}, power limit {facts['power_limit_w']} W, median SM clock {clocks.get('sm_mhz')} MHz "
          f"(max {facts['sm_max_mhz']}), throttle reasons {clocks.get('reasons')}")
    print("stream rate of each shape alone (GB/s): " +
          ", ".join(f"{k} {v['gbs']:.0f} ({v['us_per_launch']:.1f} us)" for k, v in rates.items()))
    cols = ("ideal", "span", "entry_wait", "prologue", "first_seg", "consume", "tail")
    print(f"{'role':8s} {'n':>4s} " + " ".join(f"{c:>10s}" for c in cols) + "   (us per token; phases are CTA medians summed over launches)")
    for name in ("qkv", "qk_v", "qk", "v", "o_proj", "gate_up", "down", "lm_head"):
        if name in roles:
            r = roles[name]
            print(f"{name:8s} {r['launches']:4d} " + " ".join(f"{r[c]:10.1f}" for c in cols))
    print(f"{'total':8s} {total['launches']:4d} " + " ".join(f"{total[c]:10.1f}" for c in cols))


if __name__ == "__main__":
    main()
