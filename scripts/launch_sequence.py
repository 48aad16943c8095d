"""Print the kernel launches of the Llama and GPTQ decode, verify and prompt steps (GPTQ also on act-order and AWQ
checkpoints), one line per kernel node of a captured CUDA graph, in dependency order: kernel name, grid, block, dynamic
shared memory, cluster dimensions (when set) and whether the incoming edge is programmatic (a PDL link).  Two builds of
libmrs_b200.so that print the same lines enqueue the same launches, so a refactor of host-side launch code can be
checked against its parent:

    python scripts/launch_sequence.py > new.txt
    python scripts/launch_sequence.py --lib /path/to/parent/libmrs_b200.so > old.txt
    diff old.txt new.txt

The graph is read back through the driver API, as bench.py's count_graph_kernels does.  Synthetic seeded weights, and
checkpoints written by the seeded writer of tests/test_gptq_checkpoint_host.py into a temporary directory; the values
computed do not matter here, only what is launched.  Needs a GPU."""
import argparse
import ctypes
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CU_GRAPH_NODE_TYPE_KERNEL = 0
CU_GRAPH_DEPENDENCY_TYPE_PROGRAMMATIC = 1
CU_LAUNCH_ATTRIBUTE_CLUSTER_DIMENSION = 4


class _KernelNodeParams(ctypes.Structure):     # CUDA_KERNEL_NODE_PARAMS_v2
    _fields_ = [("func", ctypes.c_void_p)] + [(n, ctypes.c_uint) for n in (
        "gridDimX", "gridDimY", "gridDimZ", "blockDimX", "blockDimY", "blockDimZ", "sharedMemBytes")] + \
               [("kernelParams", ctypes.c_void_p), ("extra", ctypes.c_void_p), ("kern", ctypes.c_void_p),
                ("ctx", ctypes.c_void_p)]


class _EdgeData(ctypes.Structure):             # CUgraphEdgeData
    _fields_ = [("from_port", ctypes.c_ubyte), ("to_port", ctypes.c_ubyte), ("type", ctypes.c_ubyte),
                ("reserved", ctypes.c_ubyte * 5)]


def _check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what}: CUresult {rc}")


def graph_lines(graph):
    """one line per kernel node of a torch CUDAGraph (captured with keep_graph=True), in dependency order"""
    cu = ctypes.CDLL("libcuda.so.1")
    raw = ctypes.c_void_p(int(graph.raw_cuda_graph()))
    n = ctypes.c_size_t(0)
    _check(cu.cuGraphGetNodes(raw, None, ctypes.byref(n)), "cuGraphGetNodes")
    nodes = (ctypes.c_void_p * n.value)()
    _check(cu.cuGraphGetNodes(raw, nodes, ctypes.byref(n)), "cuGraphGetNodes")
    order = [int(nodes[i]) for i in range(n.value)]
    ne = ctypes.c_size_t(0)
    _check(cu.cuGraphGetEdges_v2(raw, None, None, None, ctypes.byref(ne)), "cuGraphGetEdges_v2")
    src, dst = (ctypes.c_void_p * max(ne.value, 1))(), (ctypes.c_void_p * max(ne.value, 1))()
    data = (_EdgeData * max(ne.value, 1))()
    _check(cu.cuGraphGetEdges_v2(raw, src, dst, data, ctypes.byref(ne)), "cuGraphGetEdges_v2")
    preds = {v: [] for v in order}
    for i in range(ne.value):
        preds[int(dst[i])].append((int(src[i]), data[i].type == CU_GRAPH_DEPENDENCY_TYPE_PROGRAMMATIC))
    # Kahn's algorithm, ties broken by the driver's node order (capture order)
    pending = {v: len(p) for v, p in preds.items()}
    succ = {v: [] for v in order}
    for v, ps in preds.items():
        for u, _ in ps:
            succ[u].append(v)
    ready = [v for v in order if pending[v] == 0]
    rank = {v: i for i, v in enumerate(order)}
    lines = []
    while ready:
        ready.sort(key=rank.get)
        v = ready.pop(0)
        for w in succ[v]:
            pending[w] -= 1
            if pending[w] == 0:
                ready.append(w)
        ty = ctypes.c_int(-1)
        _check(cu.cuGraphNodeGetType(ctypes.c_void_p(v), ctypes.byref(ty)), "cuGraphNodeGetType")
        if ty.value != CU_GRAPH_NODE_TYPE_KERNEL:
            lines.append(f"node type {ty.value}")
            continue
        p = _KernelNodeParams()
        _check(cu.cuGraphKernelNodeGetParams_v2(ctypes.c_void_p(v), ctypes.byref(p)), "cuGraphKernelNodeGetParams")
        name = ctypes.c_char_p()
        if p.func:
            _check(cu.cuFuncGetName(ctypes.byref(name), ctypes.c_void_p(p.func)), "cuFuncGetName")
        else:
            _check(cu.cuKernelGetName(ctypes.byref(name), ctypes.c_void_p(p.kern)), "cuKernelGetName")
        attr = (ctypes.c_uint * 16)()              # CUlaunchAttributeValue: clusterDim {x, y, z} first
        cl = ""
        if cu.cuGraphKernelNodeGetAttribute(ctypes.c_void_p(v), CU_LAUNCH_ATTRIBUTE_CLUSTER_DIMENSION, attr) == 0 and attr[0]:
            cl = f" cluster=({attr[0]},{attr[1]},{attr[2]})"
        pdl = any(prog for _, prog in preds[v])
        lines.append(f"{name.value.decode()} grid=({p.gridDimX},{p.gridDimY},{p.gridDimZ}) "
                     f"block=({p.blockDimX},{p.blockDimY},{p.blockDimZ}) smem={p.sharedMemBytes}{cl}"
                     f"{' pdl' if pdl else ''}")
    if len(lines) != len(order):
        raise RuntimeError("the captured graph has a cycle")
    return lines


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--lib", default=None, help="another build of libmrs_b200.so (same C ABI)")
    args = ap.parse_args()
    import __graft_entry__ as entry
    pkg = entry.load_package()
    if args.lib:
        pkg.LIB_PATH = os.path.abspath(args.lib)
    import torch
    from mistralrs_b200 import model as M

    dev = torch.device("cuda:0")
    tdt = {"bf16": torch.bfloat16, "f16": torch.float16}
    weights = {}

    def model(quant, dt="bf16", big=False):
        key = (quant, dt, big)
        if key not in weights:
            if big:   # Llama-3-8B Q4_K_M shapes; layer 0 has a uniform QKV, layer 1 q|k + a Q6_K v
                cfg = M.LlamaConfig.llama3_8b(n_layers=2, max_pos=4096)
            else:
                kw = dict(synth_scale_exp=(-15, -13)) if (quant, dt) == ("q4_k_m", "f16") else {}
                cfg = M.LlamaConfig.tiny_test(quant=quant, n_layers=2, max_pos=4096, **kw)
            weights[key] = M.LlamaWeights(cfg, dev, dtype=tdt[dt])
        return weights[key]

    def capture(fn):
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph(keep_graph=True)
        with torch.cuda.graph(g):
            fn()
        torch.cuda.synchronize()
        return g

    def report(name, graph):
        lines = graph_lines(graph)
        print(f"== {name}: {len(lines)} nodes")
        for l in lines:
            print(l)
        sys.stdout.flush()

    # ---- decode steps: advance + layer stack + lm_head + argmax
    decode = []
    for quant in ("q4_k_m", "q8_0"):
        for B in (1, 4, 16, 64):
            decode.append((f"decode {quant} B={B}", quant, B, {}, "bf16", False))
    decode += [("decode q4_k_m B=1 f16", "q4_k_m", 1, {}, "f16", False),
               ("decode q4_k_m B=1 unfused attention", "q4_k_m", 1, dict(fused_attention=False), "bf16", False),
               ("decode q4_k_m B=1 pdl off", "q4_k_m", 1, dict(pdl=False), "bf16", False),
               ("decode q4_k_m B=1 comm no-op", "q4_k_m", 1, dict(comm=lambda *a: None), "bf16", False),
               ("decode llama-3-8b q4_k_m B=1", "q4_k_m", 1, {}, "bf16", True),
               ("decode llama-3-8b q4_k_m B=16", "q4_k_m", 16, {}, "bf16", True)]
    for name, quant, B, kw, dt, big in decode:
        kw = dict(dict(pdl=True), **kw)
        run = M.LlamaRunner(model(quant, dt, big), batch=B, max_ctx=64, **kw)
        run.set_tokens([(7 * b + 1) % 500 for b in range(B)])
        run.step()
        report(name, capture(run.step))
        del run

    # ---- GPTQ decode steps: advance + W4A16 layer stack + dense lm_head + argmax, split plan (HND) and unsplit (vLLM)
    from mistralrs_b200 import gptq_model as G

    def gptq_decode(name, gw, layout, B, skip_mask=0):
        run = G.GptqRunner(gw, batch=B, max_ctx=400, cache_layout=layout)
        run.step_struct.skip_mask = skip_mask
        run.set_tokens([(5 * b + 3) % 500 for b in range(B)])
        run.step()
        report(name, capture(run.step))
        del run

    # ---- GPTQ verify steps (HND): advance_multi + W4A16 layer stack over B*q rows + lm_head + argmax + acceptance
    def gptq_verify(name, gw, B, q):
        run = G.GptqRunner(gw, batch=B, max_ctx=400)
        run.set_tokens([(5 * b + 3) % 500 for b in range(B)])
        run.step()
        ver = G.GptqVerifier(run, draft_len=q - 1)
        ver.sync_from_runner()
        ver.set_drafts([[(b + i) % 500 for i in range(q - 1)] for b in range(B)])
        ver.step()
        report(name, capture(ver.step))
        del ver, run

    gw = G.GptqWeights(G.GptqConfig.tiny_test(max_pos=4096), dev)
    for layout in ("hnd", "vllm"):
        for B in (4, 32):
            gptq_decode(f"gptq decode {layout} B={B}", gw, layout, B)
    # skip_mask bit 0: bench.py's linears-only graph; bit 2: plain stream order
    gptq_decode("gptq decode hnd B=32 skip_mask=1", gw, "hnd", 32, skip_mask=1)
    gptq_decode("gptq decode hnd B=32 skip_mask=4", gw, "hnd", 32, skip_mask=4)
    for B, q in ((4, 4), (32, 8)):
        gptq_verify(f"gptq verify hnd B={B} q={q}", gw, B, q)

    # ---- verify steps: advance_multi + layer stack + lm_head + argmax + acceptance
    for B, q in ((1, 4), (2, 4), (16, 4), (33, 8)):
        run = M.LlamaRunner(model("q4_k_m"), batch=B, max_ctx=64, pdl=True)
        run.set_tokens([(3 * b + 2) % 500 for b in range(B)])
        run.step()
        ver = M.LlamaVerifier(run, draft_len=q - 1)
        ver.sync_from_runner()
        ver.set_drafts([[(b + i) % 500 for i in range(q - 1)] for b in range(B)])
        ver.step()
        report(f"verify q4_k_m B={B} q={q}", capture(ver.step))
        del ver, run

    # ---- prompt steps: only the step call (pre.STEP), the plan built eagerly before the capture
    def prefill_case(name, pre, prompts, cached, tables, lm_rows, slots=None):
        p, _, plan = pre.make_plan(prompts, cached, tables, lm_rows, slots)    # plan: the device arrays p points into

        def call():
            rc = getattr(pkg.lib(), pre.STEP)(ctypes.byref(pre.step_struct), ctypes.byref(p),
                                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
            if rc != 0:
                raise RuntimeError(f"{pre.STEP} failed: cudaError {rc}")
        call()                                    # eager warm-up: module loads and kernel attributes
        report(name, capture(call))
        del plan

    # the Llama prompt cases, repeated for the GPTQ prompt step: Prefill(weights, max_tokens=, runner=) and Runner(weights,
    # batch=, max_ctx=) build the step's objects
    def prefill_cases(tag, Prefill, Runner, w):
        pre = Prefill(w, max_tokens=64)
        prefill_case(f"{tag} n=1 unpaged lm_rows=1", pre, [list(range(5, 25))], [0], [pre.table], 1)
        runner = Runner(w, batch=12, max_ctx=128)
        pre = Prefill(w, max_tokens=128, runner=runner)
        prompts = [[(11 * i + j) % 500 for j in range(6 + i)] for i in range(9)]
        tables = [list(runner.tables[i]) for i in range(9)]
        pre.forward_batch([p[:4] for p in prompts[::3]], tables=tables[::3], final=False)
        cached = [4 if i % 3 == 0 else 0 for i in range(9)]
        prefill_case(f"{tag} n=9 paged lm_rows=1 commit", pre, [p[c:] for p, c in zip(prompts, cached)], cached, tables, 1,
                     slots=list(range(9)))
        pre = Prefill(w, max_tokens=64)
        own = [[1 + i] for i in range(4)]
        prefill_case(f"{tag} n=4 lm_rows=2", pre, [[(5 * i + j) % 500 for j in range(8)] for i in range(4)], [0] * 4, own, 2)
        pre = Prefill(w, max_tokens=2400)
        own = [list(range(1 + 18 * i, 19 + 18 * i)) for i in range(8)]
        prefill_case(f"{tag} n=8 T=2240 lm_rows=0", pre, [[(13 * i + j) % 500 for j in range(280)] for i in range(8)],
                     [0] * 8, own, 0)

    # the vLLM-layout GPTQ prompt step (unpaged only) with a commit into a vLLM-layout runner
    def gptq_prefill_vllm(name, gw):
        runner = G.GptqRunner(gw, batch=4, max_ctx=128, cache_layout="vllm")
        pre = G.GptqPrefill(gw, max_tokens=64, runner=runner)
        prefill_case(name, pre, [[(7 * i + j) % 500 for j in range(5 + 3 * i)] for i in range(4)], [0] * 4,
                     [list(runner.tables[i]) for i in range(4)], 1, slots=list(range(4)))

    prefill_cases("prefill", M.LlamaPrefill, lambda w, **kw: M.LlamaRunner(w, pdl=True, **kw), model("q4_k_m"))
    prefill_cases("gptq prefill", G.GptqPrefill, G.GptqRunner, gw)
    gptq_prefill_vllm("gptq prefill vllm n=4 unpaged lm_rows=1 commit", gw)
    pre = G.GptqPrefill(gw, max_tokens=64, pdl=False)
    prefill_case("gptq prefill n=1 unpaged lm_rows=1 pdl off", pre, [list(range(5, 25))], [0], [pre.table], 1)
    del pre, gw

    # ---- act-order GPTQ and AWQ checkpoints (the seeded writer of the host tests, into a temporary directory)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gptq_checkpoint_host import make_checkpoint
    with tempfile.TemporaryDirectory() as tmp:
        cfg = G.GptqConfig.tiny_test(max_pos=4096)
        gw = G.GptqWeights.from_checkpoint(make_checkpoint(os.path.join(tmp, "act"), cfg, act_order=True), dev)
        for layout in ("hnd", "vllm"):
            gptq_decode(f"gptq act-order decode {layout} B=32", gw, layout, 32)
        gptq_verify("gptq act-order verify hnd B=4 q=4", gw, 4, 4)
        prefill_cases("gptq act-order prefill", G.GptqPrefill, G.GptqRunner, gw)
        gptq_prefill_vllm("gptq act-order prefill vllm n=4 unpaged lm_rows=1 commit", gw)
        del gw
        gw = G.GptqWeights.from_checkpoint(make_checkpoint(os.path.join(tmp, "awq"), cfg, method="awq"), dev)
        for layout in ("hnd", "vllm"):
            gptq_decode(f"awq decode {layout} B=4", gw, layout, 4)
        del gw


if __name__ == "__main__":
    main()
