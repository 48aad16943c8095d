"""Runs the UNMODIFIED reference CUDA kernels (oracle/_ref/*.so, built from the reference sources by
oracle/build_ref.sh) on seeded inputs and stores their outputs as golden vectors:
    python tests/golden/make_ref_golden.py OUT.npz     (on a GPU machine)
The committed copy tests/golden/ref_golden.npz pins the CPU oracle (tests/test_oracle_golden.py) and the product
kernels (tests/test_ref_golden_gpu.py) against what the reference itself computes.  To keep the file small, the
larger products are stored as a fixed, seeded sample (`sample` below): the first output columns, and for the
token-batched products a subset of token rows (`*_rows`); a token row's output depends on that row's input only."""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402

dev = torch.device("cuda:0")
P = lambda t: ctypes.c_void_p(t.data_ptr())
ST = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
TYPES = ["q4_0", "q4_1", "q5_0", "q5_1", "q8_0", "q2_k", "q3_k", "q4_k", "q5_k", "q6_k"]
out = {}
rng = np.random.default_rng(77)

# ---- Q8_1 quantiser + MMVQ (f32 outputs: no output rounding) -------------------------------
L = oracle.ref_lib("mmvq")
K, N, B = 1024, 24, 2
x = oracle.round_dtype(rng.standard_normal((B, K)).astype(np.float32), "bf16")
out["mmvq_x"] = x
xb = torch.from_numpy(x).to(dev).to(torch.bfloat16)
y = torch.zeros(B * (K // 32) * 36, dtype=torch.uint8, device=dev)
L.launch_mmvq_gguf_quantize_q8_1_bf16(P(xb), P(y), K, K, B, ST())
out["q8_1_bytes"] = y.cpu().numpy()
for t in TYPES:
    wb = oracle.random_blocks(t, N * K // oracle.BLOCK_ELEMS[t], rng)
    w = torch.from_numpy(wb.reshape(-1)).to(dev)
    dst = torch.zeros(B, N, dtype=torch.float32, device=dev)
    getattr(L, f"launch_mmvq_gguf_{t}_f32_plain")(P(w), P(y), P(dst), K, N, K // 32, N, B, ST())
    out[f"mmvq_{t}_w"] = wb
    out[f"mmvq_{t}_y"] = dst.cpu().numpy()
    # fused GLU (silu), bf16 out
    wu = oracle.random_blocks(t, N * K // oracle.BLOCK_ELEMS[t], rng)
    w2 = torch.from_numpy(wu.reshape(-1)).to(dev)
    dg = torch.zeros(B, N, dtype=torch.bfloat16, device=dev)
    getattr(L, f"launch_mmvq_gguf_{t}_bf16_fused_glu")(P(w), P(w2), P(y), P(dg), K, N, K // 32, N, B, 0, ST())
    out[f"mmvq_{t}_up"] = wu
    out[f"mmvq_{t}_glu"] = dg.float().cpu().numpy()

# ---- fused_glu elementwise ---------------------------------------------------------------
L = oracle.ref_lib("ops")
a = oracle.round_dtype(3 * rng.standard_normal((4, 256)).astype(np.float32), "bf16")
b = oracle.round_dtype(rng.standard_normal((4, 256)).astype(np.float32), "bf16")
out["glu_a"], out["glu_b"] = a, b
ta, tb = torch.from_numpy(a).to(dev).to(torch.bfloat16), torch.from_numpy(b).to(dev).to(torch.bfloat16)
for act in range(5):
    o = torch.zeros_like(ta)
    L.fused_glu_bf16(P(ta), P(tb), P(o), ctypes.c_uint32(4), ctypes.c_uint32(256), ctypes.c_uint32(256), ctypes.c_uint32(256), act, ST())
    out[f"glu_out_{act}"] = o.float().cpu().numpy()

# ---- rotary ------------------------------------------------------------------------------
L = oracle.ref_lib("rotary")
T_, H, KVH, D = 5, 4, 2, 128
cos, sin = oracle.llama3_rope_table(64, D, 500000.0, None)
cos, sin = oracle.round_dtype(cos, "bf16"), oracle.round_dtype(sin, "bf16")
q = oracle.round_dtype(rng.standard_normal((T_, H * D)).astype(np.float32), "bf16")
k = oracle.round_dtype(rng.standard_normal((T_, KVH * D)).astype(np.float32), "bf16")
pos = np.array([0, 3, 17, 40, 63], dtype=np.uint32)
out.update(rope_q=q, rope_k=k, rope_cos=cos, rope_sin=sin, rope_pos=pos)
for neox in (1, 0):
    tq, tk = torch.from_numpy(q).to(dev).to(torch.bfloat16), torch.from_numpy(k).to(dev).to(torch.bfloat16)
    tc, ts = torch.from_numpy(cos).to(dev).to(torch.bfloat16), torch.from_numpy(sin).to(dev).to(torch.bfloat16)
    tp = torch.from_numpy(pos.astype(np.int32)).to(dev)
    L.rotary_embedding_positions(P(tq), P(tk), P(tc), P(ts), P(tp), neox, D, ctypes.c_int64(T_), D // 2, 64, H, KVH,
                                 ctypes.c_int64(H * D), ctypes.c_int64(KVH * D), ctypes.c_uint32(1), ctypes.c_int64(torch.cuda.current_stream().cuda_stream))
    out[f"rope_q_out_{neox}"] = tq.float().cpu().numpy()
    out[f"rope_k_out_{neox}"] = tk.float().cpu().numpy()

# ---- add_rms_norm ------------------------------------------------------------------------
L = oracle.ref_lib("rmsnorm")
xr = oracle.round_dtype(rng.standard_normal((3, 1024)).astype(np.float32), "bf16")
rr = oracle.round_dtype(rng.standard_normal((3, 1024)).astype(np.float32), "bf16")
wr = oracle.round_dtype(1 + 0.1 * rng.standard_normal(1024).astype(np.float32), "bf16")
out.update(rms_x=xr, rms_res=rr, rms_w=wr)
tx, tr, tw = (torch.from_numpy(v).to(dev).to(torch.bfloat16) for v in (xr, rr, wr))
s_, n_ = torch.zeros_like(tx), torch.zeros_like(tx)
L.add_rms_norm_bf16(P(tx), P(tr), P(tw), P(s_), P(n_), 3, 1024, ctypes.c_float(1e-5), ctypes.c_int64(torch.cuda.current_stream().cuda_stream))
out["rms_sum"], out["rms_norm"] = s_.float().cpu().numpy(), n_.float().cpu().numpy()

# ---- reshape_and_cache (both layouts) + paged attention ------------------------------------
Lc = oracle.ref_lib("cache")
S, H, KVH, D, BS, NB = 2, 8, 2, 128, 16, 9
ctx = [37, 70]
kv = oracle.round_dtype(rng.standard_normal((sum(ctx), KVH * D)).astype(np.float32), "bf16")
vv = oracle.round_dtype(rng.standard_normal((sum(ctx), KVH * D)).astype(np.float32), "bf16")
tables = [[1, 2, 3, 0, 0], [4, 5, 6, 7, 8]]
slots = []
for s, c in enumerate(ctx):
    slots += [tables[s][i // BS] * BS + i % BS for i in range(c)]
slots = np.array(slots, dtype=np.int64)
out.update(pa_k=kv, pa_v=vv, pa_slots=slots, pa_tables=np.array(tables, dtype=np.int32), pa_ctx=np.array(ctx, dtype=np.int32))
tk_, tv_ = torch.from_numpy(kv).to(dev).to(torch.bfloat16), torch.from_numpy(vv).to(dev).to(torch.bfloat16)
tsl = torch.from_numpy(slots).to(dev)
kc = torch.zeros(NB, KVH, D // 8, BS, 8, dtype=torch.bfloat16, device=dev)
vc = torch.zeros(NB, KVH, D, BS, dtype=torch.bfloat16, device=dev)
Lc.reshape_and_cache(P(tk_), P(tv_), P(kc), P(vc), P(tsl), len(slots), KVH, D, BS, 8, KVH * D, KVH * D, ST(),
                     ctypes.c_uint32(1), ctypes.c_uint32(1), ctypes.c_void_p(0), ctypes.c_void_p(0))
out["cache_k_vllm"] = kc.view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)
out["cache_v_vllm"] = vc.view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)
qa = oracle.round_dtype(rng.standard_normal((S, H, D)).astype(np.float32), "bf16")
out["pa_q"] = qa
tq = torch.from_numpy(qa).to(dev).to(torch.bfloat16)
La = oracle.ref_lib("pagedattn")
if La is not None:
    o = torch.zeros(S, H, D, dtype=torch.bfloat16, device=dev)
    bt = torch.tensor(tables, dtype=torch.int32, device=dev)
    cl = torch.tensor(ctx, dtype=torch.int32, device=dev)
    La.paged_attention_v1_bf16(P(o), P(tq), P(kc), P(vc), ctypes.c_void_p(0), KVH, ctypes.c_float(1.0 / np.sqrt(D)), ctypes.c_float(1.0),
                               P(bt), P(cl), BS, max(ctx), S, H, D, 5, H * D, kc.stride(0), kc.stride(1), ST(), ctypes.c_uint32(1),
                               ctypes.c_void_p(0), ctypes.c_void_p(0), ctypes.c_void_p(0))
    out["pa_out_v1"] = o.float().cpu().numpy()
Lf = oracle.ref_lib("flashinfer")
if Lf is not None:
    kch = torch.zeros(NB, KVH, BS, D, dtype=torch.bfloat16, device=dev)
    vch = torch.zeros_like(kch)
    Lf.reshape_and_cache_flashinfer(P(tk_), P(tv_), P(kch), P(vch), P(tsl), len(slots), KVH, D, BS, KVH * D, KVH * D,
                                    ctypes.c_float(1.0), ctypes.c_float(1.0), ctypes.c_uint32(1), ctypes.c_uint32(1), ST())
    out["cache_k_hnd"] = kch.view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)
    out["cache_v_hnd"] = vch.view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)
    I = lambda a: torch.tensor(a, dtype=torch.int32, device=dev)
    indptr, indices, last = I([0, 3, 8]), I([1, 2, 3, 4, 5, 6, 7, 8]), I([37 - 32, 70 - 64])
    req, tile, oind, chunk = I([0, 1]), I([0, 0]), I([0, 1, 2]), I([16])
    mask = torch.ones(2, dtype=torch.uint8, device=dev)
    o = torch.zeros(S, H, D, dtype=torch.bfloat16, device=dev)
    Lf.flashinfer_decode.restype = ctypes.c_int32
    rc = Lf.flashinfer_decode(P(tq), P(kch), P(vch), P(indptr), P(indices), P(last), P(req), P(tile), P(oind), P(chunk), P(mask),
                              P(o), ctypes.c_void_p(0), ctypes.c_void_p(0), S, S, H, KVH, D, BS, H * D, D, ctypes.c_float(1.0 / np.sqrt(D)),
                              -1, ctypes.c_float(0.0), ctypes.c_float(1.0), ctypes.c_float(1.0), ctypes.c_uint32(1), ctypes.c_uint32(1), ST())
    torch.cuda.synchronize()
    out["fi_rc"] = np.array(rc)
    out["fi_out"] = o.float().cpu().numpy()
# ---- MMQ (prefill GEMM with int8 activations): quantize + launch_mmq_gguf_<q> -------------------
# call shape: REF fast_mmq.rs:388-447 (DenseMmqRun::launch), k_padded / workspace sizes :599-603,
# ds layouts :91-100, type codes :591-596 (bf16 = 30)
Lm = oracle.ref_lib("mmq")
if Lm is not None:
    Mq, Nq, Kq = 64, 256, 1024
    xm = oracle.round_dtype(rng.standard_normal((Mq, Kq)).astype(np.float32), "bf16")
    out["mmq_x"] = xm
    txm = torch.from_numpy(xm).to(dev).to(torch.bfloat16)
    kp = (Kq + 511) // 512 * 512
    ws = torch.zeros(Mq * (kp // 128) * 144 + 128 * 144, dtype=torch.uint8, device=dev)
    nsm = torch.cuda.get_device_properties(dev).multi_processor_count
    fix = torch.zeros(nsm * 128 * 128, dtype=torch.float32, device=dev)
    I64 = ctypes.c_int64
    for t, layout in (("q4_k", "DS4"), ("q6_k", "D4"), ("q8_0", "D4")):
        wb = oracle.random_blocks(t, Nq * Kq // oracle.BLOCK_ELEMS[t], rng)
        w = torch.from_numpy(wb.reshape(-1)).to(dev)
        getattr(Lm, f"launch_mmq_quantize_q8_1_{layout}")(P(txm), ctypes.c_void_p(0), P(ws), 30, I64(Kq), I64(Kq), I64(0), I64(0),
                                                         I64(kp), I64(Mq), I64(1), I64(1), ST())
        dst = torch.zeros(Mq, Nq, dtype=torch.bfloat16, device=dev)
        getattr(Lm, f"launch_mmq_gguf_{t}")(P(fix), P(w), P(ws), P(dst), I64(Kq), I64(Nq), I64(Mq),
                                           I64(Kq // oracle.BLOCK_ELEMS[t]), I64(Nq), 1000, nsm, I64(232448), 32, 30, ST())
        torch.cuda.synchronize()
        out[f"mmq_{t}_w"] = wb
        out[f"mmq_{t}_y"] = dst.float().cpu().numpy()

# ---- Marlin GPTQ int4 (sym, group 128): gptq_marlin_repack + marlin_gptq_4bit_f16 ---------------
# load-time transforms: REF gptq/gptq_cuda.rs:530-602 (repack with perm = argsort(g_idx), scale
# permutation `marlin_permute_scales`), forward: gptq/marlin_backend.rs:20-140
Lr = oracle.ref_lib("marlin")
if Lr is not None:
    for tag, Mg in (("m32", 32), ("m1", 1), ("m300", 300)):
        Kg, Ng, G = 1024, 512, 128
        xg = (rng.standard_normal((Mg, Kg)).astype(np.float32)).astype(np.float16)
        qw = rng.integers(0, 2 ** 32, size=(Kg // 8, Ng), dtype=np.uint64).astype(np.uint32).view(np.int32)
        sc = np.exp2(rng.uniform(-8, -6, size=(Kg // G, Ng))).astype(np.float16)
        out[f"marlin_{tag}_x"], out[f"marlin_{tag}_qweight"], out[f"marlin_{tag}_scales"] = xg, qw, sc
        tqw = torch.from_numpy(qw).to(dev)
        perm = torch.arange(Kg, dtype=torch.int32, device=dev)       # g_idx[k] = k / G  ->  argsort = identity
        rep = torch.zeros(Kg // 16, Ng * 16 // 8, dtype=torch.int32, device=dev)
        Lr.gptq_marlin_repack(P(tqw), P(perm), P(rep), Kg, Ng, 4, ctypes.c_int64(torch.cuda.current_stream().cuda_stream))
        scale_perm = [i + 8 * j for i in range(8) for j in range(8)]
        sp = sc.reshape(-1, 64)[:, scale_perm].reshape(-1, Ng)       # group_size < size_k: the 64-wide permutation
        tsp = torch.from_numpy(np.ascontiguousarray(sp)).to(dev)
        wsg = torch.zeros(Ng // 8, dtype=torch.int32, device=dev)
        og = torch.zeros(Mg, Ng, dtype=torch.float16, device=dev)
        txg = torch.from_numpy(xg).to(dev)
        Lr.marlin_gptq_4bit_f16.restype = ctypes.c_int
        rc = Lr.marlin_gptq_4bit_f16(P(txg), P(rep), P(tsp), ctypes.c_void_p(0), P(og), Mg, Kg, Ng, P(wsg), G,
                                     ctypes.c_int64(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        out[f"marlin_{tag}_rc"] = np.array(rc)
        out[f"marlin_{tag}_y"] = og.float().cpu().numpy()

# ---- paged_attention_v2 (split) + ALiBi / sinks / softcap variants of v1 ------------------------
if La is not None:
    bt = torch.tensor(tables, dtype=torch.int32, device=dev)
    cl = torch.tensor(ctx, dtype=torch.int32, device=dev)
    slopes = (0.25 * 2.0 ** -np.arange(H)).astype(np.float32)
    sinks = rng.standard_normal(H).astype(np.float32)
    out["pa_alibi"], out["pa_sinks"] = slopes, sinks
    tsl_, tsk_ = torch.from_numpy(slopes).to(dev), torch.from_numpy(sinks).to(dev)
    for name, al, cap, sk in (("alibi", tsl_, 1.0, None), ("softcap", None, 30.0, None), ("sinks", None, 1.0, tsk_)):
        o = torch.zeros(S, H, D, dtype=torch.bfloat16, device=dev)
        La.paged_attention_v1_bf16(P(o), P(tq), P(kc), P(vc), P(al) if al is not None else ctypes.c_void_p(0), KVH,
                                   ctypes.c_float(1.0 / np.sqrt(D)), ctypes.c_float(cap), P(bt), P(cl), BS, max(ctx), S, H, D, 5,
                                   H * D, kc.stride(0), kc.stride(1), ST(), ctypes.c_uint32(1), ctypes.c_void_p(0), ctypes.c_void_p(0),
                                   P(sk) if sk is not None else ctypes.c_void_p(0))
        out[f"pa_out_v1_{name}"] = o.float().cpu().numpy()

# ---- sampling tail: topk_large_f32_packed + top1_large_f32_packed (mistralrs-core/src/cuda/sort.cu) --------------------
# input regenerated by tests/test_sampler_gpu.py: default_rng(5), 128256 bf16-rounded logits, k = 40, temperature 0.8
Ls = oracle.ref_lib("rmsnorm")
if Ls is not None:
    ncols, k = 128256, 40
    nblocks = -(-ncols // 2048)
    xs = torch.from_numpy(np.random.default_rng(5).standard_normal(ncols).astype(np.float32) * 3).to(torch.bfloat16).float().to(dev)
    bv = torch.zeros(nblocks * k, dtype=torch.float32, device=dev); bi = torch.zeros(nblocks * k, dtype=torch.int32, device=dev)
    bm = torch.zeros(nblocks, dtype=torch.float32, device=dev); bs = torch.zeros(nblocks, dtype=torch.float32, device=dev)
    packed = torch.zeros(2 * k + 2, dtype=torch.float32, device=dev)
    st = ctypes.c_int64(torch.cuda.current_stream().cuda_stream)
    Ls.topk_large_f32_packed(P(xs), P(bv), P(bi), P(bm), P(bs), P(packed), ncols, k, 2048, nblocks, ctypes.c_float(1.0 / 0.8), st)
    p1 = torch.zeros(2, dtype=torch.float32, device=dev); tok = torch.zeros(1, dtype=torch.int32, device=dev)
    Ls.top1_large_f32_packed(P(xs), P(bv), P(bi), P(p1), P(tok), ncols, 2048, nblocks, st)
    torch.cuda.synchronize()
    out["sort_topk_packed"], out["sort_top1_packed"], out["sort_top1_token"] = packed.cpu().numpy(), p1.cpu().numpy(), tok.cpu().numpy()

torch.cuda.synchronize()


def sample(z):
    """the stored subset: 8 of the 24 MMVQ outputs, 32 of the 256 MMQ / 512 Marlin output columns (and the weight rows
    behind them), 15 of the 64 MMQ token rows, 8 of the 32 and 22 of the 300 Marlin token rows"""
    rng = np.random.default_rng(300)
    rows_of = lambda m, n, must: np.unique(np.concatenate([must, rng.choice(m, n, replace=False)])).astype(np.int32)
    for t in TYPES:
        per = 1024 // oracle.BLOCK_ELEMS[t]
        for s in ("w", "up"):
            z[f"mmvq_{t}_{s}"] = np.ascontiguousarray(z[f"mmvq_{t}_{s}"][: 8 * per])
        for s in ("y", "glu"):
            z[f"mmvq_{t}_{s}"] = np.ascontiguousarray(z[f"mmvq_{t}_{s}"][:, :8])
    if "mmq_x" in z:
        r = rows_of(64, 14, [0, 63])
        z["mmq_rows"], z["mmq_x"] = r, np.ascontiguousarray(z["mmq_x"][r])
        for t in ("q4_k", "q6_k", "q8_0"):
            z[f"mmq_{t}_w"] = np.ascontiguousarray(z[f"mmq_{t}_w"][: 32 * (1024 // oracle.BLOCK_ELEMS[t])])
            z[f"mmq_{t}_y"] = np.ascontiguousarray(z[f"mmq_{t}_y"][r][:, :32])
    if "marlin_m1_y" in z:
        for tag in ("m1", "m32", "m300"):
            for s in ("qweight", "scales", "y"):
                z[f"marlin_{tag}_{s}"] = np.ascontiguousarray(z[f"marlin_{tag}_{s}"][:, :32])
        for tag, m, n, must in (("m300", 300, 16, [0, 127, 128, 255, 256, 299]), ("m32", 32, 6, [0, 31])):
            r = rows_of(m, n, must)
            z[f"marlin_{tag}_rows"] = r
            z[f"marlin_{tag}_x"] = np.ascontiguousarray(z[f"marlin_{tag}_x"][r])
            z[f"marlin_{tag}_y"] = np.ascontiguousarray(z[f"marlin_{tag}_y"][r])
    return z


np.savez_compressed(sys.argv[1], **sample(out))
print("wrote", sys.argv[1], "with", len(out), "arrays")
