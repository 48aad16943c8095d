"""Dev (GPU box): bring-up of csrc/prefill_attn_tc.cu against csrc/prefill_attn.cu (same entry point, knob-selected)."""
import ctypes, os, sys, itertools
import torch
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
import __graft_entry__ as g
g.load_package()
from mistralrs_b200 import lib, paged_attn
dev = torch.device("cuda:0")
L = lib()


def run(q, k, v, scale, causal, cu=None, enable=1, lbo=0, sbo=0):
    L.mrs_prefill_attn_tc_debug(ctypes.c_int32(enable), ctypes.c_uint32(lbo), ctypes.c_uint32(sbo))
    out = paged_attn.prefill_attention(q, k, v, scale, causal=causal, cu_seqlens=cu) if cu is not None else paged_attn.prefill_attention(q, k, v, scale, causal=causal)
    torch.cuda.synchronize()
    return out


def case(T, H, KVH, dt, causal, cu=None, seed=0, **kn):
    gen = torch.Generator(device=dev).manual_seed(seed)
    q = torch.randn(T, H, 128, device=dev, generator=gen).to(dt)
    k = torch.randn(T, KVH, 128, device=dev, generator=gen).to(dt)
    v = torch.randn(T, KVH, 128, device=dev, generator=gen).to(dt)
    ref = run(q, k, v, 128 ** -0.5, causal, cu, enable=0).float()
    got = run(q, k, v, 128 ** -0.5, causal, cu, enable=1, **kn).float()
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    bad = int((~torch.isfinite(got)).sum().item())
    return err, bad


import inspect
print("prefill_attention signature:", inspect.signature(paged_attn.prefill_attention))
variants = [(16384, 1024), (1024, 16384), (16, 1024), (1024, 1024), (2048, 1024), (16384, 2048)]
ok_variant = None
for lbo, sbo in variants:
    e, bad = case(256, 4, 2, torch.bfloat16, True, lbo=lbo, sbo=sbo)
    print(f"V descriptor lbo={lbo} sbo={sbo}: rel err {e:.3e} non-finite {bad}", flush=True)
    if e < 2e-2 and bad == 0 and ok_variant is None:
        ok_variant = (lbo, sbo)
print("first matching variant:", ok_variant, flush=True)
if ok_variant:
    lbo, sbo = ok_variant
    cu = torch.tensor([0, 200, 517, 900], dtype=torch.int32, device=dev)
    for name, args in (("T=300 causal bf16", dict(T=300, H=8, KVH=2, dt=torch.bfloat16, causal=True)),
                       ("T=1000 non-causal f16", dict(T=1000, H=4, KVH=4, dt=torch.float16, causal=False)),
                       ("var-len 3 seqs causal bf16", dict(T=900, H=8, KVH=8, dt=torch.bfloat16, causal=True, cu=cu)),
                       ("T=4096 H=32 KVH=8 causal bf16", dict(T=4096, H=32, KVH=8, dt=torch.bfloat16, causal=True))):
        e, bad = case(lbo=lbo, sbo=sbo, **args)
        print(f"{name}: rel err vs mma.sync kernel {e:.3e}, non-finite {bad}", flush=True)
    # timing
    T, H, KVH = 4096, 32, 8
    q = torch.randn(T, H, 128, device=dev).to(torch.bfloat16); k = torch.randn(T, KVH, 128, device=dev).to(torch.bfloat16); v = torch.randn(T, KVH, 128, device=dev).to(torch.bfloat16)
    for en in (0, 1):
        L.mrs_prefill_attn_tc_debug(ctypes.c_int32(en), ctypes.c_uint32(lbo), ctypes.c_uint32(sbo))
        for _ in range(3): paged_attn.prefill_attention(q, k, v, 128 ** -0.5)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10): paged_attn.prefill_attention(q, k, v, 128 ** -0.5)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        fl = 4.0 * T * T * 128 * H / 2
        print(f"{'wgmma' if en else 'mma.sync'}: {ms*1e3:8.1f} us per layer-call  {fl/ms/1e9:7.1f} TFLOP/s (causal flops)", flush=True)
