"""Product kernels vs the stored outputs of the UNMODIFIED reference kernels
(tests/golden/ref_golden.npz) on the same inputs, through the C ABI."""
import ctypes
import os

import numpy as np
import pytest
import torch

from mistralrs_b200 import kv_index, lib, ops, paged_attn, quant
from util import to_dev

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TYPES = ["q4_0", "q4_1", "q5_0", "q5_1", "q8_0", "q2_k", "q3_k", "q4_k", "q5_k", "q6_k"]


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(G, "ref_golden.npz"))


def bf16_ulp(x):
    x = np.abs(np.asarray(x, dtype=np.float32)).clip(1e-30)
    return np.exp2(np.floor(np.log2(x)) - 7)


def test_q8_1_bytes_identical(cuda, ref):
    got = quant.quantize_q8_1(to_dev(ref["mmvq_x"], cuda, "bf16"), 1024).cpu().numpy()
    assert np.array_equal(got, ref["q8_1_bytes"])   # same approximate divisions -> bit-identical


@pytest.mark.parametrize("t", TYPES)
def test_mmvq_plain_and_glu(cuda, ref, t):
    K, B = 1024, 2
    N = ref[f"mmvq_{t}_y"].shape[1]
    w = quant.QTensor(to_dev(ref[f"mmvq_{t}_w"].reshape(-1), cuda), t, (N, K))
    up = quant.QTensor(to_dev(ref[f"mmvq_{t}_up"].reshape(-1), cuda), t, (N, K))
    y = quant.plain(w, to_dev(ref["mmvq_x"], cuda, "f32") if False else to_dev(ref["mmvq_x"], cuda, "bf16").float()).cpu().numpy()
    want = ref[f"mmvq_{t}_y"]
    assert np.abs(y - want).max() <= 3e-6 * np.abs(want).max()
    g = quant.fused_glu(w, up, to_dev(ref["mmvq_x"], cuda, "bf16"), quant.GluActivationType.Silu).float().cpu().numpy()
    wg = ref[f"mmvq_{t}_glu"]
    assert (np.abs(g - wg) <= 2 * bf16_ulp(wg) + 1e-30).all() and (g == wg).mean() > 0.95


def test_fused_glu_elementwise(cuda, ref):
    for act in range(5):
        got = ops.fused_glu(to_dev(ref["glu_a"], cuda, "bf16"), to_dev(ref["glu_b"], cuda, "bf16"), act).float().cpu().numpy()
        want = ref[f"glu_out_{act}"]
        # same fast-math intrinsics as the reference build -> bit-identical (a stray ulp is tolerated)
        assert (np.abs(got - want) <= bf16_ulp(np.maximum(np.abs(want), 1e-2 * np.abs(ref["glu_a"] * ref["glu_b"])))).all(), act
        assert (got == want).mean() > 0.999, act


def test_rotary_bit_identical(cuda, ref):
    for neox in (1, 0):
        q = to_dev(ref["rope_q"], cuda, "bf16").reshape(5, 4, 128).clone()
        k = to_dev(ref["rope_k"], cuda, "bf16").reshape(5, 2, 128).clone()
        ops.apply_rotary_qk(q, k, to_dev(ref["rope_cos"], cuda, "bf16"), to_dev(ref["rope_sin"], cuda, "bf16"),
                            torch.from_numpy(ref["rope_pos"].astype(np.int32)).to(cuda), is_neox=bool(neox))
        assert np.array_equal(q.float().cpu().numpy().reshape(5, -1), ref[f"rope_q_out_{neox}"])
        assert np.array_equal(k.float().cpu().numpy().reshape(5, -1), ref[f"rope_k_out_{neox}"])


def test_add_rms_norm(cuda, ref):
    s, n = ops.add_rms_norm(to_dev(ref["rms_x"], cuda, "bf16"), to_dev(ref["rms_res"], cuda, "bf16"), to_dev(ref["rms_w"], cuda, "bf16"), 1e-5)
    assert np.array_equal(s.float().cpu().numpy(), ref["rms_sum"])
    n = n.float().cpu().numpy()
    assert (np.abs(n - ref["rms_norm"]) <= bf16_ulp(ref["rms_norm"])).all() and (n == ref["rms_norm"]).mean() > 0.98


def test_cache_and_attention(cuda, ref):
    KVH, D, BS, NB, H, S = 2, 128, 16, 9, 8, 2
    k = to_dev(ref["pa_k"], cuda, "bf16").reshape(-1, KVH, D)
    v = to_dev(ref["pa_v"], cuda, "bf16").reshape(-1, KVH, D)
    slots = torch.from_numpy(ref["pa_slots"]).to(cuda)
    kc = torch.zeros(NB, KVH, D // 8, BS, 8, dtype=torch.bfloat16, device=cuda)
    vc = torch.zeros(NB, KVH, D, BS, dtype=torch.bfloat16, device=cuda)
    paged_attn.reshape_and_cache(k, v, None, None, kc, vc, slots)
    u16 = lambda t: t.view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)
    assert np.array_equal(u16(kc), ref["cache_k_vllm"]) and np.array_equal(u16(vc), ref["cache_v_vllm"])
    kh = torch.zeros(NB, KVH, BS, D, dtype=torch.bfloat16, device=cuda)
    vh = torch.zeros_like(kh)
    paged_attn.reshape_and_cache_flashinfer(k, v, kh, vh, slots)
    assert np.array_equal(u16(kh), ref["cache_k_hnd"]) and np.array_equal(u16(vh), ref["cache_v_hnd"])
    q = to_dev(ref["pa_q"], cuda, "bf16")
    scale = 1.0 / np.sqrt(D)
    ctx = ref["pa_ctx"].tolist()
    o1 = paged_attn.paged_attention(q, None, None, kc, vc, to_dev(ref["pa_tables"], cuda), to_dev(ref["pa_ctx"], cuda), None, max(ctx), scale)
    want = ref["pa_out_v1"]
    assert np.abs(o1.float().cpu().numpy() - want).max() <= 2.5 * 2.0 ** -8 * np.abs(want).max()
    tables = [ref["pa_tables"][0][:3].tolist(), ref["pa_tables"][1][:5].tolist()]
    indptr, indices, last = kv_index.make_paged_kv_tensors(tables, ctx, BS, 8)
    req, tile, oind, chunk, mask = kv_index.make_paged_kv_decode_tensors(tables, ctx, BS, None, 2)
    d = lambda a: to_dev(np.ascontiguousarray(a), cuda)
    o2 = paged_attn.flashinfer_decode(q, kh, vh, d(indptr), d(indices), d(last), d(req), d(tile), d(oind), d(chunk), d(mask), scale)
    want = ref["fi_out"]
    assert np.abs(o2.float().cpu().numpy() - want).max() <= 2.5 * 2.0 ** -8 * np.abs(want).max()


def _need(ref, key):
    if key not in ref.files:
        pytest.skip(f"tests/golden/ref_golden.npz has no `{key}` (regenerate with tests/golden/make_ref_golden.py)")


@pytest.mark.parametrize("t", ["q4_k", "q6_k", "q8_0"])
def test_prefill_gemm_vs_reference_mmq(cuda, ref, t):
    """`mrs_mmq_gguf` (bf16 activations x dequantised weights on wgmma) against the output of the
    reference's own MMQ kernels (`launch_mmq_quantize_q8_1_*` + `launch_mmq_gguf_<q>`, int8
    activations).  The two differ by the reference's activation quantisation noise (its own
    self-consistency bound is 5e-3 relative, fast_mmq.rs:1583-1703); both must sit inside that
    envelope of each other, and ours must be the closer one to the exact product."""
    import oracle
    from mistralrs_b200 import mmq
    _need(ref, f"mmq_{t}_y")
    # the stored vectors are a sample of the reference's 64 x 256 product: rows `mmq_rows` of x and y, the first weight
    # rows; the other token rows of the 64-token launch are zero
    M, K = 64, 1024
    wb, x, want, rows = ref[f"mmq_{t}_w"], ref["mmq_x"], ref[f"mmq_{t}_y"], ref["mmq_rows"]
    N = want.shape[1]
    xf = np.zeros((M, K), np.float32)
    xf[rows] = x
    w = quant.QTensor(to_dev(wb.reshape(-1), cuda), t, (N, K))
    got = mmq.forward(w, to_dev(xf, cuda, "bf16")).float().cpu().numpy()[rows]
    exact = oracle.matmul_exact(t, wb, x, K, N)
    scale = np.abs(exact).max()
    e_ref, e_ours = np.abs(want - exact).max() / scale, np.abs(got - exact).max() / scale
    assert np.abs(got - want).max() <= 2e-2 * scale, (e_ref, e_ours)
    assert e_ours <= 2.0 ** -7 and e_ours <= e_ref + 2.0 ** -8, (e_ref, e_ours)   # one bf16 output rounding vs int8 activations


@pytest.mark.parametrize("tag,M", [("m32", 32), ("m1", 1), ("m300", 300)])
def test_gptq_vs_reference_marlin(cuda, ref, tag, M):
    """GPTQ int4 (sym, g128) through `GptqLayer` against `gptq_marlin_repack` + `marlin_gptq_4bit_f16`
    of the reference on the same checkpoint tensors: same arithmetic class (w = f16((q-8)*s), f16
    MMA, f32 accumulate), so agreement is limited by accumulation order and one f16 output rounding."""
    from mistralrs_b200 import gptq
    _need(ref, f"marlin_{tag}_y")
    assert int(ref[f"marlin_{tag}_rc"]) == 0
    x, qw, sc, want = ref[f"marlin_{tag}_x"], ref[f"marlin_{tag}_qweight"], ref[f"marlin_{tag}_scales"], ref[f"marlin_{tag}_y"]
    rows = ref[f"marlin_{tag}_rows"] if f"marlin_{tag}_rows" in ref.files else np.arange(M)
    xf = np.zeros((M, x.shape[1]), np.float16)   # stored: a sample of the token rows; the others are zero
    xf[rows] = x
    layer = gptq.GptqLayer(torch.from_numpy(qw).to(cuda), torch.from_numpy(sc).to(cuda), group_size=128)
    got = layer.forward_raw(torch.from_numpy(xf).to(cuda)).float().cpu().numpy()[rows]
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= 2.0 ** -10 * scale + 1e-6, float(np.abs(got - want).max() / scale)


@pytest.mark.parametrize("name", ["alibi", "softcap", "sinks"])
def test_paged_attention_v1_variants(cuda, ref, name):
    """ALiBi slopes, logit soft-capping and attention sinks of `paged_attention_v1` against the
    reference kernel's outputs (pagedattention.cuh:189-420)."""
    _need(ref, f"pa_out_v1_{name}")
    KVH, D, BS, NB, H, S = 2, 128, 16, 9, 8, 2
    k = to_dev(ref["pa_k"], cuda, "bf16").reshape(-1, KVH, D)
    v = to_dev(ref["pa_v"], cuda, "bf16").reshape(-1, KVH, D)
    kc = torch.zeros(NB, KVH, D // 8, BS, 8, dtype=torch.bfloat16, device=cuda)
    vc = torch.zeros(NB, KVH, D, BS, dtype=torch.bfloat16, device=cuda)
    paged_attn.reshape_and_cache(k, v, None, None, kc, vc, torch.from_numpy(ref["pa_slots"]).to(cuda))
    q = to_dev(ref["pa_q"], cuda, "bf16")
    ctx = ref["pa_ctx"].tolist()
    al = torch.from_numpy(ref["pa_alibi"]).to(cuda) if name == "alibi" else None
    sk = torch.from_numpy(ref["pa_sinks"]).to(cuda) if name == "sinks" else None
    o = paged_attn.paged_attention(q, None, None, kc, vc, to_dev(ref["pa_tables"], cuda), to_dev(ref["pa_ctx"], cuda), al,
                                   max(ctx), 1.0 / np.sqrt(D), softcapping=30.0 if name == "softcap" else 1.0, sinks=sk)
    want = ref[f"pa_out_v1_{name}"]
    assert np.abs(o.float().cpu().numpy() - want).max() <= 2.5 * 2.0 ** -8 * np.abs(want).max()
