"""Pins the CPU oracle (no GPU needed):
  * block decoders vs gguf-py 0.19.0 (tests/golden/gguf_dequant.npz, make_gguf_golden.py) — bit-exact;
  * Q8_1 quantiser, MMVQ arithmetic, fused GLU, RoPE, add_rms_norm, KV-cache scatter and paged
    attention vs OUTPUTS OF THE UNMODIFIED REFERENCE KERNELS compiled from the reference sources and
    run on an H100 (tests/golden/ref_golden.npz, make_ref_golden.py)."""
import os

import numpy as np
import pytest

import oracle

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TYPES = ["q4_0", "q4_1", "q5_0", "q5_1", "q8_0", "q2_k", "q3_k", "q4_k", "q5_k", "q6_k"]


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(G, "ref_golden.npz"))


def bf16_ulp(x):
    x = np.abs(np.asarray(x, dtype=np.float32)).clip(1e-30)
    return np.exp2(np.floor(np.log2(x)) - 7)


@pytest.mark.parametrize("t", TYPES)
def test_block_decoders_match_gguf_py(t):
    z = np.load(os.path.join(G, "gguf_dequant.npz"))
    got = oracle.dequantize(t, z[f"{t}_blocks"])
    assert np.array_equal(got, z[f"{t}_deq"])
    try:  # live cross-check when the package is importable
        from gguf import GGMLQuantizationType as T, quants
        live = quants.dequantize(z[f"{t}_blocks"], getattr(T, t.upper())).reshape(-1).astype(np.float32)
        assert np.array_equal(got, live)
    except ImportError:
        pass


def test_q8_1_quantiser_vs_reference_kernel(ref):
    want = ref["q8_1_bytes"].reshape(-1, 36)
    got, _ = oracle.quantize_q8_1(ref["mmvq_x"], 1024)
    got = got.reshape(-1, 36)
    # d and the butterfly sum (half2 header): bit-exact
    assert np.array_equal(got[:, :4], want[:, :4])
    dq = np.abs(got[:, 4:].view(np.int8).astype(int) - want[:, 4:].view(np.int8).astype(int))
    # the reference divides with --use_fast_math: an exact .5 tie may round the other way
    assert dq.max() <= 1 and (dq != 0).mean() < 1e-3


@pytest.mark.parametrize("t", TYPES)
def test_mmvq_arithmetic_vs_reference_kernel(ref, t):
    K, B = 1024, 2
    N = ref[f"mmvq_{t}_y"].shape[1]   # a sample of the reference's output columns (column n uses weight row n)
    want = ref[f"mmvq_{t}_y"]
    got = oracle.mmvq_q8_1(t, ref[f"mmvq_{t}_w"], ref["q8_1_bytes"], K, N, K // 32, B)
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= 3e-6 * scale, (t, np.abs(got - want).max() / scale)
    # fused GLU output (bf16): act(bf16(gate)) * bf16(up)
    up = oracle.mmvq_q8_1(t, ref[f"mmvq_{t}_up"], ref["q8_1_bytes"], K, N, K // 32, B)
    mine = oracle.fused_glu(oracle.round_dtype(got.astype(np.float32), "bf16"), oracle.round_dtype(up.astype(np.float32), "bf16"), 0, "bf16")
    w = ref[f"mmvq_{t}_glu"]
    assert (np.abs(mine - w) <= 2 * bf16_ulp(w) + 1e-30).all()
    assert (mine == w).mean() > 0.9


def test_fused_glu_vs_reference_kernel(ref):
    for act in range(5):
        got = oracle.fused_glu(ref["glu_a"], ref["glu_b"], act, "bf16")
        want = ref[f"glu_out_{act}"]
        # the reference is built with --use_fast_math (approximate exp / div / tanh): allow two
        # ulps of the product, measured at the magnitude of |a*b| where the result cancels to ~0
        tol = 2 * bf16_ulp(np.maximum(np.abs(want), 1e-2 * np.abs(ref["glu_a"] * ref["glu_b"])))
        assert (np.abs(got - want) <= tol + 1e-30).all(), act
        assert (got == want).mean() > 0.9, act


def test_rotary_vs_reference_kernel(ref):
    for neox in (1, 0):
        q, k = oracle.rotary(ref["rope_q"], ref["rope_k"], ref["rope_cos"], ref["rope_sin"], ref["rope_pos"], bool(neox),
                             128, 64, 4, 2, "bf16")
        assert np.array_equal(q, ref[f"rope_q_out_{neox}"]) and np.array_equal(k, ref[f"rope_k_out_{neox}"])


def test_add_rms_norm_vs_reference_kernel(ref):
    s, n = oracle.add_rms_norm(ref["rms_x"], ref["rms_res"], ref["rms_w"], 1e-5, "bf16")
    assert np.array_equal(s, ref["rms_sum"])
    assert (np.abs(n - ref["rms_norm"]) <= bf16_ulp(ref["rms_norm"])).all() and (n == ref["rms_norm"]).mean() > 0.98


def _u16(a):
    return oracle.round_dtype(a, "bf16").view(np.uint32).__rshift__(16).astype(np.uint16)


def test_cache_scatter_vs_reference_kernels(ref):
    KVH, D, BS, NB = 2, 128, 16, 9
    k, v = _u16(ref["pa_k"]), _u16(ref["pa_v"])
    for layout, names in ((0, ("cache_k_vllm", "cache_v_vllm")), (1, ("cache_k_hnd", "cache_v_hnd"))):
        kc = np.zeros(NB * KVH * D * BS, dtype=np.uint16); vc = np.zeros_like(kc)
        oracle.reshape_and_cache(k, v, kc, vc, ref["pa_slots"], KVH, D, BS, 8, layout)
        assert np.array_equal(kc, ref[names[0]]) and np.array_equal(vc, ref[names[1]])


def test_paged_attention_vs_reference_kernels(ref):
    KVH, D, BS = 2, 128, 16
    scale = 1.0 / np.sqrt(D)
    for layout, kn, vn, on in ((0, "cache_k_vllm", "cache_v_vllm", "pa_out_v1"), (1, "cache_k_hnd", "cache_v_hnd", "fi_out")):
        got = oracle.paged_attention(ref["pa_q"], ref[kn], ref[vn], ref["pa_tables"], ref["pa_ctx"], KVH, D, BS, scale, layout, "bf16")
        want = ref[on]
        assert np.abs(got - want).max() <= 2.5 * 2.0 ** -8 * np.abs(want).max(), (on, np.abs(got - want).max())


# ---- round 2: the reference kernels' outputs for MMQ, Marlin and the paged-attention variants pin the oracle too ----
def _need(ref, key):
    if key not in ref.files:
        pytest.skip(f"tests/golden/ref_golden.npz has no `{key}`")


@pytest.mark.parametrize("t", ["q4_k", "q6_k", "q8_0"])
def test_exact_product_vs_reference_mmq_kernel(ref, t):
    """`oracle.matmul_exact` (f64 sum of dequantised weights x activations: the target of our prefill GEMMs) against
    the reference's own MMQ kernels (`launch_mmq_quantize_q8_1_*` + `launch_mmq_gguf_<q>`, int8 activations): they may
    differ by the reference's activation-quantisation noise only (its self-consistency bound, fast_mmq.rs:1583-1703)."""
    _need(ref, f"mmq_{t}_y")
    N, K = ref[f"mmq_{t}_y"].shape[1], 1024   # a sample of the reference's rows and columns (output row m uses input row m)
    exact = oracle.matmul_exact(t, ref[f"mmq_{t}_w"], ref["mmq_x"], K, N)
    want = ref[f"mmq_{t}_y"]
    scale = np.abs(exact).max()
    assert np.abs(want - exact).max() <= 2e-2 * scale
    assert np.abs(want - exact).mean() <= 3e-3 * scale


@pytest.mark.parametrize("tag", ["m1", "m32", "m300"])
def test_gptq_oracle_vs_reference_marlin_kernel(ref, tag):
    """oracle/gptq.py (w = f16((q - 8) * s), f64 product) against `gptq_marlin_repack` + `marlin_gptq_4bit_f16` of the
    reference on the same checkpoint tensors: accumulation order + one f16 output rounding apart."""
    from oracle import gptq as og
    _need(ref, f"marlin_{tag}_y")
    assert int(ref[f"marlin_{tag}_rc"]) == 0
    x, qw, sc, want = ref[f"marlin_{tag}_x"], ref[f"marlin_{tag}_qweight"], ref[f"marlin_{tag}_scales"], ref[f"marlin_{tag}_y"]
    got = og.gemm(x, og.dequant_gptq(qw, sc, None, 128))
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= 2.0 ** -10 * scale + 1e-6, float(np.abs(got - want).max() / scale)


@pytest.mark.parametrize("name", ["plain", "alibi", "softcap", "sinks"])
def test_paged_attention_variants_vs_reference_kernel(ref, name):
    """oracle/paged_attn_np.py (ALiBi with the reference's unsigned wrap, soft-capping, sinks) against
    `paged_attention_v1` of the reference (pagedattention.cuh:270-345)."""
    from oracle import paged_attn_np
    key = "pa_out_v1" if name == "plain" else f"pa_out_v1_{name}"
    _need(ref, key)
    KVH, D, BS = 2, 128, 16
    got = paged_attn_np.paged_attention_v1(ref["pa_q"], ref["pa_k"], ref["pa_v"], ref["pa_slots"], ref["pa_tables"], ref["pa_ctx"], KVH, D,
                                           BS, 1.0 / np.sqrt(D), "bf16", softcapping=30.0 if name == "softcap" else 1.0,
                                           alibi_slopes=ref["pa_alibi"] if name == "alibi" else None,
                                           sinks=ref["pa_sinks"] if name == "sinks" else None)
    want = ref[key]
    assert np.abs(got - want).max() <= 2.5 * 2.0 ** -8 * np.abs(want).max(), float(np.abs(got - want).max())
