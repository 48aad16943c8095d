"""The error bound of tests/attn_cases.py against numpy emulations of online-softmax decode attention (CPU only).

A correct emulation (f32 online softmax over 64- or 128-token tiles, P rounded to the activation dtype, split-KV
partials stored in it and merged by log-sum-exp) stays within the bound on every score profile and at every plan shape
tests/test_attn_scores_gpu.py runs, so the bound is not tighter than correct arithmetic.  Each emulation with a known
online-softmax bug exceeds it on at least one profile; the printout shows how far each one gets on the N(0, 1) control,
where most of them are within the bound."""
import numpy as np
import pytest

import attn_cases as ac

# (kv_len, loaded rows, tile, chunk): the unsplit and split-KV plans of the GPU file, with the stale rows of a
# 16-token last page, the vLLM v2 partitions (512 tokens) and the prompt kernels' 64 / 128-row tiles
PLANS = [(300, 304, 64, None), (300, 304, 64, 64), (2049, 2064, 64, 256), (1100, 1104, 128, 512),
         (4096, 4096, 128, None), (700, 704, 64, 128)]
H, KVH, D = 8, 2, 128


def _needles(n_ctx, chunk, window_left=None):
    out = {0, 15, 16, n_ctx - 1}
    if chunk:
        out.add(chunk)
    if n_ctx > 512:
        out |= {511, 512}
    if window_left is not None:
        out = {max(0, n_ctx - 1 - window_left)}
    return sorted(j for j in out if j < n_ctx)


def _profiles(n_ctx, chunk, window_left=None):
    for prof in ac.PROFILES:
        if prof == "needle":
            for j in _needles(n_ctx, chunk, window_left):
                yield prof, j
        else:
            yield prof, None


def _ratio(prof, needle, n_ctx, n_rows, tile, chunk, dt, seed, window_left=None, softcap=None, sinks=None, bug=None):
    rng = np.random.default_rng(seed)
    q, k, v, vis, scale = ac.decode_case(rng, prof, n_ctx, n_rows, H, KVH, D, dt, window_left, needle)
    o, st = ac.reference(q[None], k, v, scale, vis[None], softcap, sinks)
    tol = ac.tolerance(o, st, dt, n_ctx, softcap)[0]
    got = ac.emulate(q, k, v, scale, n_ctx, dt, tile, chunk, window_left, softcap, sinks, bug)
    return ac.err_ratio(got, o[0], tol)


@pytest.mark.parametrize("dt", ["bf16", "f16"])
@pytest.mark.parametrize("plan", PLANS, ids=lambda p: "-".join(map(str, p)))
def test_correct_emulation_is_within_tolerance(plan, dt):
    n_ctx, n_rows, tile, chunk = plan
    worst = 0.0
    for i, (prof, needle) in enumerate(_profiles(n_ctx, chunk)):
        r = _ratio(prof, needle, n_ctx, n_rows, tile, chunk, dt, seed=i)
        assert r <= 1.0, (prof, needle, r)
        worst = max(worst, r)
    # window, soft-cap and sinks in the same plan (sinks as vLLM v2 applies them: in the merge only)
    for i, (prof, needle) in enumerate(_profiles(n_ctx, chunk, 100)):
        r = _ratio(prof, needle, n_ctx, n_rows, tile, chunk, dt, seed=100 + i, window_left=100)
        assert r <= 1.0, ("window", prof, needle, r)
        worst = max(worst, r)
    for prof in ("normal", "ramp_up", "shift+100", "poison"):
        r = _ratio(prof, None, n_ctx, n_rows, tile, chunk, dt, seed=200, softcap=30.0)
        assert r <= 1.0, ("softcap", prof, r)
        for sinks in (np.full(H, 3.0), np.full(H, 80.0), np.full(H, 200.0)):
            r = _ratio(prof, None, n_ctx, n_rows, tile, chunk, dt, seed=300, sinks=sinks)
            assert r <= 1.0, ("sinks", prof, sinks[0], r)
            worst = max(worst, r)
    print(f"\n{plan} {dt}: worst err/tol {worst:.3f}")


# each bug with the plan that can show it: (mutant, kv_len, rows, tile, chunk, window_left, sinks)
MUTANT_CASES = [
    ("no_max", 300, 304, 64, None, None, None),
    ("max_starts_at_zero", 300, 304, 64, None, None, None),
    ("max_frozen", 700, 704, 64, None, None, None),
    ("max_includes_masked", 300, 304, 64, None, 100, None),
    ("merge_max_first_partial", 2049, 2064, 64, 256, None, None),
    ("empty_partial_lse_zero", 700, 704, 64, 128, 100, None),
    ("sink_dropped_in_merge", 1100, 1104, 128, 512, None, "sink"),
    ("sink_in_partials_and_merge", 1100, 1104, 128, 512, None, "sink"),
    ("window_off_by_one", 700, 704, 64, 128, 100, None),
]


@pytest.mark.parametrize("case", MUTANT_CASES, ids=lambda c: c[0])
def test_each_bug_fails_on_a_shaped_profile(case):
    bug, n_ctx, n_rows, tile, chunk, window_left, sinks = case
    assert bug in ac.MUTANTS
    dt = "bf16"
    ratios = {}
    for i, (prof, needle) in enumerate(_profiles(n_ctx, chunk, window_left)):
        # the sink logit sits near the visible scores of each profile, so dropping or doubling it shows
        sk = None
        if sinks:
            top = {"shift+100": 100.0, "shift-100": -100.0, "ramp_up": 60.0, "ramp_down": 60.0, "needle": 45.0}.get(prof, 3.0)
            sk = np.full(H, top)
        key = prof if needle is None else f"needle@{needle}"
        ratios[key] = _ratio(prof, needle, n_ctx, n_rows, tile, chunk, dt, seed=i, window_left=window_left, sinks=sk, bug=bug)
    shaped = {k: r for k, r in ratios.items() if k != "normal"}
    caught = sorted(k for k, r in shaped.items() if r > 1.0)
    print(f"\n{bug}: err/tol on normal {ratios['normal']:.3g}; caught by {caught}")
    assert caught, ratios
