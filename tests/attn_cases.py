"""Score-shaped attention inputs, float64 references, an error bound computed from the inputs, and numpy emulations of
online-softmax attention (one correct, several with a known bug), shared by tests/test_attn_scores_host.py and
tests/test_attn_scores_gpu.py.

Why shaped scores: with q, k ~ N(0, 1) and scale 1/sqrt(D) every score is O(1) and softmax is nearly flat, so a kernel
that never subtracts its running max, never raises it after the first tile, lets masked positions into it, or merges
split-KV partials against the wrong max still gives the right answer (softmax does not change when every score moves by
the same amount).  The profiles below put the max where those bugs change the result:

  normal      q, k ~ N(0, 1) (the control; what the older tests use)
  ramp_up     scores rise by 120 nats over the visible keys: every tile raises the running max
  ramp_down   the max is in the first tile; later tiles' probabilities all flush to zero
  sink        key 0 sits 12 above an N(0, 1) background
  needle      one key sits 40 above all others: the output is that key's V row to within rounding
  shift+100   every score + 100 nats (e^s overflows f32 without max subtraction)
  shift-100   every score - 100 nats (e^s underflows with a running max that starts at 0)
  poison      every position the query must not see scores 200 above every visible key, with a V row of large finite
              values (a masked score in the max flushes every visible probability to zero)

Every KV head gets one unit direction u shared by its query heads: q_h = a u + small noise, k_j = c_j u + noise, so that
scale * q_h . k_j = target_j + N(0, 1).  Elements stay well inside f16 range (|q| ~ 4, |k| < 40).
"""
import numpy as np
import torch

UNIT = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11, "f32": 2.0 ** -24}
SUBNORMAL = {"bf16": 2.0 ** -133, "f16": 2.0 ** -24, "f32": 2.0 ** -149}   # smallest positive value of each dtype
TORCH_DT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
PROFILES = ("normal", "ramp_up", "ramp_down", "sink", "needle", "shift+100", "shift-100", "poison")
SCORE_GAIN = 4.0      # scale * a: the query's length along u, in nats per unit of c
POISON_V = 1000.0


def round_to(x, dt):
    """float32 copy of x rounded through dtype dt ('bf16' | 'f16' | 'f32')"""
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    return t.to(TORCH_DT[dt]).float().numpy()


def low_freq_direction(rng, D):
    """A unit vector on the lowest RoPE frequencies (both NeoX and interleaved pairings), so rotating it by a few
    positions barely moves it: the rows of one verify step see nearly the same scores."""
    u = np.zeros(D)
    dims = np.r_[D // 2 - 8:D // 2, D - 16:D]
    u[dims] = rng.standard_normal(len(dims))
    return u / np.linalg.norm(u)


def make_queries(rng, profile, H, KVH, D, scale, low_freq=False):
    """q [H, D] float32 (not rounded).  normal: N(0, 1); otherwise a u_g + noise for the heads of KV head g."""
    if profile == "normal":
        return rng.standard_normal((H, D)).astype(np.float32)
    a = SCORE_GAIN / scale
    q = np.empty((H, D))
    g = H // KVH
    for kvh in range(KVH):
        if low_freq:
            u = low_freq_direction(rng, D)
        else:
            u = rng.standard_normal(D); u /= np.linalg.norm(u)
        q[kvh * g:(kvh + 1) * g] = a * u + 0.1 * rng.standard_normal((g, D))
    return q.astype(np.float32)


def target_scores(profile, n, visible, needle=None):
    """Target scaled score (nats) of each of n keys before the N(0, 1) noise.  visible: bool [n], the keys the query
    sees; under 'poison' every other key scores 200 over the top visible target (plus the noise margin)."""
    t = np.zeros(n)
    idx = np.flatnonzero(visible)
    if profile == "ramp_up":
        t[idx] = np.linspace(-60.0, 60.0, len(idx))
    elif profile == "ramp_down":
        t[idx] = np.linspace(60.0, -60.0, len(idx))
    elif profile == "sink":
        t[0] = 12.0
    elif profile == "needle":
        t[needle] = 45.0
    elif profile == "shift+100":
        t += 100.0
    elif profile == "shift-100":
        t -= 100.0
    elif profile == "poison":
        t[~visible] = (t[idx].max() if len(idx) else 0.0) + 210.0
    return t


def make_keys(rng, profile, q, KVH, targets, scale):
    """Keys [n, KVH, D] float32 for queries q [H, D] (as the kernel sees them, i.e. after RoPE) so that scale * q_h . k_j
    = targets[j] + N(0, 1) for every head of the group.  normal: N(0, 1) keys."""
    H, D = q.shape
    n = len(targets)
    if profile == "normal":
        return rng.standard_normal((n, KVH, D)).astype(np.float32)
    g = H // KVH
    k = np.empty((n, KVH, D))
    for kvh in range(KVH):
        mean = q[kvh * g:(kvh + 1) * g].astype(np.float64).mean(0)
        a = np.linalg.norm(mean)
        u = mean / a
        # noise xi ~ N(0, 1 / (scale a)^2) per element: scale a (u . xi) ~ N(0, 1) nats
        k[:, kvh] = (np.asarray(targets)[:, None] * u + rng.standard_normal((n, D))) / (scale * a)
    return k.astype(np.float32)


def make_values(rng, n, KVH, D, visible=None, poison=False, big=POISON_V):
    """V rows N(0, 1); under poison, rows nobody may see hold +-big (finite)"""
    v = rng.standard_normal((n, KVH, D)).astype(np.float32)
    if poison and visible is not None:
        hid = ~visible
        v[hid] = big * np.sign(rng.standard_normal((int(hid.sum()), KVH, D))).astype(np.float32)
    return v


def poison_rows(rng, q, KVH, top, scale, big=POISON_V):
    """One key and one value row per KV head for cache slots nobody owns: score top + 200 for every head of the group"""
    k = make_keys(rng, "poison", q, KVH, np.array([top + 210.0]), scale)[0]
    v = big * np.sign(rng.standard_normal(k.shape)).astype(np.float32)
    return k, v


# ---------------------------------------------------------------- float64 reference and error bound
def reference(q, k, v, scale, mask, softcap=None, sinks=None):
    """fp64 attention of query rows q [R, H, D] over k / v [n, KVH, D]; mask bool [R, n] (True = visible); sinks [H]
    logits that join the softmax denominator only.  Returns (o [R, H, D], stats) with the sums tolerance() needs:
    s1 = sum_j p_j |v_j|; s2 = sum_j p_j |v_j - o|; flush = sum of p_j |v_j| over p_j < e^-80; qk [R, H] = scale * max
    over visible j of sum_i |q_i k_ji|."""
    R, H, D = q.shape
    KVH = k.shape[1]
    g = H // KVH
    qd, kd, vd = q.astype(np.float64), k.astype(np.float64), v.astype(np.float64)
    o, s1, s2, fl = (np.zeros((R, H, D)) for _ in range(4))
    qk = np.zeros((R, H))
    for h in range(H):
        kh, vh = kd[:, h // g], vd[:, h // g]
        s = (qd[:, h] @ kh.T) * scale
        if softcap:
            s = softcap * np.tanh(s / softcap)
        s = np.where(mask, s, -np.inf)
        m = s.max(1, keepdims=True)
        if sinks is not None:
            m = np.maximum(m, sinks[h])
        p = np.exp(s - m)
        p /= p.sum(1, keepdims=True) + (np.exp(sinks[h] - m) if sinks is not None else 0.0)
        o[:, h] = p @ vh
        s1[:, h] = p @ np.abs(vh)
        fl[:, h] = np.where(p < np.exp(-80.0), p, 0.0) @ np.abs(vh)
        for r in range(R):
            nz = p[r] > 0
            s2[r, h] = p[r, nz] @ np.abs(vh[nz] - o[r, h])
        qa = (np.abs(qd[:, h]) @ np.abs(kh).T) * scale
        qk[:, h] = np.where(mask, qa, 0.0).max(1)
    return o, dict(s1=s1, s2=s2, flush=fl, qk=qk)


def tolerance(o, st, dt, n, softcap=None):
    """Element-wise bound on |kernel - fp64| from the inputs alone (st: the sums reference() returns):
        1.25 [ u (2 sum p|v| + |o|) + c sum p|v| + delta sum p|v - o| + 2 s ] + sum_{p < e^-80} p|v|
    u: unit roundoff of dt.  2u: P rounded to dt before the PV product, and split partials stored in dt; u|o|: the output
    rounding.  c = 2^-24 (n/4 + 64): f32 accumulation and rescaling of up to n/8 tokens in one chain, plus the merges.
    delta: absolute error of one scaled score, 2^-21 scale max_j sum_i |q_i k_ji| for the f32 dot product, plus 2^-21 for
    ex2.approx and the log2(e) scaling (and the tanh of a soft-cap).  The last term: probabilities that f32 flushes to
    zero relative to the running max.  s: the smallest subnormal of dt, for an output or partial that underflows."""
    u = UNIT[dt]
    c = 2.0 ** -24 * (n / 4 + 64)
    delta = 2.0 ** -21 * st["qk"] + 2.0 ** -21 * (1.0 + (softcap or 0.0))
    return 1.25 * (u * (2 * st["s1"] + abs(o)) + c * st["s1"] + delta[..., None] * st["s2"] + 2 * SUBNORMAL[dt]) + st["flush"]


def err_ratio(got, want, tol):
    """max |got - want| / tol; inf when got is not finite"""
    got = np.asarray(got, dtype=np.float64)
    if not np.isfinite(got).all():
        return float("inf")
    return float((np.abs(got - want) / tol).max())


# ---------------------------------------------------------------- numpy emulations of a decode kernel
MUTANTS = ("no_max", "max_starts_at_zero", "max_frozen", "max_includes_masked", "merge_max_first_partial",
           "empty_partial_lse_zero", "sink_dropped_in_merge", "sink_in_partials_and_merge", "window_off_by_one")


def emulate(q, k, v, scale, kv_len, dt, tile=64, chunk=None, window_left=None, softcap=None, sinks=None, bug=None):
    """One query row per head, q [H, D], over k / v [n, KVH, D] where rows >= kv_len are loaded but masked (stale rows of
    a last page).  f32 online softmax over `tile`-token tiles; P rounded to dt before PV; with `chunk`, split-KV partials
    of `chunk` tokens stored in dt with an f32 log-sum-exp and merged by lse (sinks join the merge only, as vLLM v2
    does); without, sinks join the final normalisation.  `bug` names one of MUTANTS.  Returns [H, D] in dt (float32)."""
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        return _emulate(q, k, v, scale, kv_len, dt, tile, chunk, window_left, softcap, sinks, bug)


def _emulate(q, k, v, scale, kv_len, dt, tile, chunk, window_left, softcap, sinks, bug):
    H, D = q.shape
    n, KVH = k.shape[0], k.shape[1]
    g = H // KVH
    f32 = np.float32
    kf = np.repeat(k.astype(f32), g, axis=1).transpose(1, 0, 2)      # [H, n, D]
    vf = np.repeat(v.astype(f32), g, axis=1).transpose(1, 0, 2)
    s = np.einsum("hd,hnd->hn", (q.astype(f32) * f32(scale)), kf).astype(f32)
    if softcap:
        s = (f32(softcap) * np.tanh(s / f32(softcap))).astype(f32)
    lo = max(0, kv_len - 1 - window_left) if window_left is not None else 0
    if bug == "window_off_by_one" and window_left is not None:
        lo += 1
    j = np.arange(n)
    live = (j >= lo) & (j < kv_len)
    chunks = [(0, kv_len)] if chunk is None else [(c0, min(kv_len, c0 + chunk)) for c0 in range(0, kv_len, chunk)]
    split = chunk is not None
    parts = []
    for ci, (c0, c1) in enumerate(chunks):
        m = np.full(H, -np.inf if bug not in ("no_max", "max_starts_at_zero") else 0.0, dtype=f32)
        l = np.zeros(H, f32)
        o = np.zeros((H, D), f32)
        hi = c1 if ci < len(chunks) - 1 else max(c1, min(n, -(-c1 // tile) * tile))   # last tile loads past kv_len
        for t0 in range(c0, hi, tile):
            t1 = min(t0 + tile, hi)
            st = s[:, t0:t1]
            vis = live[t0:t1]
            seen = np.where(vis[None], st, -np.inf)
            tmax = (st if bug == "max_includes_masked" else seen).max(1)
            if bug == "no_max" or (bug == "max_frozen" and t0 > c0):
                mn = m
            else:
                mn = np.maximum(m, tmax).astype(f32)
            ok = mn > -np.inf
            corr = np.where(ok, np.exp(m - mn), f32(1)).astype(f32)
            p = np.where(ok[:, None] & vis[None], np.exp(seen - mn[:, None]), f32(0)).astype(f32)
            l = (l * corr + p.sum(1, dtype=f32)).astype(f32)
            pr = round_to(p, dt)
            o = (o * corr[:, None] + np.einsum("ht,htd->hd", pr, vf[:, t0:t1])).astype(f32)
            m = mn
        if bug == "sink_in_partials_and_merge" and sinks is not None and split:
            sk = sinks.astype(f32)
            mn = np.maximum(m, sk)
            l = (l * np.exp(m - mn) + np.exp(sk - mn)).astype(f32)
            o = (o * np.exp(m - mn)[:, None]).astype(f32)
            m = mn
        if not split:
            if sinks is not None:
                sk = sinks.astype(f32)
                mn = np.maximum(m, sk)
                l = (l * np.exp(m - mn) + np.exp(sk - mn)).astype(f32)
                o = (o * np.exp(m - mn)[:, None]).astype(f32)
            return round_to(np.where(l[:, None] > 0, o / l[:, None], 0.0), dt)
        part_o = round_to(np.where(l[:, None] > 0, o / l[:, None], 0.0), dt)
        lse = np.where(l > 0, m + np.log(l), -np.inf if bug != "empty_partial_lse_zero" else 0.0).astype(f32)
        parts.append((part_o, lse))
    lses = np.stack([p[1] for p in parts])               # [P, H]
    M = lses[0] if bug == "merge_max_first_partial" else lses.max(0)
    use_sink = sinks is not None and bug != "sink_dropped_in_merge"
    if use_sink:
        M = np.maximum(M, sinks.astype(f32))
    w = np.where(M > -np.inf, np.exp(lses - M), 0.0).astype(f32)
    W = w.sum(0, dtype=f32) + (np.exp(sinks.astype(f32) - M) if use_sink else 0.0)
    acc = np.einsum("ph,phd->hd", w, np.stack([p[0] for p in parts])).astype(f32)
    return round_to(np.where(W[:, None] > 0, acc / W[:, None], 0.0), dt)


def decode_case(rng, profile, n_ctx, n_rows, H, KVH, D, dt, window_left=None, needle=None):
    """A single-query decode problem with kv_len = n_ctx over n_rows >= n_ctx loaded rows (the rest stale): returns
    q [H, D], k, v [n_rows, KVH, D] rounded to dt, the visible mask [n_rows] and the scale."""
    scale = D ** -0.5
    j = np.arange(n_rows)
    lo = max(0, n_ctx - 1 - window_left) if window_left is not None else 0
    vis = (j >= lo) & (j < n_ctx)
    q = round_to(make_queries(rng, profile, H, KVH, D, scale), dt)
    t = target_scores(profile, n_rows, vis, needle)
    k = round_to(make_keys(rng, profile, q, KVH, t, scale), dt)
    v = round_to(make_values(rng, n_rows, KVH, D, vis, profile == "poison"), dt)
    return q, k, v, vis, scale
