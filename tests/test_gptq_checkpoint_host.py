"""GPTQ / AWQ checkpoint directories on the host (gptq_model.GptqCheckpoint, GptqWeights.from_checkpoint before any
device work): config parsing from config.json's `quantization_config` and from quantize_config.json, one shard and
two shards with an index, every rejection naming its key or tensor, and the act-order transform of the stack's
tensors against the checkpoint's own product (oracle/gptq.py dequantisation, numpy f64).

The checkpoint writer and the seeded checkpoint generator below are also used by tests/test_gptq_checkpoint_gpu.py and
scripts/bench_gptq_checkpoint.py."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import gptq as og
from mistralrs_b200 import gptq_model as G

_ST = {np.dtype(np.int32): "I32", np.dtype(np.float16): "F16", np.dtype(np.float32): "F32", np.dtype(np.uint16): "BF16"}


def write_safetensors(path, tensors):
    """name -> numpy array (uint16 arrays are written as BF16); tensors back to back in name order"""
    header, off = {}, 0
    names = sorted(tensors)
    for n in names:
        a = tensors[n]
        header[n] = {"dtype": _ST[a.dtype], "shape": list(a.shape), "data_offsets": [off, off + a.nbytes]}
        off += a.nbytes
    h = json.dumps(header).encode()
    h += b" " * (-len(h) % 8)
    with open(path, "wb") as f:
        f.write(len(h).to_bytes(8, "little"))
        f.write(h)
        for n in names:
            f.write(np.ascontiguousarray(tensors[n]).tobytes())


def write_checkpoint(d, config, tensors, shards=1, quantize_config=None):
    """a Hugging Face checkpoint directory: config.json (+ quantize_config.json), one model.safetensors or `shards`
    files with model.safetensors.index.json"""
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(config, f)
    if quantize_config is not None:
        with open(os.path.join(d, "quantize_config.json"), "w") as f:
            json.dump(quantize_config, f)
    names = sorted(tensors)
    if shards == 1:
        write_safetensors(os.path.join(d, "model.safetensors"), tensors)
        return d
    files = [f"model-{i + 1:05d}-of-{shards:05d}.safetensors" for i in range(shards)]
    wmap = {n: files[i * shards // len(names)] for i, n in enumerate(names)}
    for fname in files:
        write_safetensors(os.path.join(d, fname), {n: tensors[n] for n in names if wmap[n] == fname})
    with open(os.path.join(d, "model.safetensors.index.json"), "w") as f:
        json.dump({"metadata": {}, "weight_map": wmap}, f)
    return d


def hf_config(cfg, quant, arch="MistralForCausalLM", tied=False, sliding_window=None, rope_scaling=None):
    return {"architectures": [arch], "model_type": "mistral" if arch.startswith("Mistral") else "llama",
            "hidden_size": cfg.hidden, "intermediate_size": cfg.inter, "num_hidden_layers": cfg.n_layers,
            "num_attention_heads": cfg.n_heads, "num_key_value_heads": cfg.n_kv_heads, "head_dim": cfg.head_dim,
            "vocab_size": cfg.vocab, "rms_norm_eps": cfg.rms_eps, "rope_theta": cfg.rope_theta,
            "max_position_embeddings": cfg.max_pos, "sliding_window": sliding_window, "tie_word_embeddings": tied,
            "rope_scaling": rope_scaling, "quantization_config": quant}


def gptq_quant(group, desc_act=False, fmt=None):
    q = {"quant_method": "gptq", "bits": 4, "group_size": group, "sym": True, "desc_act": desc_act}
    if fmt is not None:
        q["checkpoint_format"] = fmt
    return q


def awq_quant(group):
    return {"quant_method": "awq", "bits": 4, "group_size": group, "zero_point": True, "version": "gemm"}


def linear_shapes(cfg):
    nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
    return {"q_proj": (cfg.hidden, nq), "k_proj": (cfg.hidden, nkv), "v_proj": (cfg.hidden, nkv), "o_proj": (nq, cfg.hidden),
            "gate_proj": (cfg.hidden, cfg.inter), "up_proj": (cfg.hidden, cfg.inter), "down_proj": (cfg.inter, cfg.hidden)}


def synth_tensors(cfg, method="gptq", act_order=False, seed=0, fmt=None, tied=False, host=None):
    """seeded checkpoint tensors in Hugging Face names.  GPTQ: uniform nibbles, scales 2^U(-8,-6), symmetric qzeros (7s,
    or 8s for gptq_v2), g_idx k // group or (act_order) a shuffle of it shared by q/k/v and by gate/up.  AWQ: uniform
    nibbles and zero points.  host: a GptqWeights.host of the synthetic model (keep_host=True) to write instead of
    seeded linears / norms / embeddings (natural order, f16)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    G_ = cfg.group_size
    t = {}
    f16 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float16)
    zero = np.uint32(0x88888888 if fmt == "gptq_v2" else 0x77777777)
    for l in range(cfg.n_layers):
        orders = {}
        for name, (K, N) in linear_shapes(cfg).items():
            base = G.GptqCheckpoint.key(l, name)
            if host is not None:
                qw, sc = host[(l, name)]
            elif method == "gptq":
                qw = rng.integers(0, 2 ** 32, size=(K // 8, N), dtype=np.uint32).view(np.int32)
                sc = f16(np.exp2(rng.uniform(-8, -6, size=(K // G_, N))))
            else:
                qw = rng.integers(0, 2 ** 32, size=(K, N // 8), dtype=np.uint32).view(np.int32)
                sc = f16(np.exp2(rng.uniform(-8, -6, size=(K // G_, N))))
            t[f"{base}.qweight"], t[f"{base}.scales"] = qw, sc
            if method == "gptq":
                t[f"{base}.qzeros"] = np.full((K // G_, N // 8), zero, dtype=np.uint32).view(np.int32)
                share = {"k_proj": "q_proj", "v_proj": "q_proj", "up_proj": "gate_proj"}.get(name, name)
                if share not in orders:
                    g = np.arange(K, dtype=np.int32) // G_
                    orders[share] = rng.permutation(g).astype(np.int32) if act_order else g
                t[f"{base}.g_idx"] = orders[share]
            else:
                t[f"{base}.qzeros"] = rng.integers(0, 2 ** 32, size=(K // G_, N // 8), dtype=np.uint32).view(np.int32)
        for key, n in (("attn_norm", "input_layernorm"), ("ffn_norm", "post_attention_layernorm")):
            t[f"model.layers.{l}.{n}.weight"] = f16(host[(l, key)] if host is not None
                                                    else 1.0 + 0.1 * rng.standard_normal(cfg.hidden))
    t["model.norm.weight"] = f16(host[(0, "final_norm")] if host is not None else 1.0 + 0.1 * rng.standard_normal(cfg.hidden))
    t["model.embed_tokens.weight"] = f16(host[(0, "tok_embd")] if host is not None
                                         else 0.5 * rng.standard_normal((cfg.vocab, cfg.hidden)))
    if not tied:
        t["lm_head.weight"] = f16(host[(0, "lm_head")] if host is not None
                                  else 0.05 * rng.standard_normal((cfg.vocab, cfg.hidden)))
    return t


def make_checkpoint(d, cfg, method="gptq", act_order=False, seed=0, shards=1, fmt=None, tied=False, host=None, **cfg_kw):
    quant = gptq_quant(cfg.group_size, act_order, fmt) if method == "gptq" else awq_quant(cfg.group_size)
    return write_checkpoint(d, hf_config(cfg, quant, tied=tied, **cfg_kw),
                            synth_tensors(cfg, method, act_order, seed, fmt, tied, host), shards)


# ---------------------------------------------------------------------------------------------------------------------
TINY = G.GptqConfig.tiny_test


def test_config_from_config_json_one_and_two_shards(tmp_path):
    cfg = TINY()
    for shards in (1, 2):
        d = make_checkpoint(str(tmp_path / f"s{shards}"), cfg, act_order=True, shards=shards, sliding_window=128)
        ck = G.GptqCheckpoint(d)
        c = ck.cfg
        assert (c.hidden, c.inter, c.n_layers, c.n_heads, c.n_kv_heads, c.head_dim, c.vocab) == \
               (cfg.hidden, cfg.inter, cfg.n_layers, cfg.n_heads, cfg.n_kv_heads, cfg.head_dim, cfg.vocab)
        assert c.group_size == 64 and c.rms_eps == cfg.rms_eps and c.rope_theta == cfg.rope_theta
        assert c.sliding_window == 128 and c.max_pos == 128          # capped to the window
        assert ck.method == "gptq" and not ck.tied and len(ck.files) == shards
        assert all(p["qkv"] is not None and p["o"] is not None for p in ck.perms)
        ck.close()
    assert G.GptqCheckpoint(d, max_pos=96).cfg.max_pos == 96
    with pytest.raises(ValueError, match="sliding_window"):
        G.GptqCheckpoint(d, max_pos=256)


def test_config_from_quantize_config_json_tied_and_llama3(tmp_path):
    cfg = TINY()
    t = synth_tensors(cfg, tied=True)
    sc = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
          "original_max_position_embeddings": 64}
    conf = hf_config(cfg, None, arch="LlamaForCausalLM", tied=True, rope_scaling=sc)
    del conf["quantization_config"]
    d = write_checkpoint(str(tmp_path / "q"), conf, t, quantize_config={"bits": 4, "group_size": 64, "desc_act": False,
                                                                       "sym": True})
    ck = G.GptqCheckpoint(d)
    assert ck.tied and ck.cfg.tie_word_embeddings and ck.method == "gptq"
    assert ck.cfg.rope_scaling == {k: sc[k] for k in ("factor", "low_freq_factor", "high_freq_factor",
                                                       "original_max_position_embeddings")}
    assert ck.cfg.max_pos == cfg.max_pos and ck.cfg.sliding_window is None
    emb, head, _ = ck.top()
    assert head is None and emb.shape == (cfg.vocab, cfg.hidden)
    assert all(p == dict(qkv=None, o=None, gate_up=None, down=None) for p in ck.perms)   # natural order: no permutation


def _mutate_config(key, value, quant=False):
    def f(conf, t):
        (conf["quantization_config"] if quant else conf)[key] = value
    return f


def _retype(name, dtype):
    def f(conf, t):
        t[name] = t[name].astype(dtype)
    return f


def _add(name, value):
    def f(conf, t):
        t[name] = value
    return f


def _bad_zero(conf, t):
    z = t["model.layers.1.mlp.up_proj.qzeros"].view(np.uint32).copy()
    z[0, 3] = 0x77777787
    t["model.layers.1.mlp.up_proj.qzeros"] = z.view(np.int32)


def _uneven_groups(conf, t):
    g = t["model.layers.0.self_attn.o_proj.g_idx"].copy()
    g[g == 0] = 1
    t["model.layers.0.self_attn.o_proj.g_idx"] = g


def _diverge(name):
    def f(conf, t):
        g = t[name].copy()
        g[[0, -1]] = g[[-1, 0]]
        t[name] = g if not np.array_equal(g, t[name]) else np.roll(g, 1)
    return f


def _head_dim_96(conf, t):
    conf["head_dim"] = 96


REJECT = {
    "arch": (_mutate_config("architectures", ["Qwen2ForCausalLM"]), NotImplementedError, "architectures"),
    "method": (_mutate_config("quant_method", "bitsandbytes", True), NotImplementedError, "quant_method"),
    "bits": (_mutate_config("bits", 8, True), NotImplementedError, "bits = 8"),
    "group_-1": (_mutate_config("group_size", -1, True), NotImplementedError, "group_size = -1"),
    "group_256": (_mutate_config("group_size", 256, True), NotImplementedError, "group_size = 256"),
    "asym": (_mutate_config("sym", False, True), NotImplementedError, "sym = False"),
    "marlin": (_mutate_config("checkpoint_format", "marlin", True), NotImplementedError, "checkpoint_format"),
    "lm_head_flag": (_mutate_config("lm_head", True, True), NotImplementedError, "lm_head"),
    "lm_head_q": (_add("lm_head.qweight", np.zeros((32, 512), np.int32)), NotImplementedError, "lm_head.qweight"),
    "bias": (_add("model.layers.1.self_attn.v_proj.bias", np.zeros(128, np.float16)), NotImplementedError,
             "model.layers.1.self_attn.v_proj.bias"),
    "head_dim": (_head_dim_96, NotImplementedError, "head_dim = 96"),
    "group_div": (_mutate_config("intermediate_size", 544), ValueError, "intermediate_size = 544"),
    "window": (_mutate_config("sliding_window", 64), ValueError, "sliding_window"),   # with max_pos=128 below
    "shape": (lambda c, t: t.__setitem__("model.layers.0.self_attn.o_proj.scales",
                                         t["model.layers.0.self_attn.o_proj.scales"].T.copy()),
              ValueError, "model.layers.0.self_attn.o_proj.scales"),
    "dtype": (_retype("model.layers.1.mlp.up_proj.qweight", np.float32), ValueError, "model.layers.1.mlp.up_proj.qweight"),
    "norm_dtype": (_retype("model.norm.weight", np.int32), ValueError, "model.norm.weight"),
    "missing": (lambda c, t: t.pop("model.layers.1.mlp.down_proj.scales"), ValueError, "model.layers.1.mlp.down_proj.scales"),
    "qzeros": (_bad_zero, ValueError, "model.layers.1.mlp.up_proj.qzeros"),
    "v2_zeros": (_mutate_config("checkpoint_format", "gptq_v2", True), ValueError, "qzeros"),
    "uneven": (_uneven_groups, ValueError, "model.layers.0.self_attn.o_proj.g_idx"),
    "qkv_order": (_diverge("model.layers.1.self_attn.k_proj.g_idx"), ValueError, "model.layers.1.self_attn.k_proj.g_idx"),
    "gate_up_order": (_diverge("model.layers.0.mlp.up_proj.g_idx"), ValueError, "model.layers.0.mlp.up_proj.g_idx"),
}
REJECT_AWQ = {
    "gemv": (_mutate_config("version", "gemv", True), NotImplementedError, "version"),
    "no_zero": (_mutate_config("zero_point", False, True), NotImplementedError, "zero_point"),
    "not_convert": (_mutate_config("modules_to_not_convert", ["mlp.down_proj"], True), NotImplementedError,
                    "modules_to_not_convert"),
    "awq_shape": (lambda c, t: t.__setitem__("model.layers.0.mlp.gate_proj.qweight",
                                             np.zeros((256 // 8, 512), np.int32)),
                  ValueError, "model.layers.0.mlp.gate_proj.qweight"),
}


def _reject(tmp_path, monkeypatch, method, mutate, exc, text):
    cfg = TINY()
    conf = hf_config(cfg, gptq_quant(64, True) if method == "gptq" else awq_quant(64))
    t = synth_tensors(cfg, method, act_order=True, seed=3)
    mutate(conf, t)
    d = write_checkpoint(str(tmp_path / "c"), conf, t)

    def no_device(*a, **k):
        raise AssertionError("device work before the checkpoint was checked")
    monkeypatch.setattr(G, "lib", no_device)
    monkeypatch.setattr(torch.Tensor, "to", no_device)
    with pytest.raises(exc, match=text.replace(".", r"\.").replace("[", r"\[")):
        G.GptqWeights.from_checkpoint(d, torch.device("cuda:0"), max_pos=128)


@pytest.mark.parametrize("case", sorted(REJECT))
def test_gptq_rejections_name_the_field(tmp_path, monkeypatch, case):
    _reject(tmp_path, monkeypatch, "gptq", *REJECT[case])


@pytest.mark.parametrize("case", sorted(REJECT_AWQ))
def test_awq_rejections_name_the_field(tmp_path, monkeypatch, case):
    _reject(tmp_path, monkeypatch, "awq", *REJECT_AWQ[case])


# ---- the host transform against the checkpoint's product -------------------------------------------------------------
def _unpack_k(qw):
    qw = qw.view(np.uint32)
    q = np.empty((qw.shape[0] * 8, qw.shape[1]), dtype=np.int32)
    for j in range(8):
        q[j::8] = (qw >> np.uint32(4 * j)) & 0xF
    return q


def _stack_w(qw, sc, perm, group):
    """what the device computes with a stack linear: gptq_marlin_repack's tile row i is checkpoint row perm[i], scales
    in natural group order"""
    q = _unpack_k(qw)
    if perm is not None:
        q = q[perm]
    return og.dequant_gptq(og.pack_gptq(q), sc, None, group).astype(np.float64)


def _close(a, b):
    return np.abs(a - b).max() <= 1e-12 * np.abs(b).max()


def test_act_order_transform_matches_checkpoint_product(tmp_path):
    cfg = TINY()
    d = make_checkpoint(str(tmp_path / "a"), cfg, act_order=True, seed=11, shards=2)
    ck = G.GptqCheckpoint(d)
    Gs = cfg.group_size
    rng = np.random.default_rng(5)
    ref = lambda l, n: og.dequant_gptq(**{k: v for k, v in ck.raw(l, n).items() if k != "scales"},
                                       scales=ck.raw(l, n)["scales"], group=Gs).astype(np.float64)
    silu = lambda v: v / (1.0 + np.exp(-v))
    for l in range(cfg.n_layers):
        S = ck.layer(l)
        assert all(S[p] is not None for p in ("perm_qkv", "perm_o", "perm_gate_up", "perm_down"))
        x = rng.standard_normal((5, cfg.hidden))
        want = x @ np.concatenate([ref(l, n) for n in ("q_proj", "k_proj", "v_proj")], axis=1)
        got = x[:, S["perm_qkv"]] @ _stack_w(*S["wqkv"][:2], S["perm_qkv"], Gs)
        assert _close(got, want)
        a = rng.standard_normal((5, cfg.n_heads * cfg.head_dim))
        assert _close(a[:, S["perm_o"]] @ _stack_w(*S["wo"][:2], S["perm_o"], Gs), a @ ref(l, "o_proj"))
        # gate||up: columns in down_proj's order, so SiLU(gate) * up arrives as down's permuted input
        gu = x[:, S["perm_gate_up"]] @ _stack_w(*S["w_gate_up"][:2], S["perm_gate_up"], Gs)
        act = silu(gu[:, :cfg.inter]) * gu[:, cfg.inter:]
        act_ref = silu(x @ ref(l, "gate_proj")) * (x @ ref(l, "up_proj"))
        assert _close(act, act_ref[:, S["perm_down"]])
        assert _close(act @ _stack_w(*S["w_down"][:2], S["perm_down"], Gs), act_ref @ ref(l, "down_proj"))
    ck.close()


def test_awq_layout_concatenates_along_n(tmp_path):
    cfg = TINY()
    ck = G.GptqCheckpoint(make_checkpoint(str(tmp_path / "w"), cfg, method="awq", seed=2))
    assert ck.method == "awq" and all(p == dict(qkv=None, o=None, gate_up=None, down=None) for p in ck.perms)
    S = ck.layer(1)
    for f, names in (("wqkv", ("q_proj", "k_proj", "v_proj")), ("w_gate_up", ("gate_proj", "up_proj"))):
        qw, sc, qz = S[f]
        parts = [og.dequant_awq(r["qweight"], r["scales"], r["qzeros"], cfg.group_size)
                 for r in (ck.raw(1, n) for n in names)]
        assert np.array_equal(og.dequant_awq(qw, sc, qz, cfg.group_size), np.concatenate(parts, axis=1))
    ck.close()


def test_identity_g_idx_under_desc_act_stores_no_permutation(tmp_path):
    cfg = TINY()
    t = synth_tensors(cfg, act_order=False, seed=4)
    d = write_checkpoint(str(tmp_path / "i"), hf_config(cfg, gptq_quant(64, desc_act=True)), t)
    ck = G.GptqCheckpoint(d)
    assert all(v is None for p in ck.perms for v in p.values())
    assert G.act_order_perm(np.arange(256) // 64, 64, "x") is None
    ck.close()
