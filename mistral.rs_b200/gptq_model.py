"""GPTQ / AWQ int4 decode runner over the C ABI (`mrs_gptq_decode_step`, include/mrs_b200_model.h) —
BASELINE config 4 (Mistral-7B GPTQ int4 g128, decode batch 32, paged KV block_size 16).

Python is the harness only (device memory, struct filling, CUDA-graph capture); the layer stack is
C++ (csrc/gptq_decoder.cu) over the reference's Marlin symbols' kernel (csrc/w4a16.cu).

Synthetic checkpoints follow SURVEY §8(d): `qweight` uniform u4 packed [K/8, N] i32, `scales` f16
2^U(-8,-6) [K/128, N], symmetric (`qzeros` = 0x77777777 in the checkpoint, ignored by the Marlin
path), `g_idx[k] = k/128`; dense f16 embeddings / lm_head / norms.  Load flow = the reference's
`gptq_linear` (gptq_cuda.rs:451-623): `gptq_marlin_repack` per tensor (q/k/v and gate/up are
concatenated along N first, which the row-tile format allows) — scales stay unpermuted because
this stack calls the kernel's native entry (`mrs_w4a16_gemm`, scale_perm 0).

Checkpoints on disk (`GptqCheckpoint`, `GptqWeights.from_checkpoint`): Hugging Face GPTQ (symmetric, 4-bit, with or
without act-order) and AWQ (GEMM, zero points) directories of Llama / Mistral models.  Act-order linears are repacked
with perm = argsort(g_idx) and take their input as x[:, perm]: the norm in front of q||k||v and gate||up writes in that
order, a column gather feeds o_proj, and down_proj's order is folded into the N columns of gate||up on the host."""
import ctypes
import glob
import json
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import lib
from .model import (MAX_PREFILL_SEQS, LlamaWeights, PagedDecodeRunner, PromptPrefill, SpecVerifier, _point,
                    check_runner_args, rope_tables, runner_split_pages)


@dataclass
class GptqConfig:
    hidden: int = 4096
    inter: int = 14336
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: int = 8
    head_dim: int = 128
    vocab: int = 32000
    rms_eps: float = 1e-5
    rope_theta: float = 10000.0
    rope_scaling: dict = None
    rope_freq_factors: object = None
    max_pos: int = 4096
    group_size: int = 128
    block_size: int = 16
    rope_neox: bool = True
    name: str = "mistral-7b-gptq"
    scale_exp: tuple = (-8, -6)
    tie_word_embeddings: bool = False
    sliding_window: int = None      # Mistral's attention window; max_pos is capped to it (full attention within it)

    @staticmethod
    def mistral_7b(**kw):
        return GptqConfig(**kw)

    @staticmethod
    def tiny_test(**kw):
        d = dict(hidden=256, inter=512, n_layers=2, n_heads=4, n_kv_heads=2, head_dim=64, vocab=512, max_pos=256,
                 group_size=64, name="tiny-gptq")
        d.update(kw)
        return GptqConfig(**d)


class _W4(ctypes.Structure):
    _fields_ = [("tiles", ctypes.c_void_p), ("scales", ctypes.c_void_p), ("qzeros", ctypes.c_void_p),
                ("k", ctypes.c_int32), ("n", ctypes.c_int32)]


class _Layer(ctypes.Structure):
    _fields_ = [(n, _W4) for n in ("wqkv", "wo", "w_gate_up", "w_down")] + \
               [(n, ctypes.c_void_p) for n in ("attn_norm", "ffn_norm", "k_cache", "v_cache", "perm_qkv", "perm_o",
                                               "perm_gate_up")]


class _Step(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("hidden", "n_layers", "n_heads", "n_kv_heads", "head_dim", "vocab",
                                              "block_size", "act_dtype", "group_size")] + \
               [("rms_eps", ctypes.c_float), ("sm_scale", ctypes.c_float)] + \
               [(n, ctypes.c_int32) for n in ("rope_neox", "cache_layout", "batch", "padded_tiles", "max_blocks_per_seq",
                                              "skip_mask")] + \
               [("layers", ctypes.POINTER(_Layer))] + \
               [(n, ctypes.c_void_p) for n in ("tok_embd", "lm_head", "final_norm", "rope_cos", "rope_sin", "token_ids",
                                               "positions", "slot_mapping", "kv_indptr", "kv_indices", "kv_last_page_len",
                                               "request_indices", "kv_tile_indices", "o_indptr", "kv_chunk_size",
                                               "block_valid_mask", "block_tables", "context_lens", "x", "x2", "h", "qkv",
                                               "attn_out", "o", "gate_up", "act", "logits", "tmp_v", "tmp_s", "out_token",
                                               "attn_counters", "argmax_scratch", "attn_perm")]


def synth_gptq(K, N, group, seed, scale_exp=(-8, -6)):
    """(qweight [K/8, N] i32, scales [K/group, N] f16) per SURVEY §8(d)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    qweight = rng.integers(0, 2 ** 32, size=(K // 8, N), dtype=np.uint64).astype(np.uint32).view(np.int32)
    scales = np.exp2(rng.uniform(scale_exp[0], scale_exp[1], size=(K // group, N))).astype(np.float16)
    return qweight, scales


HF_ARCHITECTURES = ("LlamaForCausalLM", "MistralForCausalLM")
_ATTN_LINEARS = ("q_proj", "k_proj", "v_proj", "o_proj")
_FLOAT_DTYPES = ("F16", "BF16", "F32")


def act_order_perm(g_idx, group, name):
    """perm = argsort(g_idx, stable) as int32, or None when g_idx is the natural k // group (no permutation).  Every
    group must hold exactly `group` rows: then sorted row i belongs to group i // group and the scales stay as stored."""
    g = np.asarray(g_idx).astype(np.int64)
    K = g.size
    if np.array_equal(g, np.arange(K) // group):
        return None
    if g.min() < 0 or g.max() >= K // group or np.any(np.bincount(g, minlength=K // group) != group):
        raise ValueError(f"`{name}`: act-order groups must each hold exactly group_size = {group} rows with indices in "
                         f"0..{K // group - 1}")
    return np.argsort(g, kind="stable").astype(np.int32)


class GptqCheckpoint:
    """A Hugging Face GPTQ / AWQ int4 checkpoint directory (Llama / Mistral), read on the host into the int4 stack's
    layout.  The constructor parses `config.json` (and `quantization_config`, or `quantize_config.json`), checks every
    tensor's presence, dtype and shape, the GPTQ zero points and act-order groups, and derives the permutations; it
    raises NotImplementedError / ValueError naming the offending key or tensor and touches no device.  `layer(l)` and
    `top()` then return host arrays.  Weights come from `model.safetensors.index.json` and its shards, or else from the
    directory's single `*.safetensors`, through `uqff_file.SafetensorsFile`."""

    def __init__(self, path, max_pos=None):
        from .uqff_file import SafetensorsFile
        self.path = os.fspath(path)
        cpath = os.path.join(self.path, "config.json")
        if not os.path.isfile(cpath):
            raise ValueError(f"{self.path}: no config.json")
        with open(cpath) as f:
            cj = json.load(f)
        archs = cj.get("architectures") or []
        if not any(a in HF_ARCHITECTURES for a in archs):
            raise NotImplementedError(f"config.json `architectures` = {archs}: the int4 stack runs "
                                      f"{' / '.join(HF_ARCHITECTURES)}")
        q, qsrc = cj.get("quantization_config"), "config.json `quantization_config`"
        if q is None:
            qpath = os.path.join(self.path, "quantize_config.json")
            if not os.path.isfile(qpath):
                raise ValueError(f"{self.path}: config.json has no `quantization_config` and there is no quantize_config.json")
            with open(qpath) as f:
                q, qsrc = json.load(f), "quantize_config.json"
        self._quant(q, qsrc)
        self.cfg = self._model(cj, max_pos)
        idx = os.path.join(self.path, "model.safetensors.index.json")
        if os.path.isfile(idx):
            with open(idx) as f:
                wmap = json.load(f).get("weight_map")
            if not isinstance(wmap, dict) or not wmap:
                raise ValueError(f"{idx}: no `weight_map`")
            files = sorted(set(wmap.values()))
        else:
            files = sorted(os.path.basename(p) for p in glob.glob(os.path.join(self.path, "*.safetensors")))
            if len(files) != 1:
                raise ValueError(f"{self.path}: no model.safetensors.index.json and {len(files)} *.safetensors files "
                                 "(need exactly one)")
        self.files = [SafetensorsFile(os.path.join(self.path, f)) for f in files]
        self._where = {}
        for sf in self.files:
            for name in sf.entries:
                if name in self._where:
                    raise ValueError(f"tensor `{name}` is in two shards")
                self._where[name] = sf
        self._check()

    def _quant(self, q, src):
        self.method = str(q.get("quant_method", "gptq")).lower()
        if self.method not in ("gptq", "awq"):
            raise NotImplementedError(f"{src}: quant_method = {self.method!r}; GPTQ and AWQ checkpoints are read")
        bits = q.get("bits")
        if bits != 4:
            raise NotImplementedError(f"{src}: bits = {bits}; the int4 stack takes 4-bit checkpoints")
        group = q.get("group_size")
        if group is None:
            raise ValueError(f"{src}: `group_size` is missing")
        if group == -1:
            raise NotImplementedError(f"{src}: group_size = -1 (one group per column) is not supported")
        if group not in (32, 64, 128):
            raise NotImplementedError(f"{src}: group_size = {group}; 32, 64 and 128 are supported")
        self.group, self.zero, self.not_convert = int(group), None, []
        if self.method == "gptq":
            if q.get("sym", True) is not True:
                raise NotImplementedError(f"{src}: sym = {q.get('sym')}; asymmetric GPTQ is not supported")
            fmt = q.get("checkpoint_format")
            if fmt not in (None, "gptq", "gptq_v2"):
                raise NotImplementedError(f"{src}: checkpoint_format = {fmt!r}; `gptq` and `gptq_v2` are read")
            self.zero = 8 if fmt == "gptq_v2" else 7        # the stored symmetric zero point (v1 stores z - 1)
            if q.get("lm_head"):
                raise NotImplementedError(f"{src}: lm_head = true; a quantised lm_head is not supported")
        else:
            if q.get("zero_point", True) is not True:
                raise NotImplementedError(f"{src}: zero_point = {q.get('zero_point')}; AWQ without zero points is not supported")
            version = str(q.get("version", "gemm")).lower()
            if version != "gemm":
                raise NotImplementedError(f"{src}: version = {q.get('version')!r}; only the AWQ GEMM layout is read")
            self.not_convert = list(q.get("modules_to_not_convert") or [])

    def _model(self, cj, max_pos):
        try:
            lc = LlamaWeights.config_from_hf(cj)
        except KeyError as e:
            raise ValueError(f"config.json: {e.args[0]!r} is missing") from None
        if lc.head_dim not in (64, 128):
            raise NotImplementedError(f"config.json: head_dim = {lc.head_dim}; the fused attention runs 64 and 128")
        window = cj.get("sliding_window")
        window = int(window) if window else None
        mp = lc.max_pos if window is None else min(lc.max_pos, window)
        if max_pos is not None:
            if window is not None and int(max_pos) > window:
                raise ValueError(f"max_pos = {max_pos} exceeds config.json `sliding_window` = {window} (windowed attention "
                                 "is not implemented; within the window it equals full attention)")
            mp = int(max_pos)
        cfg = GptqConfig(hidden=lc.hidden, inter=lc.inter, n_layers=lc.n_layers, n_heads=lc.n_heads,
                         n_kv_heads=lc.n_kv_heads, head_dim=lc.head_dim, vocab=lc.vocab, rms_eps=lc.rms_eps,
                         rope_theta=lc.rope_theta, rope_scaling=lc.rope_scaling, max_pos=mp, group_size=self.group,
                         name=lc.name, tie_word_embeddings=bool(cj.get("tie_word_embeddings", False)),
                         sliding_window=window)
        nq = cfg.n_heads * cfg.head_dim
        for key, K in (("hidden_size", cfg.hidden), ("num_attention_heads * head_dim", nq), ("intermediate_size", cfg.inter)):
            if K % self.group or K % 64:
                raise ValueError(f"config.json: {key} = {K} is not a multiple of group_size {self.group} and of 64")
        return cfg

    # ---- tensors ------------------------------------------------------------------------------------------------
    def shapes(self):
        c = self.cfg
        nq, nkv = c.n_heads * c.head_dim, c.n_kv_heads * c.head_dim
        return {"q_proj": (c.hidden, nq), "k_proj": (c.hidden, nkv), "v_proj": (c.hidden, nkv), "o_proj": (nq, c.hidden),
                "gate_proj": (c.hidden, c.inter), "up_proj": (c.hidden, c.inter), "down_proj": (c.inter, c.hidden)}   # (K, N)

    @staticmethod
    def key(l, name):
        return f"model.layers.{l}.{'self_attn' if name in _ATTN_LINEARS else 'mlp'}.{name}"

    def _entry(self, name, dtypes, shape):
        if name not in self._where:
            raise ValueError(f"tensor `{name}` is missing from {self.path}")
        dt, shp = self._where[name].entries[name][:2]
        if dt not in dtypes:
            raise ValueError(f"tensor `{name}` has dtype {dt}, expected {' / '.join(dtypes)}")
        if tuple(shp) != tuple(shape):
            raise ValueError(f"tensor `{name}` has shape {list(shp)}, expected {list(shape)}")
        return name

    def array(self, name):
        """the stored tensor as a numpy array (BF16 widened to f32)"""
        sf = self._where[name]
        a = np.array(sf.array(name))
        if sf.entries[name][0] == "BF16":
            a = (a.astype(np.uint32) << 16).view(np.float32)
        return a

    def _check(self):
        c, G = self.cfg, self.group
        H = c.hidden
        if "lm_head.qweight" in self._where:
            raise NotImplementedError("tensor `lm_head.qweight`: a quantised lm_head is not supported")
        self._entry("model.embed_tokens.weight", _FLOAT_DTYPES, (c.vocab, H))
        self._entry("model.norm.weight", _FLOAT_DTYPES, (H,))
        self.tied = c.tie_word_embeddings
        if not self.tied:
            self._entry("lm_head.weight", _FLOAT_DTYPES, (c.vocab, H))
        self.perms = []
        for l in range(c.n_layers):
            for n in ("input_layernorm", "post_attention_layernorm"):
                self._entry(f"model.layers.{l}.{n}.weight", _FLOAT_DTYPES, (H,))
            g_idx = {}
            for name, (K, N) in self.shapes().items():
                base = self.key(l, name)
                if f"{base}.bias" in self._where:
                    raise NotImplementedError(f"tensor `{base}.bias`: linear biases are not supported")
                cover = [m for m in self.not_convert if m in base]
                if cover:
                    raise NotImplementedError(f"quantization_config `modules_to_not_convert` entry {cover[0]!r} covers "
                                              f"`{base}`: dense linears are not supported")
                if f"{base}.qweight" not in self._where and f"{base}.weight" in self._where:
                    raise NotImplementedError(f"tensor `{base}.weight`: dense linears are not supported")
                self._entry(f"{base}.qweight", ("I32",), (K // 8, N) if self.method == "gptq" else (K, N // 8))
                self._entry(f"{base}.qzeros", ("I32",), (K // G, N // 8))
                self._entry(f"{base}.scales", ("F16", "BF16"), (K // G, N))
                if self.method == "gptq":
                    z = self._where[f"{base}.qzeros"].array(f"{base}.qzeros").view(np.uint32)
                    if np.any(z != np.uint32(self.zero * 0x11111111)):
                        raise ValueError(f"tensor `{base}.qzeros`: not every zero point is the symmetric {self.zero} "
                                         "(an asymmetric checkpoint, which this stack does not run)")
                    gname = f"{base}.g_idx"
                    g_idx[name] = (self.array(self._entry(gname, ("I32",), (K,))) if gname in self._where
                                   else np.arange(K, dtype=np.int32) // G)
            perms = dict(qkv=None, o=None, gate_up=None, down=None)
            if self.method == "gptq":
                for group, names in (("qkv", ("q_proj", "k_proj", "v_proj")), ("gate_up", ("gate_proj", "up_proj"))):
                    for n in names[1:]:
                        if not np.array_equal(g_idx[n], g_idx[names[0]]):
                            raise ValueError(f"tensor `{self.key(l, n)}.g_idx` differs from `{self.key(l, names[0])}.g_idx` "
                                             "(modules that share an input must share its act order)")
                    perms[group] = act_order_perm(g_idx[names[0]], G, f"{self.key(l, names[0])}.g_idx")
                perms["o"] = act_order_perm(g_idx["o_proj"], G, f"{self.key(l, 'o_proj')}.g_idx")
                perms["down"] = act_order_perm(g_idx["down_proj"], G, f"{self.key(l, 'down_proj')}.g_idx")
            self.perms.append(perms)

    def raw(self, l, name):
        """one linear's tensors as stored: dict(qweight, scales f32, and g_idx (GPTQ) or qzeros (AWQ))"""
        base = self.key(l, name)
        d = dict(qweight=self.array(f"{base}.qweight"), scales=self.array(f"{base}.scales").astype(np.float32))
        if self.method == "awq":
            d["qzeros"] = self.array(f"{base}.qzeros")
        else:
            d["g_idx"] = (self.array(f"{base}.g_idx") if f"{base}.g_idx" in self._where
                          else np.arange(self.shapes()[name][0], dtype=np.int32) // self.group)
        return d

    def layer(self, l):
        """layer l in the stack's layout: wqkv / wo / w_gate_up / w_down as (qweight, scales, qzeros or None) with
        q||k||v and gate||up concatenated along N (AWQ qweight / qzeros along their N/8 axis), gate's and up's N columns
        in down_proj's act order; perm_qkv / perm_o / perm_gate_up (int32 [K] or None) for gptq_marlin_repack; the
        two norms as f32."""
        P = self.perms[l]

        def cat(names, col_perm=None):
            parts = [self.raw(l, n) for n in names]
            # col_perm is GPTQ only: qweight [K/8, N] and scales [K/g, N] hold N as their columns
            sel = (lambda a: a) if col_perm is None else (lambda a: a[:, col_perm])
            qw = np.concatenate([sel(p["qweight"]) for p in parts], axis=1)
            sc = np.concatenate([sel(p["scales"]) for p in parts], axis=1)
            qz = np.concatenate([p["qzeros"] for p in parts], axis=1) if self.method == "awq" else None
            return np.ascontiguousarray(qw), np.ascontiguousarray(sc), qz
        out = dict(wqkv=cat(("q_proj", "k_proj", "v_proj")), wo=cat(("o_proj",)),
                   w_gate_up=cat(("gate_proj", "up_proj"), P["down"]), w_down=cat(("down_proj",)),
                   perm_qkv=P["qkv"], perm_o=P["o"], perm_gate_up=P["gate_up"], perm_down=P["down"])
        for key, n in (("attn_norm", "input_layernorm"), ("ffn_norm", "post_attention_layernorm")):
            out[key] = self.array(f"model.layers.{l}.{n}.weight").astype(np.float32)
        return out

    def top(self):
        """(embedding [vocab, hidden], lm_head or None when tied, final norm [hidden]) as f32"""
        emb = self.array("model.embed_tokens.weight").astype(np.float32)
        head = None if self.tied else self.array("lm_head.weight").astype(np.float32)
        return emb, head, self.array("model.norm.weight").astype(np.float32)

    def close(self):
        for f in self.files:
            f.close()


class GptqWeights:
    """Synthetic device-resident GPTQ checkpoint in the decode stack's layout (int4 tiles); `from_checkpoint` loads a
    GPTQ / AWQ checkpoint directory into the same layout."""
    NAMES = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")

    def __init__(self, cfg: GptqConfig, device, dtype=torch.float16, keep_host=False):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        self.host = {} if keep_host else None
        H, I = cfg.hidden, cfg.inter
        nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
        shapes = {"q_proj": (H, nq), "k_proj": (H, nkv), "v_proj": (H, nkv), "o_proj": (nq, H), "gate_proj": (H, I),
                  "up_proj": (H, I), "down_proj": (I, H)}            # (K, N)
        self.layers, self.nbytes = [], 0
        for l in range(cfg.n_layers):
            raw = {}
            for i, name in enumerate(self.NAMES):
                K, N = shapes[name]
                raw[name] = synth_gptq(K, N, cfg.group_size, 0xC400 + l * 16 + i, cfg.scale_exp)
                if self.host is not None:
                    self.host[(l, name)] = raw[name]
            L = {"wqkv": self._pack([raw["q_proj"], raw["k_proj"], raw["v_proj"]]), "wo": self._pack([raw["o_proj"]]),
                 "w_gate_up": self._pack([raw["gate_proj"], raw["up_proj"]]), "w_down": self._pack([raw["down_proj"]])}
            for j, name in enumerate(("attn_norm", "ffn_norm")):
                L[name] = self._norm(0xC400 + l * 16 + 8 + j, (l, name))
            self.layers.append(L)
        rng = np.random.Generator(np.random.PCG64(0xC3FF))
        emb = (0.5 * rng.standard_normal((cfg.vocab, H))).astype(np.float32)
        head = (0.05 * rng.standard_normal((cfg.vocab, H))).astype(np.float32)
        self.tok_embd = torch.from_numpy(emb).to(device).to(dtype)
        self.lm_head = torch.from_numpy(head).to(device).to(dtype)
        self.final_norm = self._norm(0xC3FE, (0, "final_norm"))
        if self.host is not None:
            self.host[(0, "tok_embd")] = self.tok_embd.float().cpu().numpy()
            self.host[(0, "lm_head")] = self.lm_head.float().cpu().numpy()
        self.nbytes += 2 * self.lm_head.numel()
        cos, sin = rope_tables(cfg)
        self.rope_cos = torch.from_numpy(cos).to(device).to(dtype)
        self.rope_sin = torch.from_numpy(sin).to(device).to(dtype)

    def _norm(self, seed, key):
        rng = np.random.Generator(np.random.PCG64(seed))
        t = torch.from_numpy((1.0 + 0.1 * rng.standard_normal(self.cfg.hidden)).astype(np.float32)).to(self.device).to(self.dtype)
        if self.host is not None:
            self.host[key] = t.float().cpu().numpy()
        return t

    def _pack(self, parts):
        """concatenate checkpoint tensors along N, repack to int4 tiles (gptq_marlin_repack)."""
        qw = np.concatenate([p[0] for p in parts], axis=1)
        sc = np.concatenate([p[1] for p in parts], axis=1)
        K, N = qw.shape[0] * 8, qw.shape[1]
        tq = torch.from_numpy(np.ascontiguousarray(qw)).to(self.device)
        tiles = torch.empty(K // 16, N * 16 // 8, dtype=torch.int32, device=self.device)
        lib().gptq_marlin_repack(ctypes.c_void_p(tq.data_ptr()), ctypes.c_void_p(0), ctypes.c_void_p(tiles.data_ptr()),
                                 ctypes.c_int(K), ctypes.c_int(N), ctypes.c_int(4),
                                 ctypes.c_int64(torch.cuda.current_stream(self.device).cuda_stream))
        torch.cuda.synchronize()
        scales = torch.from_numpy(np.ascontiguousarray(sc)).to(self.device).to(self.dtype)
        self.nbytes += tiles.numel() * 4 + scales.numel() * 2
        return (tiles, scales, K, N)

    @classmethod
    def from_checkpoint(cls, path, device, dtype=torch.float16, max_pos=None, keep_host=False):
        """Device-resident weights of a GPTQ / AWQ checkpoint directory (see GptqCheckpoint, which checks everything
        before the first upload).  Linears are repacked by gptq_marlin_repack with their act-order perm (or by
        awq_marlin_repack, with the AWQ zero points kept raw); norms, embedding and lm_head are converted to `dtype`,
        and a tied checkpoint's lm_head is the embedding's tensor.  max_pos: RoPE table length (default the config's,
        capped to its sliding window).  keep_host: `host` holds what a CPU reference model needs, the linears as
        stored (dicts of qweight, scales and g_idx or qzeros) and the rest rounded through `dtype`."""
        ck = GptqCheckpoint(path, max_pos)
        try:
            self = cls.__new__(cls)
            cfg = self.cfg = ck.cfg
            self.device, self.dtype, self.quant_method = device, dtype, ck.method
            self.host = {} if keep_host else None
            self.layers, self.nbytes = [], 0
            for l in range(cfg.n_layers):
                S = ck.layer(l)
                L, qz = {}, {}
                for f, perm in (("wqkv", S["perm_qkv"]), ("wo", S["perm_o"]), ("w_gate_up", S["perm_gate_up"]),
                                ("w_down", S["perm_down"])):
                    L[f], qz[f] = self._upload_w4(*S[f], perm)
                L["qzeros"] = qz
                for f in ("perm_qkv", "perm_o", "perm_gate_up"):
                    L[f] = None if S[f] is None else torch.from_numpy(S[f]).to(device)
                for f in ("attn_norm", "ffn_norm"):
                    L[f] = self._put(S[f], (l, f))
                if self.host is not None:
                    for name in self.NAMES:
                        self.host[(l, name)] = ck.raw(l, name)
                self.layers.append(L)
            emb, head, final = ck.top()
            self.tok_embd = self._put(emb, (0, "tok_embd"))
            self.lm_head = self.tok_embd if head is None else self._put(head, (0, "lm_head"))
            if head is None and self.host is not None:
                self.host[(0, "lm_head")] = self.host[(0, "tok_embd")]
            self.final_norm = self._put(final, (0, "final_norm"))
        finally:
            ck.close()
        self.nbytes += 2 * self.lm_head.numel()
        cos, sin = rope_tables(cfg)
        self.rope_cos = torch.from_numpy(cos).to(device).to(dtype)
        self.rope_sin = torch.from_numpy(sin).to(device).to(dtype)
        return self

    def _put(self, a, key):
        t = torch.from_numpy(np.ascontiguousarray(a)).to(self.device).to(self.dtype)
        if self.host is not None:
            self.host[key] = t.float().cpu().numpy()
        return t

    def _upload_w4(self, qw, sc, qzeros, perm):
        """one stack linear from checkpoint tensors -> ((tiles, scales, K, N), AWQ qzeros on the device or None)"""
        awq = self.quant_method == "awq"
        K, N = (qw.shape[0], qw.shape[1] * 8) if awq else (qw.shape[0] * 8, qw.shape[1])
        tq = torch.from_numpy(np.ascontiguousarray(qw)).to(self.device)
        tp = None if perm is None else torch.from_numpy(perm).to(self.device)
        tiles = torch.empty(K // 16, N * 16 // 8, dtype=torch.int32, device=self.device)
        st = ctypes.c_int64(torch.cuda.current_stream(self.device).cuda_stream)
        if awq:
            lib().awq_marlin_repack(ctypes.c_void_p(tq.data_ptr()), ctypes.c_void_p(0), ctypes.c_void_p(tiles.data_ptr()),
                                    ctypes.c_int(K), ctypes.c_int(N // 8), ctypes.c_int(4), st)
        else:
            lib().gptq_marlin_repack(ctypes.c_void_p(tq.data_ptr()), ctypes.c_void_p(0 if tp is None else tp.data_ptr()),
                                     ctypes.c_void_p(tiles.data_ptr()), ctypes.c_int(K), ctypes.c_int(N), ctypes.c_int(4), st)
        torch.cuda.synchronize()
        scales = torch.from_numpy(np.ascontiguousarray(sc)).to(self.device).to(self.dtype)
        qz = None if qzeros is None else torch.from_numpy(np.ascontiguousarray(qzeros)).to(self.device)
        self.nbytes += tiles.numel() * 4 + scales.numel() * 2 + (0 if qz is None else qz.numel() * 4)
        return (tiles, scales, K, N), qz

    @property
    def act_order_o(self):
        """True when some layer's o_proj is act-order (its input needs the attn_perm scratch)"""
        return any(L.get("perm_o") is not None for L in self.layers)


def _model_step(weights, k_cache, v_cache, cache_layout):
    """(layer array, mrs_gptq_step) with the model fields only: weights, norms, caches in `cache_layout` ("hnd" or
    "vllm"), dims, RoPE tables; no per-step metadata or scratch.  The layer array must outlive the struct's use."""
    cfg = weights.cfg
    layers = (_Layer * cfg.n_layers)()
    for l, L in enumerate(weights.layers):
        for f in ("wqkv", "wo", "w_gate_up", "w_down"):
            tiles, scales, K, N = L[f]
            qz = L.get("qzeros", {}).get(f)
            setattr(layers[l], f, _W4(tiles.data_ptr(), scales.data_ptr(), 0 if qz is None else qz.data_ptr(), K, N))
        for f in ("perm_qkv", "perm_o", "perm_gate_up"):
            setattr(layers[l], f, None if L.get(f) is None else L[f].data_ptr())
        layers[l].attn_norm, layers[l].ffn_norm = L["attn_norm"].data_ptr(), L["ffn_norm"].data_ptr()
        layers[l].k_cache, layers[l].v_cache = k_cache[l].data_ptr(), v_cache[l].data_ptr()
    s = _Step()
    s.hidden, s.n_layers, s.n_heads, s.n_kv_heads, s.head_dim, s.vocab = (cfg.hidden, cfg.n_layers, cfg.n_heads,
                                                                          cfg.n_kv_heads, cfg.head_dim, cfg.vocab)
    s.block_size, s.act_dtype, s.group_size = cfg.block_size, {torch.float16: 0, torch.bfloat16: 1}[weights.dtype], cfg.group_size
    s.rms_eps, s.sm_scale = cfg.rms_eps, 1.0 / float(np.sqrt(cfg.head_dim))
    s.rope_neox, s.cache_layout, s.skip_mask = int(cfg.rope_neox), 1 if cache_layout == "hnd" else 0, 0
    s.layers = ctypes.cast(layers, ctypes.POINTER(_Layer))
    s.tok_embd, s.lm_head, s.final_norm = weights.tok_embd.data_ptr(), weights.lm_head.data_ptr(), weights.final_norm.data_ptr()
    s.rope_cos, s.rope_sin = weights.rope_cos.data_ptr(), weights.rope_sin.data_ptr()
    return layers, s


class GptqRunner(PagedDecodeRunner):
    """KV cache + scratch + per-step metadata for a decode batch; drives mrs_gptq_decode_step.  The vLLM cache layout
    runs the unsplit attention plan."""

    def __init__(self, weights: GptqWeights, batch=32, max_ctx=512, cache_layout="hnd", sm_count=132):
        check_runner_args(batch)
        cfg = weights.cfg
        super().__init__(weights, batch, max_ctx, runner_split_pages(cfg.block_size, batch, cfg.n_kv_heads, max_ctx, sm_count)
                         if cache_layout == "hnd" else 0)
        batch, dev, dt, nb = self.B, self.dev, self.dt, self.B * self.max_blocks + 1
        bs, D, KVH, NH, H = cfg.block_size, cfg.head_dim, cfg.n_kv_heads, cfg.n_heads, cfg.hidden
        a = lambda *s: torch.zeros(*s, dtype=dt, device=dev)
        nq, nkv = NH * D, KVH * D
        self.buf = dict(x=a(batch, H), x2=a(batch, H), h=a(batch, H), qkv=a(batch, nq + 2 * nkv), attn_out=a(batch, nq),
                        o=a(batch, H), gate_up=a(batch, 2 * cfg.inter), act=a(batch, cfg.inter), logits=a(batch, cfg.vocab),
                        tmp_v=a(self.padded_tiles, NH, D), tmp_s=torch.zeros(self.padded_tiles, NH, dtype=torch.float32, device=dev),
                        out_token=self.meta["token_ids"],
                        attn_counters=torch.zeros(batch * KVH * 2, dtype=torch.int32, device=dev),
                        argmax_scratch=torch.zeros(16 * batch + 16, dtype=torch.uint8, device=dev))
        if weights.act_order_o:
            self.buf["attn_perm"] = a(batch, nq)
        self.layout = cache_layout
        if cache_layout == "hnd":
            self.k_cache = [a(nb, KVH, bs, D) for _ in range(cfg.n_layers)]
            self.v_cache = [a(nb, KVH, bs, D) for _ in range(cfg.n_layers)]
        else:
            self.k_cache = [a(nb, KVH, D // 8, bs, 8) for _ in range(cfg.n_layers)]
            self.v_cache = [a(nb, KVH, D, bs) for _ in range(cfg.n_layers)]
        self._layers, s = _model_step(weights, self.k_cache, self.v_cache, cache_layout)
        s.batch, s.padded_tiles, s.max_blocks_per_seq = batch, self.padded_tiles, self.max_blocks
        _point(s, self.meta, dict(block_tables=self.block_tables, context_lens=self.context_lens), self.buf)
        self.step_struct = s

    def forward(self):
        rc = lib().mrs_gptq_decode_step(ctypes.byref(self.step_struct), self._stream())
        if rc != 0:
            raise RuntimeError(f"mrs_gptq_decode_step failed: cudaError {rc}")


class GptqPrefill(PromptPrefill):
    """Prompt processing of a GPTQ / AWQ model through `mrs_gptq_prefill_step` (include/mrs_b200_model.h): the packed
    rows of up to 256 sequences through the int4 layer stack in one pass -- whole-K W4A16 GEMMs (q||k||v, o, gate||up
    with the SiLU*mul epilogue, down), RoPE, the var-len causal prompt attention and the KV scatter, the dense lm_head on
    each sequence's last row (or every row) and argmax.  `forward` and `forward_batch` mean what they mean on
    LlamaPrefill.  With a GptqRunner the K/V go into the runner's caches in its layout, and `forward_batch(slots=...)`
    followed by `runner.replay()` continues those rows in the decode graph; without one the prefill writes its own HND
    caches.  Prompts over cached rows (cached > 0) need the HND layout: the paged prompt attention reads HND pages."""
    STEP = "mrs_gptq_prefill_step"

    def __init__(self, weights: GptqWeights, max_tokens=4096, runner: GptqRunner = None, pdl=True):
        """max_tokens: new rows per call (all sequences together); the scratch for them is allocated here.
        pdl: run the GEMMs and norms as a programmatic-dependent-launch chain."""
        self._init_caches(weights, max_tokens, runner)
        self.layout = runner.layout if runner is not None else "hnd"
        cfg, dev, dt = self.cfg, self.dev, self.dt
        T, H = self.max_tokens, cfg.hidden
        nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
        a = lambda *s: torch.empty(*s, dtype=dt, device=dev)
        self.buf = dict(x=a(T, H), x2=a(T, H), h=a(T, H), q=a(T, nq + 2 * nkv), attn_out=a(T, nq), act=a(T, cfg.inter),
                        h_last=a(MAX_PREFILL_SEQS, H),
                        argmax_scratch=torch.zeros(16 * MAX_PREFILL_SEQS + 16, dtype=torch.uint8, device=dev))
        self._layers, self.step_struct = _model_step(weights, self.k_cache, self.v_cache, self.layout)
        self.step_struct.skip_mask = 0 if pdl else 4
        self._attn_perm = a(T, nq) if weights.act_order_o else None       # act-order o_proj input, [T, nq]
        if self._attn_perm is not None:
            self.step_struct.attn_perm = self._attn_perm.data_ptr()

    def make_plan(self, ids, cached, tables, lm_rows, slots=None):
        if self.layout != "hnd" and any(int(c) for c in cached):
            raise ValueError("GptqPrefill: cached rows need the HND cache layout (the paged prompt attention reads HND "
                             f"pages), the runner's is {self.layout!r}")
        return super().make_plan(ids, cached, tables, lm_rows, slots)


def check_gptq_verifier_args(runner, draft_len):
    """ValueError unless `runner` (a GptqRunner) can run verify steps of `draft_len` drafts (see GptqVerifier).  There is
    no GEMV route in the GPTQ stack, so every batch 1..256 takes every draft_len 1..7."""
    k = int(draft_len)
    if not 1 <= k <= 7:
        raise ValueError(f"draft_len must be 1..7, got {draft_len}")
    if runner.layout != "hnd":
        raise ValueError(f"verify steps need the HND cache layout (the multi-query attention reads HND pages), the "
                         f"runner's is {runner.layout!r}")
    if runner.cfg.head_dim not in (64, 128):
        raise ValueError(f"verify attention supports head_dim 64 / 128, got {runner.cfg.head_dim}")
    if runner.dt not in (torch.float16, torch.bfloat16):
        raise ValueError(f"verify steps run in f16 / bf16, got {runner.dt}")
    if runner.max_ctx < k + 1:
        raise ValueError(f"the runner's context ({runner.max_ctx}) is shorter than one verify step ({k + 1} rows)")
    return k


class GptqVerifier(SpecVerifier):
    """Speculative decoding on a GptqRunner's sequences through `mrs_gptq_verify_step` (include/mrs_b200_model.h; see
    SpecVerifier): the int4 layer stack over the B*q rows with the runner's GEMM route, the multi-query fused attention
    reading q, k and v inside the q||k||v rows, the dense lm_head on every row, argmax and the acceptance.  Needs the
    HND cache layout.  `speculative_generate` drives it as it drives a LlamaVerifier."""
    STEP = "mrs_gptq_verify_step"

    def __init__(self, runner: GptqRunner, draft_len: int):
        k = check_gptq_verifier_args(runner, draft_len)
        super().__init__(runner, k)
        cfg, dev, dt, B, q = runner.cfg, runner.dev, runner.dt, self.B, self.q
        R, D, KVH, NH, H, P = B * q, cfg.head_dim, cfg.n_kv_heads, cfg.n_heads, cfg.hidden, runner.padded_tiles
        a = lambda *s: torch.zeros(*s, dtype=dt, device=dev)
        z = lambda *s, d=torch.int32: torch.zeros(*s, dtype=d, device=dev)
        nsub = -(-(NH // KVH) * q // 16)
        self.buf = dict(x=a(R, H), x2=a(R, H), h=a(R, H), qkv=a(R, (NH + 2 * KVH) * D), attn_out=a(R, NH * D),
                        o=a(R, H), gate_up=a(R, 2 * cfg.inter), act=a(R, cfg.inter), logits=a(R, cfg.vocab),
                        tmp_v=a(P, q * NH, D), tmp_s=z(P, q * NH, d=torch.float32), out_token=z(R),
                        attn_counters=z(B * KVH * nsub), argmax_scratch=z(16 * R + 16, d=torch.uint8))
        if runner.w.act_order_o:
            self.buf["attn_perm"] = a(R, NH * D)
        s = _Step.from_buffer_copy(runner.step_struct)   # weights, caches, shapes, tables, lengths: the runner's
        _point(s, self.meta, self.buf)
        self.step_struct = s
