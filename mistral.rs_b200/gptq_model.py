"""GPTQ / AWQ int4 decode runner over the C ABI (`mrs_gptq_decode_step`, include/mrs_b200_model.h) —
BASELINE config 4 (Mistral-7B GPTQ int4 g128, decode batch 32, paged KV block_size 16).

Python is the harness only (device memory, struct filling, CUDA-graph capture); the layer stack is
C++ (csrc/gptq_decoder.cu) over the reference's Marlin symbols' kernel (csrc/w4a16.cu).

Synthetic checkpoints follow SURVEY §8(d): `qweight` uniform u4 packed [K/8, N] i32, `scales` f16
2^U(-8,-6) [K/128, N], symmetric (`qzeros` = 0x77777777 in the checkpoint, ignored by the Marlin
path), `g_idx[k] = k/128`; dense f16 embeddings / lm_head / norms.  Load flow = the reference's
`gptq_linear` (gptq_cuda.rs:451-623): `gptq_marlin_repack` per tensor (q/k/v and gate/up are
concatenated along N first, which the row-tile format allows) — scales stay unpermuted because
this stack calls the kernel's native entry (`mrs_w4a16_gemm`, scale_perm 0)."""
import ctypes
from dataclasses import dataclass

import numpy as np
import torch

from . import lib
from .model import (MAX_PREFILL_SEQS, PagedDecodeRunner, PromptPrefill, SpecVerifier, _point, check_runner_args,
                    rope_tables, runner_split_pages)


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
               [(n, ctypes.c_void_p) for n in ("attn_norm", "ffn_norm", "k_cache", "v_cache")]


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
                                               "attn_counters", "argmax_scratch")]


def synth_gptq(K, N, group, seed, scale_exp=(-8, -6)):
    """(qweight [K/8, N] i32, scales [K/group, N] f16) per SURVEY §8(d)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    qweight = rng.integers(0, 2 ** 32, size=(K // 8, N), dtype=np.uint64).astype(np.uint32).view(np.int32)
    scales = np.exp2(rng.uniform(scale_exp[0], scale_exp[1], size=(K // group, N))).astype(np.float16)
    return qweight, scales


class GptqWeights:
    """Synthetic device-resident GPTQ checkpoint in the decode stack's layout (int4 tiles)."""
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


def _model_step(weights, k_cache, v_cache, cache_layout):
    """(layer array, mrs_gptq_step) with the model fields only: weights, norms, caches in `cache_layout` ("hnd" or
    "vllm"), dims, RoPE tables; no per-step metadata or scratch.  The layer array must outlive the struct's use."""
    cfg = weights.cfg
    layers = (_Layer * cfg.n_layers)()
    for l, L in enumerate(weights.layers):
        for f in ("wqkv", "wo", "w_gate_up", "w_down"):
            tiles, scales, K, N = L[f]
            setattr(layers[l], f, _W4(tiles.data_ptr(), scales.data_ptr(), 0, K, N))
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
        s = _Step.from_buffer_copy(runner.step_struct)   # weights, caches, shapes, tables, lengths: the runner's
        _point(s, self.meta, self.buf)
        self.step_struct = s
