"""Llama-family decode runner over the C ABI (`mrs_llama_decode_step`, include/mrs_b200_model.h).

Python here is only the harness: it allocates device memory with torch, fills the C structs with
raw pointers and drives CUDA-graph capture/replay.  The layer stack itself (which kernels run, in
which order) is C++ inside libmrs_b200.so.

Synthetic weights follow SURVEY §8(d): ggml blocks with uniformly random quants over their full
bit range, f16 scales d = 2^U(-9,-7), dmin = d*U(0,0.5); tensor-type map for Q4_K_M = the
llama.cpp recipe (Q4_K everywhere; Q6_K for `output`, and for attn_v + ffn_down on layers
i < n/8, i >= 7n/8 or (i - n/8) % 3 == 2).
"""
import ctypes
import os
from dataclasses import dataclass, field

import numpy as np
import torch

from . import BLOCK_BYTES, BLOCK_ELEMS, GGML, kv_index, lib

F16_FIELDS = {"q4_0": [0], "q4_1": [0, 2], "q5_0": [0], "q5_1": [0, 2], "q8_0": [0],
              "q2_k": [80, 82], "q3_k": [108], "q4_k": [0, 2], "q5_k": [0, 2], "q6_k": [208]}


@dataclass
class LlamaConfig:
    hidden: int = 4096
    inter: int = 14336
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: int = 8
    head_dim: int = 128
    vocab: int = 128256
    rms_eps: float = 1e-5
    rope_theta: float = 500000.0
    rope_scaling: dict = None
    max_pos: int = 8192
    quant: str = "q4_k_m"      # "q4_k_m" | any ggml type name for a uniform model
    block_size: int = 16
    name: str = "llama-3-8b"
    rope_neox: bool = True     # rotate-half pairing; GGUF llama files use the interleaved pairing (False)
    rope_freq_factors: object = None   # optional per-frequency divisors (GGUF `rope_freqs.weight`, Llama-3.1 scaling)
    synth_scale_exp: tuple = (-9, -7)  # synthetic weights: block scales d = 2^U(lo, hi) (SURVEY §8(d))

    # Real-size models take block super-scales 2^U(-15,-13): with the 6-bit sub-scales (1..63) and 4-bit
    # quants of the k-quants that gives |w| ~ 0.016, i.e. unit-scale activations at K = 4096 .. 28672.
    # SURVEY §8(d)'s 2^U(-9,-7) (|w| ~ 1) sends the 14336-wide down projection past f16's range, and the
    # Q8_1 block scale is a half (REF mmvq_gguf.cu:146-152): the reference itself would produce NaN.
    @staticmethod
    def llama3_8b(**kw):
        kw.setdefault("synth_scale_exp", (-15, -13))
        return LlamaConfig(rope_scaling=None, **kw)

    @staticmethod
    def llama3_70b(**kw):
        kw.setdefault("synth_scale_exp", (-15, -13))
        return LlamaConfig(hidden=8192, inter=28672, n_layers=80, n_heads=64, n_kv_heads=8, name="llama-3-70b", **kw)

    @staticmethod
    def tinyllama(**kw):
        return LlamaConfig(hidden=2048, inter=5632, n_layers=22, n_heads=32, n_kv_heads=4, head_dim=64, vocab=32000,
                           rope_theta=10000.0, name="tinyllama-1.1b", **kw)

    @staticmethod
    def tiny_test(**kw):
        d = dict(hidden=512, inter=1024, n_layers=3, n_heads=8, n_kv_heads=2, head_dim=64, vocab=1024,
                 rope_theta=10000.0, max_pos=512, name="tiny-test")
        d.update(kw)
        return LlamaConfig(**d)


def tensor_type(cfg: LlamaConfig, name: str, layer: int = 0) -> str:
    """ggml type of a tensor under cfg.quant (llama.cpp Q4_K_M recipe, SURVEY §8(d))."""
    if cfg.quant != "q4_k_m":
        return cfg.quant
    if name == "output":
        return "q6_k"
    if name in ("attn_v", "ffn_down"):
        n = cfg.n_layers
        if layer < n // 8 or layer >= 7 * n // 8 or (layer - n // 8) % 3 == 2:
            return "q6_k"
    return "q4_k"


TENSOR_IDS = {"attn_q": 0, "attn_k": 1, "attn_v": 2, "attn_output": 3, "ffn_gate": 4, "ffn_up": 5, "ffn_down": 6,
              "attn_norm": 7, "ffn_norm": 8, "token_embd": 9, "output": 10, "output_norm": 11}


def synth_blocks(dtype: str, nblocks: int, seed: int, scale_exp=(-9, -7)) -> np.ndarray:
    """uint8 [nblocks, block_bytes] per SURVEY §8(d), numpy PCG64(seed)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    bb = BLOCK_BYTES[dtype]
    raw = rng.integers(0, 256, size=(nblocks, bb), dtype=np.uint8)
    f = F16_FIELDS[dtype]
    d = np.exp2(rng.uniform(scale_exp[0], scale_exp[1], size=nblocks)).astype(np.float16)
    raw[:, f[0]:f[0] + 2] = d.view(np.uint8).reshape(nblocks, 2)
    if len(f) > 1:
        m = (d.astype(np.float32) * rng.uniform(0, 0.5, size=nblocks)).astype(np.float16)
        raw[:, f[1]:f[1] + 2] = m.view(np.uint8).reshape(nblocks, 2)
    return raw


def tensor_seed(layer: int, name: str) -> int:
    return 0xB200 + layer * 16 + TENSOR_IDS[name]


class _QW(ctypes.Structure):
    _fields_ = [("data", ctypes.c_void_p), ("ggml_type", ctypes.c_int32), ("rows", ctypes.c_int32),
                ("cols", ctypes.c_int32)]


class _Layer(ctypes.Structure):
    _fields_ = [(n, _QW) for n in ("wq", "wk", "wv", "wo", "w_gate", "w_up", "w_down")] + \
               [("attn_norm", ctypes.c_void_p), ("ffn_norm", ctypes.c_void_p),
                ("k_cache", ctypes.c_void_p), ("v_cache", ctypes.c_void_p)]


_AR_FN = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p)


class _Step(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("hidden", "n_layers", "n_heads", "n_kv_heads", "head_dim", "vocab",
                                              "block_size", "act_dtype")] + \
               [("rms_eps", ctypes.c_float), ("sm_scale", ctypes.c_float), ("rope_neox", ctypes.c_int32),
                ("pdl", ctypes.c_int32), ("layers", ctypes.POINTER(_Layer)), ("tok_embd", _QW), ("lm_head", _QW),
                ("final_norm", ctypes.c_void_p), ("rope_cos", ctypes.c_void_p), ("rope_sin", ctypes.c_void_p),
                ("batch", ctypes.c_int32), ("padded_tiles", ctypes.c_int32), ("max_blocks_per_seq", ctypes.c_int32),
                ("skip_mask", ctypes.c_int32), ("fused_attention", ctypes.c_int32), ("reserved0", ctypes.c_int32)] + \
               [(n, ctypes.c_void_p) for n in ("token_ids", "positions", "slot_mapping", "kv_indptr", "kv_indices",
                                               "kv_last_page_len", "request_indices", "kv_tile_indices", "o_indptr",
                                               "kv_chunk_size", "block_valid_mask", "x", "x2", "q", "k", "v",
                                               "attn_out", "act", "logits", "tmp_v", "tmp_s", "out_token",
                                               "attn_counters", "argmax_scratch")] + \
               [("all_reduce", _AR_FN), ("all_reduce_user", ctypes.c_void_p), ("tp", ctypes.c_void_p), ("h", ctypes.c_void_p)]


class _TpCtx(ctypes.Structure):
    _fields_ = [("world", ctypes.c_int32), ("rank", ctypes.c_int32), ("peer_base", ctypes.c_void_p * 8),
                ("flags_offset", ctypes.c_int64), ("slot_offset", ctypes.c_int64 * 2), ("seq_counter", ctypes.c_void_p),
                ("ll_offset", ctypes.c_int64), ("ll_slot_stride", ctypes.c_int64), ("ll_src_stride", ctypes.c_int64)]


class PeerAllReduce:
    """Symmetric buffer + peer mappings for the in-graph peer-memory all-reduce (`mrs_tp_ctx`).
    One process per GPU; the rendezvous goes through torch.distributed._symmetric_memory (plumbing:
    allocation + IPC handle exchange), the data path is our own kernel over NVLink loads."""

    def __init__(self, elems: int, dtype, device, group=None, low_latency=None):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        group = group or dist.group.WORLD
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if self.world > 8:
            raise ValueError("peer-memory all-reduce supports up to 8 ranks (one NVSwitch domain)")
        slot = (elems * torch.empty(0, dtype=dtype).element_size() + 255) // 256 * 256
        # low-latency region: [2 slots][world sources][4 bytes per element] of {element pair, sequence number} words
        if low_latency is None:
            low_latency = os.environ.get("MRS_TP_LL", "1") != "0"
        ll_src = (elems * 4 + 255) // 256 * 256 if low_latency else 0
        ll_slot = self.world * ll_src
        self.low_latency = bool(low_latency)
        self.buf = symm.empty(256 + 2 * slot + 2 * ll_slot, dtype=torch.uint8, device=device)
        self.buf.zero_()
        torch.cuda.synchronize(device)
        self.handle = symm.rendezvous(self.buf, group)
        self.seq = torch.zeros(2, dtype=torch.int32, device=device)   # [all-reduces so far, time-out flag]
        c = _TpCtx()
        c.world, c.rank = self.world, self.rank
        for r in range(self.world):
            c.peer_base[r] = int(self.handle.buffer_ptrs[r])
        c.flags_offset, c.slot_offset[0], c.slot_offset[1] = 0, 256, 256 + slot
        c.seq_counter = self.seq.data_ptr()
        if low_latency:
            c.ll_offset, c.ll_slot_stride, c.ll_src_stride = 256 + 2 * slot, ll_slot, ll_src
        self.ctx = c
        dist.barrier(group)

    def pointer(self):
        return ctypes.addressof(self.ctx)

    def timed_out(self):
        """True when a low-latency all-reduce gave up waiting for a peer (ranks out of step): results are invalid."""
        return bool(int(self.seq[1].item()) != 0)


def rope_tables(cfg: LlamaConfig):
    """cos/sin [max_pos, head_dim/2] f32 — REF mistralrs-core/src/layers.rs:1071-1160."""
    half = cfg.head_dim // 2
    inv = (1.0 / np.power(np.float32(cfg.rope_theta), np.arange(0, cfg.head_dim, 2, dtype=np.float32) / np.float32(cfg.head_dim))).astype(np.float32)
    sc = cfg.rope_scaling
    if sc is not None:
        low_wl = np.float32(sc["original_max_position_embeddings"]) / np.float32(sc["low_freq_factor"])
        high_wl = np.float32(sc["original_max_position_embeddings"]) / np.float32(sc["high_freq_factor"])
        out = []
        for f in inv:
            wl = np.float32(2 * np.pi) / f
            if wl < high_wl:
                out.append(f)
            elif wl > low_wl:
                out.append(f / np.float32(sc["factor"]))
            else:
                smooth = (np.float32(sc["original_max_position_embeddings"]) / wl - np.float32(sc["low_freq_factor"])) / \
                         (np.float32(sc["high_freq_factor"]) - np.float32(sc["low_freq_factor"]))
                out.append((1 - smooth) * f / np.float32(sc["factor"]) + smooth * f)
        inv = np.array(out, dtype=np.float32)
    if cfg.rope_freq_factors is not None:   # llama.cpp stores Llama-3.1's scaling as theta / factor per frequency
        inv = (inv / np.asarray(cfg.rope_freq_factors, dtype=np.float32)).astype(np.float32)
    freqs = np.arange(cfg.max_pos, dtype=np.float32)[:, None] * inv[None, :]
    assert freqs.shape[1] == half
    return np.cos(freqs).astype(np.float32), np.sin(freqs).astype(np.float32)


def compute_kv_shard(total_kv_heads: int, head_dim: int, rank: int, world: int):
    """Rows of a K / V projection kept by `rank`: (first_row, rows).  REF mistralrs-quant/src/distributed/layers.rs:2692-2715
    (`compute_kv_shard`): KV heads are split over the ranks; when there are more ranks than KV heads every head is
    REPLICATED on world / kv_heads consecutive ranks (each rank then holds exactly one)."""
    if world == 1:
        return 0, total_kv_heads * head_dim
    if world > total_kv_heads:
        if world % total_kv_heads:
            raise ValueError(f"tensor-parallel size {world} must be a multiple of the {total_kv_heads} KV heads to replicate them")
        replicate = world // total_kv_heads
        return (rank // replicate) * head_dim, head_dim
    if total_kv_heads % world:
        raise ValueError(f"tensor-parallel size {world} must divide the {total_kv_heads} KV heads")
    per = total_kv_heads // world
    return rank * per * head_dim, per * head_dim


def compute_n_kv_groups(total_kv_heads: int, n_heads: int, world: int) -> int:
    """Query heads per local KV head under KV-head replication.  REF distributed/layers.rs:2718-2733."""
    replicate = world // total_kv_heads if world > total_kv_heads else 1
    return (n_heads // total_kv_heads) // replicate if replicate else n_heads // total_kv_heads


class LlamaWeights:
    """Synthetic device-resident weights (optionally one tensor-parallel shard)."""

    # the quantized tensors of a layer and how tensor parallelism splits them (see _shard)
    GGUF_NAMES = {"attn_q": "col", "attn_k": "kv", "attn_v": "kv", "attn_output": "row", "ffn_gate": "col",
                  "ffn_up": "col", "ffn_down": "row"}

    def __init__(self, cfg: LlamaConfig, device, dtype=torch.bfloat16, tp_rank=0, tp_size=1, keep_host=False, fast_synth=False):
        """fast_synth: generate the (shard-shaped) blocks on the device with torch's RNG instead of numpy
        PCG64 on the host — same distribution, not the SURVEY §8(d) byte stream; for throughput runs of
        large models (config 3's 8 GB, config 5's 40 GB) where no oracle comparison is made."""
        if fast_synth and keep_host:
            raise ValueError("fast_synth weights have no host copy")
        self._setup(cfg, device, dtype, tp_rank, tp_size, keep_host)
        self.fast_synth = bool(fast_synth)
        H, I = cfg.hidden, cfg.inter
        if I % (tp_size * 256):
            raise ValueError("tensor-parallel size must divide the intermediate size in 256-wide slices")
        nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
        shape = {"attn_q": (nq, H), "attn_k": (nkv, H), "attn_v": (nkv, H), "attn_output": (H, nq), "ffn_gate": (I, H),
                 "ffn_up": (I, H), "ffn_down": (H, I), "token_embd": (cfg.vocab, H), "output": (cfg.vocab, H)}
        self._load(lambda l, name, kind: self._qtensor(l, name, *shape[name], kind), self._norm)

    def _setup(self, cfg, device, dtype, tp_rank, tp_size, keep_host):
        self.cfg, self.device, self.dtype = cfg, device, dtype
        self.tp_rank, self.tp_size = tp_rank, tp_size
        self.host = {} if keep_host else None
        self.layers, self.nbytes = [], 0
        if cfg.n_heads % tp_size:
            raise ValueError("tensor-parallel size must divide the head counts")
        compute_kv_shard(cfg.n_kv_heads, cfg.head_dim, tp_rank, tp_size)      # raises on an impossible KV head layout

    def _load(self, qtensor, norm):
        """Fills layers, tok_embd, output, output_norm and the RoPE tables.  qtensor(layer, name, kind) and
        norm(layer, name) return one tensor of the source under its GGUF name (token_embd, output and output_norm
        come as layer 0)."""
        for l in range(self.cfg.n_layers):
            L = {name: qtensor(l, name, kind) for name, kind in self.GGUF_NAMES.items()}
            for name in ("attn_norm", "ffn_norm"):
                L[name] = norm(l, name)
            self.layers.append(L)
        self.tok_embd = qtensor(0, "token_embd", "rep")
        self.output = qtensor(0, "output", "rep")
        self.output_norm = norm(0, "output_norm")
        cos, sin = rope_tables(self.cfg)
        self.rope_cos = torch.from_numpy(cos).to(self.device).to(self.dtype)
        self.rope_sin = torch.from_numpy(sin).to(self.device).to(self.dtype)

    # ---- real weights -------------------------------------------------------------------------
    @staticmethod
    def config_from_gguf(ar) -> "LlamaConfig":
        """Hyper-parameters from GGUF metadata (`llama.*` keys, as the reference's
        `quantized_llama.rs::PropsGGUF` reads them)."""
        md = ar.metadata()
        arch = md.get("general.architecture", "llama")

        def g(key, default=None):
            v = md.get(f"{arch}.{key}", default)
            if v is None:
                raise KeyError(f"GGUF metadata key `{arch}.{key}` is missing")
            return v
        hidden, n_heads = int(g("embedding_length")), int(g("attention.head_count"))
        head_dim = int(md.get(f"{arch}.attention.key_length", md.get(f"{arch}.rope.dimension_count", hidden // n_heads)))
        emb = ar.tensor_info("token_embd.weight")
        factors = None
        if ar.contains_tensor("rope_freqs.weight"):
            factors = ar.load_dense("rope_freqs.weight", "cpu").float().numpy()
        return LlamaConfig(hidden=hidden, inter=int(g("feed_forward_length")), n_layers=int(g("block_count")),
                           n_heads=n_heads, n_kv_heads=int(g("attention.head_count_kv", n_heads)), head_dim=head_dim,
                           vocab=int(md.get(f"{arch}.vocab_size", emb.shape[0])),
                           rms_eps=float(g("attention.layer_norm_rms_epsilon", 1e-5)),
                           rope_theta=float(g("rope.freq_base", 10000.0)), rope_scaling=None,
                           max_pos=int(g("context_length", 4096)), quant="gguf",
                           name=str(md.get("general.name", arch)), rope_neox=False, rope_freq_factors=factors)

    @classmethod
    def from_gguf(cls, ar, device, dtype=torch.bfloat16, tp_rank=0, tp_size=1, keep_host=False, max_pos=None):
        """Device-resident weights of a llama-architecture GGUF archive (`gguf_file.GgufArchive`):
        ggml blocks uploaded as stored (column/row TP shards cut on block boundaries, as for the
        synthetic model), norm vectors converted to the activation dtype, `output.weight` falling
        back to the tied `token_embd.weight`.  Tensor names: llama.cpp's (`blk.N.attn_q.weight` …)."""
        self = cls.__new__(cls)
        cfg = cls.config_from_gguf(ar)
        if max_pos is not None:
            cfg.max_pos = int(max_pos)
        self._setup(cfg, device, dtype, tp_rank, tp_size, keep_host)
        top = {"token_embd": "token_embd.weight", "output_norm": "output_norm.weight",
               "output": "output.weight" if ar.contains_tensor("output.weight") else "token_embd.weight"}
        src = lambda l, name: top.get(name) or f"blk.{l}.{name}.weight"
        self._load(lambda l, name, kind: self._gguf_qtensor(ar, src(l, name), (l, name), kind),
                   lambda l, name: self._put_norm(ar.load_dense(src(l, name), device, dtype), (l, name)))
        return self

    UQFF_NAMES = {"attn_q": "self_attn.q_proj", "attn_k": "self_attn.k_proj", "attn_v": "self_attn.v_proj",
                  "attn_output": "self_attn.o_proj", "ffn_gate": "mlp.gate_proj", "ffn_up": "mlp.up_proj",
                  "ffn_down": "mlp.down_proj"}

    @staticmethod
    def config_from_hf(cj: dict) -> "LlamaConfig":
        """Hyper-parameters from a Hugging Face `config.json` (llama family), the source the
        reference's non-GGUF loaders read (`models/llama.rs::Config`)."""
        heads = int(cj["num_attention_heads"])
        sc = cj.get("rope_scaling")
        if sc is not None:
            kind = sc.get("rope_type", sc.get("type"))
            if kind != "llama3":
                raise NotImplementedError(f"rope_scaling type {kind!r} is not supported (llama3 only)")
            sc = {k: sc[k] for k in ("factor", "low_freq_factor", "high_freq_factor", "original_max_position_embeddings")}
        return LlamaConfig(hidden=int(cj["hidden_size"]), inter=int(cj["intermediate_size"]),
                           n_layers=int(cj["num_hidden_layers"]), n_heads=heads,
                           n_kv_heads=int(cj.get("num_key_value_heads", heads)),
                           head_dim=int(cj.get("head_dim") or int(cj["hidden_size"]) // heads), vocab=int(cj["vocab_size"]),
                           rms_eps=float(cj.get("rms_norm_eps", 1e-5)), rope_theta=float(cj.get("rope_theta", 10000.0)),
                           rope_scaling=sc, max_pos=int(cj.get("max_position_embeddings", 4096)), quant="uqff",
                           name=str(cj.get("_name_or_path") or cj.get("model_type", "llama")), rope_neox=True)

    @classmethod
    def from_uqff(cls, ar, device, dtype=torch.bfloat16, tp_rank=0, tp_size=1, keep_host=False, max_pos=None):
        """Device-resident weights of a UQFF artifact (`uqff_file.UqffArchive`): GGML-family layer
        entries uploaded as stored, norms from `residual.safetensors`, hyper-parameters from
        `config.json`; Hugging Face tensor paths (`model.layers.N.self_attn.q_proj` …) and the
        rotate-half RoPE pairing, so the fused attention path applies."""
        if ar.config is None:
            raise ValueError("UQFF artifact has no config.json next to its shards")
        if not ar.contains("model.embed_tokens.weight.format"):
            raise NotImplementedError("this UQFF artifact keeps dense token embeddings in residual.safetensors (UQFF <= 1.1); "
                                      "the embedding gather kernel takes ggml block types")
        self = cls.__new__(cls)
        cfg = cls.config_from_hf(ar.config)
        if max_pos is not None:
            cfg.max_pos = int(max_pos)
        self._setup(cfg, device, dtype, tp_rank, tp_size, keep_host)
        tied = bool(ar.config.get("tie_word_embeddings", False)) or not ar.contains("lm_head.weight.format")
        top = {"token_embd": "model.embed_tokens", "output": "model.embed_tokens" if tied else "lm_head",
               "output_norm": "model.norm.weight"}
        names = dict(cls.UQFF_NAMES, attn_norm="input_layernorm.weight", ffn_norm="post_attention_layernorm.weight")
        src = lambda l, name: top.get(name) or f"model.layers.{l}.{names[name]}"
        self._load(lambda l, name, kind: self._uqff_qtensor(ar, src(l, name), (l, name), kind),
                   lambda l, name: self._put_norm(ar.load_tensor(src(l, name), device, dtype), (l, name)))
        return self

    def _uqff_qtensor(self, ar, key_path, key, kind):
        q = ar.load_qtensor(key_path, "cpu")
        rows, cols = q.shape
        blocks = q.data.numpy().reshape(rows, cols // BLOCK_ELEMS[q.dtype], BLOCK_BYTES[q.dtype])
        return self._upload(blocks, q.dtype, kind, key)

    def _gguf_qtensor(self, ar, name, key, kind):
        info = ar.tensor_info(name)
        if info.dtype not in BLOCK_BYTES:
            raise NotImplementedError(f"GGUF tensor `{name}` is {info.dtype}: the decode kernels take ggml block types "
                                      f"({', '.join(sorted(BLOCK_BYTES))})")
        if len(info.shape) != 2:
            raise ValueError(f"GGUF tensor `{name}` must be a matrix, got shape {info.shape}")
        rows, cols = info.shape
        blocks = ar.tensor_data(name).reshape(rows, cols // BLOCK_ELEMS[info.dtype], BLOCK_BYTES[info.dtype])
        return self._upload(blocks, info.dtype, kind, key)

    def _shard(self, rows, cols, be, kind):
        """This rank's part of a [rows, cols] matrix of `be`-element blocks: (row slice, block-column slice).
        kind: 'col' (rows sharded), 'kv' (rows sharded by KV head, replicated when ranks outnumber KV heads),
        'row' (K sharded on block boundaries), 'rep' (replicated).  Sharding rules: REF
        mistralrs-quant/src/distributed/layers.rs:1167-1294 (column), :695-975 (row), gguf/weight_source.rs:809-818
        (block-aligned K slices)."""
        r, w = self.tp_rank, self.tp_size
        nb = cols // be
        if kind == "kv" and w > 1:
            first, n = compute_kv_shard(self.cfg.n_kv_heads, self.cfg.head_dim, r, w)
            return slice(first, first + n), slice(0, nb)
        if kind == "col" and w > 1:
            if rows % w:
                raise ValueError("column-parallel rows do not divide by the tensor-parallel size")
            return slice(r * rows // w, (r + 1) * rows // w), slice(0, nb)
        if kind == "row" and w > 1:
            if nb % w:
                raise ValueError("row-parallel K does not split on block boundaries")
            return slice(0, rows), slice(r * nb // w, (r + 1) * nb // w)
        return slice(0, rows), slice(0, nb)

    def _upload(self, blocks, ggml_type, kind, key):
        """ggml blocks [rows, cols / block, block_bytes] -> (device tensor, type, rows, cols) of this rank's shard,
        counted in nbytes and kept in host[key] under keep_host.  A read-only source (an archive's mapping, which
        closes with the archive) is copied first."""
        be = BLOCK_ELEMS[ggml_type]
        rs, ks = self._shard(blocks.shape[0], blocks.shape[1] * be, be, kind)
        flat = np.ascontiguousarray(blocks[rs, ks]).reshape(-1)
        if not flat.flags.writeable:
            flat = flat.copy()
        t = torch.from_numpy(flat).to(self.device)
        self.nbytes += t.numel()
        if self.host is not None:
            self.host[key] = flat
        return (t, ggml_type, rs.stop - rs.start, (ks.stop - ks.start) * be)

    def _put_norm(self, t, key):
        """a norm vector already in the activation dtype on the device, flattened; host[key] keeps it in f32"""
        t = t.reshape(-1).contiguous()
        if self.host is not None:
            self.host[key] = t.float().cpu().numpy()
        return t

    def _norm(self, layer, name):
        rng = np.random.Generator(np.random.PCG64(tensor_seed(layer, name)))
        w = (1.0 + 0.1 * rng.standard_normal(self.cfg.hidden)).astype(np.float32)
        return self._put_norm(torch.from_numpy(w).to(self.device).to(self.dtype), (layer, name))

    def _qtensor(self, layer, name, rows, cols, kind):
        dt = tensor_type(self.cfg, name, layer)
        be, bb = BLOCK_ELEMS[dt], BLOCK_BYTES[dt]
        if self.fast_synth:
            rs, ks = self._shard(rows, cols, be, kind)
            rows, cols = rs.stop - rs.start, (ks.stop - ks.start) * be
            nblocks = rows * cols // be
            gen = torch.Generator(device=self.device).manual_seed(tensor_seed(layer, name) * 64 + self.tp_rank)
            raw = torch.randint(0, 256, (nblocks, bb), dtype=torch.uint8, device=self.device, generator=gen)
            lo, hi = self.cfg.synth_scale_exp
            f = F16_FIELDS[dt]
            d = torch.exp2(torch.empty(nblocks, device=self.device).uniform_(lo, hi, generator=gen)).to(torch.float16)
            raw[:, f[0]:f[0] + 2] = d.view(torch.uint8).reshape(nblocks, 2)
            if len(f) > 1:
                m = (d.float() * torch.empty(nblocks, device=self.device).uniform_(0, 0.5, generator=gen)).to(torch.float16)
                raw[:, f[1]:f[1] + 2] = m.view(torch.uint8).reshape(nblocks, 2)
            t = raw.reshape(-1)
            self.nbytes += t.numel()
            return (t, dt, rows, cols)
        full = synth_blocks(dt, rows * cols // be, tensor_seed(layer, name), self.cfg.synth_scale_exp).reshape(rows, cols // be, bb)
        return self._upload(full, dt, kind, (layer, name))


def runner_split_pages(block_size, batch, n_kv_heads, max_ctx, sm_count=132, min_tokens=64):
    """Split-KV chunk (in pages) for the whole-token decode path: enough tiles that
    batch x kv_heads x tiles covers the SMs (one attention CTA per SM), chunks of at least
    `min_tokens`.  The reference's host policy (metadata.rs:61-86, kv_index.decode_split_pages) never
    goes below 256-token chunks, which leaves 16 CTAs for a batch-1 8-KV-head decode; the kernels
    accept any plan, this one only changes how finely the same sum is split."""
    tiles = max(1, sm_count // max(1, batch * n_kv_heads))
    tokens = max(min_tokens, -(-max_ctx // tiles))
    return max(1, -(-tokens // block_size))


MAX_DECODE_BATCH = 256   # sequences per decode step (mrs_decode_advance / mrs_llama_decode_step)
MMVQ_MAX_BATCH = 8       # up to this many rows the linears are GEMVs; above, the dequant GEMM (the reference's MMQ branch)


def check_runner_args(batch, comm=None, peer_allreduce=None):
    """ValueError for a decode batch the decode steps reject: outside 1..256, or tensor parallel above 8 rows."""
    if isinstance(batch, bool) or not isinstance(batch, (int, np.integer)) or not 1 <= batch <= MAX_DECODE_BATCH:
        raise ValueError(f"decode batch must be an int in 1..{MAX_DECODE_BATCH}, got {batch!r}")
    if batch > MMVQ_MAX_BATCH and (comm is not None or peer_allreduce is not None):
        raise ValueError(f"LlamaRunner: tensor parallelism (comm / peer_allreduce) runs batches of up to {MMVQ_MAX_BATCH}, "
                         f"got {batch}")


def _point(struct, *tensor_dicts):
    """struct.<name> <- the device address of every tensor (None: NULL) in the dicts"""
    for d in tensor_dicts:
        for n, t in d.items():
            setattr(struct, n, None if t is None else t.data_ptr())


class PagedDecodeRunner:
    """The paged-KV side of a decode runner over `weights` (LlamaRunner, GptqRunner): block pool, per-sequence block
    tables and context lengths, the split-KV plan, the index metadata and its advance (mrs_decode_advance_multi), the
    host-side bound on the context, and CUDA-graph capture / replay of step().  A subclass checks its arguments first
    (check_runner_args), then adds its KV caches, scratch (`buf`) and step struct (`step_struct`) and implements
    forward()."""
    KEEP_GRAPH = False     # capture with keep_graph=True, so the kernel nodes can be counted afterwards

    def __init__(self, weights, batch, max_ctx, split_pages):
        """split_pages: split-KV chunk in pages, 0 for the unsplit plan (also taken when each sequence fits one chunk)"""
        cfg, dev = weights.cfg, weights.device
        self.w, self.cfg, self.dev, self.dt, self.B = weights, cfg, dev, weights.dtype, int(batch)
        self.max_blocks = -(-max_ctx // cfg.block_size)
        self.pool = kv_index.BlockPool(self.B * self.max_blocks + 1)
        self.tables = [self.pool.get_new_blocks(self.max_blocks) for _ in range(self.B)]
        self.block_tables = torch.tensor(self.tables, dtype=torch.int32, device=dev)
        self.context_lens = torch.zeros(self.B, dtype=torch.int32, device=dev)
        self.error_flag = torch.zeros(1, dtype=torch.int32, device=dev)   # bit 0: a sequence ran out of context
        self.max_ctx = min(self.max_blocks * cfg.block_size, cfg.max_pos)
        self.steps_taken = 0              # host-side count of advances since reset() (graph replays via replay())
        self.split_pages = split_pages
        self.padded_tiles = self.B * -(-self.max_blocks // split_pages) if split_pages else self.B
        if self.padded_tiles <= self.B:        # a single chunk per request: unsplit plan
            self.split_pages, self.padded_tiles = 0, self.B
        self.meta = self.decode_meta(1)
        self.graph = None

    def decode_meta(self, q):
        """the index metadata of a step that feeds q rows per sequence, over this runner's tables and plan"""
        B, R, P = self.B, self.B * q, self.padded_tiles
        z = lambda *s, d=torch.int32: torch.zeros(*s, dtype=d, device=self.dev)
        return dict(token_ids=z(R), positions=z(R), slot_mapping=z(R, d=torch.int64), kv_indptr=z(B + 1),
                    kv_indices=z(B * self.max_blocks), kv_last_page_len=z(B), request_indices=z(P), kv_tile_indices=z(P),
                    o_indptr=z(B + 1), kv_chunk_size=z(1), block_valid_mask=z(P, d=torch.uint8))

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def _advance(self, meta, q):
        """enqueue the advance of every sequence by q rows, writing `meta` (see decode_meta)"""
        rc = lib().mrs_decode_advance_multi(
            ctypes.c_void_p(self.block_tables.data_ptr()), ctypes.c_int(self.max_blocks),
            ctypes.c_void_p(self.context_lens.data_ptr()), ctypes.c_int(self.B), ctypes.c_int(self.cfg.block_size),
            ctypes.c_int(self.split_pages), ctypes.c_int(self.padded_tiles),
            *[ctypes.c_void_p(meta[n].data_ptr()) for n in ("positions", "slot_mapping", "kv_indptr", "kv_indices",
                                                            "kv_last_page_len", "request_indices", "kv_tile_indices",
                                                            "o_indptr", "kv_chunk_size", "block_valid_mask")],
            ctypes.c_int(self.cfg.max_pos), ctypes.c_void_p(self.error_flag.data_ptr()), ctypes.c_int(q), self._stream())
        if rc != 0:
            raise RuntimeError(f"mrs_decode_advance_multi failed: cudaError {rc}")

    def advance(self):
        self._advance(self.meta, 1)
        self.steps_taken += 1

    def step(self):
        """advance the KV metadata for the token in `token_ids`, run the stack, argmax -> token_ids."""
        if self.steps_taken >= self.max_ctx and not torch.cuda.is_current_stream_capturing():
            raise RuntimeError(f"{type(self).__name__}: context exhausted ({self.max_ctx} tokens: block table / RoPE table)")
        self.advance()
        self.forward()

    def reset(self, context_len=0):
        """context_len: one length for every sequence, or a sequence of B lengths (sequences at different positions,
        e.g. prompts of different lengths prefilled into their own tables).  The host-side bound on further steps
        follows the longest."""
        if isinstance(context_len, (int, np.integer)):
            self.context_lens.fill_(int(context_len))
            longest = int(context_len)
        else:
            lens = [int(c) for c in context_len]
            if len(lens) != self.B or min(lens) < 0:
                raise ValueError(f"{type(self).__name__}.reset: need {self.B} lengths >= 0, got {lens}")
            self.context_lens.copy_(torch.tensor(lens, dtype=torch.int32))
            longest = max(lens)
        self.error_flag.zero_()
        self.steps_taken = longest

    def replay(self):
        """one captured decode step; raises before a sequence would run past the allocated context
        (the kernels freeze such a sequence and set error_flag, but a caller should never get there)"""
        if self.steps_taken >= self.max_ctx:
            raise RuntimeError(f"{type(self).__name__}: context exhausted ({self.max_ctx} tokens: block table / RoPE table)")
        self.steps_taken += 1
        self.graph.replay()

    def check_overflow(self):
        if int(self.error_flag.item()) & 1:
            raise RuntimeError(f"{type(self).__name__}: a sequence ran past its allocated context (KV write skipped)")

    def capture(self):
        self.step(); self.reset()  # warm-up outside capture (module load, attributes)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph(keep_graph=self.KEEP_GRAPH)
        with torch.cuda.graph(g):
            self.step()
        self.reset()
        self.graph = g
        return g

    def set_tokens(self, ids):
        self.meta["token_ids"].copy_(torch.as_tensor(ids, dtype=torch.int32, device=self.dev))

    def logits(self):
        return self.buf["logits"]


class LlamaRunner(PagedDecodeRunner):
    """Owns KV cache + scratch + per-step metadata for a batch of sequences and drives
    mrs_llama_decode_step / mrs_decode_advance_multi (eagerly or as a captured CUDA graph).
    batch 1..8 runs the GEMV chain, 9..256 the dequant-GEMM chain (prefill numerics; see mrs_b200_model.h)."""
    KEEP_GRAPH = True

    def __init__(self, weights: LlamaWeights, batch=1, max_ctx=512, pdl=False, sm_count=132, comm=None,
                 fused_attention=True, split_policy="sm_fill", split_min_tokens=64, peer_allreduce=None):
        check_runner_args(batch, comm, peer_allreduce)
        cfg, tp, bs = weights.cfg, weights.tp_size, weights.cfg.block_size
        n_kv = max(1, cfg.n_kv_heads // tp)   # (KV heads are replicated when tp > kv heads)
        super().__init__(weights, batch, max_ctx,
                         kv_index.decode_split_pages(bs, batch, n_kv, max_ctx, sm_count=sm_count) if split_policy == "reference"
                         else runner_split_pages(bs, batch, n_kv, max_ctx, sm_count, split_min_tokens))
        batch, dev, dt, nb = self.B, self.dev, self.dt, self.B * self.max_blocks + 1
        self.n_heads, self.n_kv = cfg.n_heads // tp, n_kv
        a = lambda *s: torch.zeros(*s, dtype=dt, device=dev)
        H = cfg.hidden
        self.buf = dict(x=a(batch, H), x2=a(batch, H), q=a(batch, self.n_heads * cfg.head_dim),
                        k=a(batch, self.n_kv * cfg.head_dim), v=a(batch, self.n_kv * cfg.head_dim),
                        attn_out=a(batch, self.n_heads * cfg.head_dim), act=a(batch, cfg.inter // tp),
                        logits=a(batch, cfg.vocab), tmp_v=a(self.padded_tiles, self.n_heads, cfg.head_dim),
                        tmp_s=torch.zeros(self.padded_tiles, self.n_heads, dtype=torch.float32, device=dev),
                        out_token=self.meta["token_ids"],  # argmax feeds the next step directly
                        attn_counters=torch.zeros(batch * self.n_kv * 2, dtype=torch.int32, device=dev),
                        argmax_scratch=torch.zeros(16 * batch + 16, dtype=torch.uint8, device=dev),
                        h=a(batch, H))
        self.k_cache = [a(nb, self.n_kv, bs, cfg.head_dim) for _ in range(cfg.n_layers)]
        self.v_cache = [a(nb, self.n_kv, bs, cfg.head_dim) for _ in range(cfg.n_layers)]
        self._layers, s = _model_step(weights, self.k_cache, self.v_cache, pdl, self.n_heads, self.n_kv)
        s.batch, s.padded_tiles, s.max_blocks_per_seq = batch, self.padded_tiles, self.max_blocks
        s.fused_attention = int(fused_attention)
        _point(s, self.meta, self.buf)
        self._ar_cb, self._peer = None, peer_allreduce
        if peer_allreduce is not None:     # in-graph peer-memory sum (takes precedence over the callback)
            s.tp = peer_allreduce.pointer()
        if comm is not None:
            self._ar_cb = _AR_FN(comm)
            s.all_reduce = self._ar_cb
        self.step_struct = s

    def forward(self):
        rc = lib().mrs_llama_decode_step(ctypes.byref(self.step_struct), self._stream())
        if rc != 0:
            raise RuntimeError(f"mrs_llama_decode_step failed: cudaError {rc}")


MAX_PREFILL_SEQS = 256   # sequences per prompt step (mrs_llama_prefill_step)
PREFILL_GROUPED_MAX_ROWS = 2048   # above: separate QKV and gate / up GEMMs (needs the gate_up scratch)


class _Prefill(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("n_seqs", "total_tokens", "max_q_len", "max_kv_len", "paged", "lm_rows",
                                              "block_table_stride", "num_blocks")] + \
               [(n, ctypes.c_void_p) for n in ("token_ids", "positions", "slot_mapping", "cu_seqlens_q", "cu_seqlens_k",
                                               "block_tables", "last_rows", "x", "x2", "h", "q", "k", "v", "attn_out", "act",
                                               "gate_up", "h_last", "logits", "out_token", "argmax_scratch", "q8_scratch", "dest_rows",
                                               "runner_token_ids", "runner_context_lens")]


def _model_step(weights, k_cache, v_cache, pdl, n_heads, n_kv_heads):
    """(layer array, mrs_llama_step) with the model fields only: weights, norms, caches, dims (local head counts under
    tensor parallelism), RoPE tables; no per-step metadata or scratch.  The layer array must outlive the struct's use."""
    cfg = weights.cfg
    layers = (_Layer * cfg.n_layers)()
    for l, L in enumerate(weights.layers):
        for field_, name in (("wq", "attn_q"), ("wk", "attn_k"), ("wv", "attn_v"), ("wo", "attn_output"),
                             ("w_gate", "ffn_gate"), ("w_up", "ffn_up"), ("w_down", "ffn_down")):
            t, ty, rows, cols = L[name]
            setattr(layers[l], field_, _QW(t.data_ptr(), GGML[ty], rows, cols))
        layers[l].attn_norm, layers[l].ffn_norm = L["attn_norm"].data_ptr(), L["ffn_norm"].data_ptr()
        layers[l].k_cache, layers[l].v_cache = k_cache[l].data_ptr(), v_cache[l].data_ptr()
    s = _Step()
    s.hidden, s.n_layers, s.n_heads, s.n_kv_heads, s.head_dim, s.vocab = (cfg.hidden, cfg.n_layers, n_heads, n_kv_heads,
                                                                          cfg.head_dim, cfg.vocab)
    s.block_size, s.act_dtype = cfg.block_size, {torch.float16: 0, torch.bfloat16: 1}[weights.dtype]
    s.rms_eps, s.sm_scale, s.rope_neox, s.pdl = cfg.rms_eps, 1.0 / float(np.sqrt(cfg.head_dim)), int(cfg.rope_neox), int(pdl)
    s.layers = ctypes.cast(layers, ctypes.POINTER(_Layer))
    for field_, (t, ty, rows, cols) in (("tok_embd", weights.tok_embd), ("lm_head", weights.output)):
        setattr(s, field_, _QW(t.data_ptr(), GGML[ty], rows, cols))
    s.final_norm, s.rope_cos, s.rope_sin = weights.output_norm.data_ptr(), weights.rope_cos.data_ptr(), weights.rope_sin.data_ptr()
    return layers, s


class PromptPrefill:
    """The host side of a batched prompt step (`mrs_llama_prefill` plan, include/mrs_b200_model.h), shared by
    LlamaPrefill and GptqPrefill: argument checks, the plan, its upload, the hand-off to a decode runner's rows, and the
    KV caches (a decode runner's, or the prefill's own HND caches).  A subclass calls `_init_caches`, then adds its
    scratch (`buf`), its step struct (`step_struct`) and the name of its C entry (`STEP`)."""
    STEP = None

    def _init_caches(self, weights, max_tokens, runner):
        """max_tokens: new rows per call (all sequences together).  runner: write prompts' K/V into this decode runner's
        paged cache (sequence 0's block table by default), in its layout; without one, the prefill owns HND caches."""
        cfg, dev, dt = weights.cfg, weights.device, weights.dtype
        self.w, self.cfg, self.dev, self.dt = weights, cfg, dev, dt
        bs = cfg.block_size
        self.max_tokens = int(max_tokens)
        self.nblocks = -(-self.max_tokens // bs)
        self.runner = runner
        if runner is not None:
            if runner.max_blocks < self.nblocks:
                raise ValueError(f"{type(self).__name__}: the runner's block table is shorter than max_tokens")
            self.table, self.k_cache, self.v_cache = list(runner.tables[0]), runner.k_cache, runner.v_cache
        else:
            nb = self.nblocks + 1                                   # block 0 stays the null block
            self.table = list(range(1, self.nblocks + 1))
            self.k_cache = [torch.zeros(nb, cfg.n_kv_heads, bs, cfg.head_dim, dtype=dt, device=dev) for _ in range(cfg.n_layers)]
            self.v_cache = [torch.zeros(nb, cfg.n_kv_heads, bs, cfg.head_dim, dtype=dt, device=dev) for _ in range(cfg.n_layers)]
        self.num_cache_blocks = self.k_cache[0].shape[0]
        # first tokens [256], then a copy of the runner's context lengths: one D2H copy returns both
        self._out = torch.zeros(MAX_PREFILL_SEQS + (runner.B if runner is not None else 0), dtype=torch.int32, device=dev)

    def forward(self, tokens, all_logits=False, cached=0, table=None):
        """tokens: list[int] (1 < len <= max_tokens), the prompt at positions cached .. cached + T - 1.  Returns logits
        [vocab] of the last token, or [T, vocab] with all_logits=True.  The KV cache of every layer holds rows
        cached .. cached + T - 1 afterwards.
        cached > 0: rows 0 .. cached - 1 are already in the cache under `table` (a prefix-cache hit, or the earlier
        chunks of a chunked prompt); only `tokens` are computed, and they attend to all cached + T keys through the
        paged prefill kernel.  Then T == 1 is allowed.  table: block ids of the sequence (e.g.
        `KVCacheManager.get_block_ids`), default the prefill's own table or the runner's."""
        cfg = self.cfg
        T, cached = len(tokens), int(cached)
        bs = cfg.block_size
        if cached == 0 and table is None:
            if not 1 < T <= min(self.max_tokens, cfg.max_pos):
                raise ValueError(f"{type(self).__name__}.forward: need 1 < tokens <= {min(self.max_tokens, cfg.max_pos)}, got {T}")
        else:
            end = cached + T
            tb = self.table if table is None else table
            if cached < 0 or not (1 if cached else 2) <= T <= self.max_tokens:
                raise ValueError(f"{type(self).__name__}.forward: need cached >= 0 and {1 if cached else 2} <= tokens <= "
                                 f"{self.max_tokens}, got cached={cached}, {T} tokens")
            if end > min(cfg.max_pos, len(tb) * bs):
                raise ValueError(f"{type(self).__name__}.forward: cached + tokens = {end} exceeds max_pos {cfg.max_pos} or the "
                                 f"table's {len(tb)} blocks of {bs}")
        table = self.table if table is None else [int(b) for b in table]
        logits = self._step([tokens], [cached], [table], lm_rows=2 if all_logits else 1)
        return logits if all_logits else logits[0]

    def check_batch_args(self, prompts, cached=None, tables=None, slots=None, final=True):
        """ValueError for a forward_batch call the step cannot take; returns (token id arrays, cached, tables).  Uses only
        cfg, max_tokens, table and (optional) runner."""
        cfg, bs = self.cfg, self.cfg.block_size
        runner = getattr(self, "runner", None)
        n = len(prompts)
        if not 1 <= n <= MAX_PREFILL_SEQS:
            raise ValueError(f"{type(self).__name__}.forward_batch: need 1..{MAX_PREFILL_SEQS} sequences, got {n}")
        ids = []
        for p in prompts:
            a = p.cpu().numpy() if torch.is_tensor(p) else np.asarray(p)
            a = a.reshape(-1)
            if a.size and (a.dtype.kind not in "iu" or int(a.min()) < 0 or int(a.max()) >= cfg.vocab):
                raise ValueError(f"{type(self).__name__}.forward_batch: token ids must be integers in [0, {cfg.vocab})")
            ids.append(a.astype(np.int32))
        cached = [0] * n if cached is None else [int(c) for c in cached]
        if len(cached) != n:
            raise ValueError(f"{type(self).__name__}.forward_batch: {len(cached)} cached lengths for {n} sequences")
        if slots is not None:
            if not final:
                raise ValueError(f"{type(self).__name__}.forward_batch: slots commit first tokens, which a non-final chunk has none of")
            if runner is None:
                raise ValueError(f"{type(self).__name__}.forward_batch: slots need a {type(self).__name__} built with a runner")
            slots = [int(s) for s in slots]
            if len(slots) != n:
                raise ValueError(f"{type(self).__name__}.forward_batch: {len(slots)} slots for {n} sequences")
            if len(set(slots)) != n or min(slots) < 0 or max(slots) >= runner.B:
                raise ValueError(f"{type(self).__name__}.forward_batch: slots must be distinct runner rows in 0..{runner.B - 1}")
        if tables is None:
            if slots is not None:
                tables = [list(runner.tables[s]) for s in slots]
            elif n == 1:
                tables = [self.table]
            elif runner is not None and n <= runner.B:
                tables = [list(runner.tables[i]) for i in range(n)]
            else:
                raise ValueError(f"{type(self).__name__}.forward_batch: several sequences need their own tables (tables= or a runner)")
        tables = [[int(b) for b in t] for t in tables]
        if len(tables) != n:
            raise ValueError(f"{type(self).__name__}.forward_batch: {len(tables)} tables for {n} sequences")
        total = sum(a.size for a in ids)
        if total > self.max_tokens:
            raise ValueError(f"{type(self).__name__}.forward_batch: {total} new rows exceed max_tokens {self.max_tokens}")
        for i, (a, c, t) in enumerate(zip(ids, cached, tables)):
            if c < 0 or a.size < (1 if c else 2):
                raise ValueError(f"{type(self).__name__}.forward_batch: sequence {i} needs cached >= 0 and at least "
                                 f"{1 if c else 2} tokens, got cached={c}, {a.size} tokens")
            cap = len(t) * bs if slots is None else min(len(t), runner.max_blocks) * bs
            if c + a.size > min(cfg.max_pos, cap):
                raise ValueError(f"{type(self).__name__}.forward_batch: sequence {i}: cached + tokens = {c + a.size} exceeds max_pos "
                                 f"{cfg.max_pos} or its table's {len(t)} blocks of {bs}")
        if n > 1:
            slot_map = np.concatenate([kv_index.slot_mapping(t, bs, c, c + a.size) for a, c, t in zip(ids, cached, tables)])
            if np.unique(slot_map).size != slot_map.size:
                raise ValueError(f"{type(self).__name__}.forward_batch: two sequences' new rows map to the same cache slot")
        return ids, cached, tables, slots

    def forward_batch(self, prompts, cached=None, tables=None, slots=None, final=True):
        """n sequences' new rows (prompts: n token lists) in one prompt step (`STEP`).  cached[i] rows of sequence i
        are already in the cache under tables[i] (default 0); tables default to the runner's (rows slots[i], or 0..n-1),
        or the prefill's own table for one sequence.  Returns (last-row logits [n, vocab] on the device, first tokens
        int32 [n] on the host); with final=False (a non-final chunk group) only the KV caches are written and nothing
        is returned.
        slots (needs the runner given at construction): sequence i continues in runner row slots[i].  A given tables[i]
        becomes that row's block table; the step writes each first token and context length into the row on the
        device, and runner.steps_taken becomes the longest context of the runner.  Rows not in slots are untouched,
        so a serving loop can refill a finished row between runner.replay() calls."""
        ids, cached, tables, slots = self.check_batch_args(prompts, cached, tables, slots, final)
        if not final:
            self._step(ids, cached, tables, lm_rows=0)
            return None
        logits = self._step(ids, cached, tables, lm_rows=1, slots=slots)
        n = len(ids)
        if slots is None:
            return logits, self._out[:n].cpu()
        r = self.runner
        self._out[MAX_PREFILL_SEQS:].copy_(r.context_lens)
        host = self._out.cpu()
        r.steps_taken = int(host[MAX_PREFILL_SEQS:].max())
        return logits, host[:n].clone()

    def _step(self, ids, cached, tables, lm_rows, slots=None):
        """Build the plan, enqueue the step; returns the logits ([n, vocab] for lm_rows 1, [T, vocab] for 2) or None."""
        p, logits, _plan = self.make_plan(ids, cached, tables, lm_rows, slots)
        rc = getattr(lib(), self.STEP)(ctypes.byref(self.step_struct), ctypes.byref(p),
                                       ctypes.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream))
        if rc != 0:
            raise RuntimeError(f"{self.STEP} failed: cudaError {rc}")
        return logits

    def make_plan(self, ids, cached, tables, lm_rows, slots=None):
        """The step's `mrs_llama_prefill` for checked arguments: the plan is built on the host and sent in one pinned
        H2D copy (enqueued on the current stream).  With slots, the runner rows' block tables are written as well.
        Returns (struct, logits or None, device plan tensor the struct points into)."""
        cfg, dev, bs = self.cfg, self.dev, self.cfg.block_size
        ids = [np.asarray(p.cpu().numpy() if torch.is_tensor(p) else p, dtype=np.int32).reshape(-1) for p in ids]
        n = len(ids)
        lens = np.array([a.size for a in ids], dtype=np.int64)
        cached = np.asarray(cached, dtype=np.int64)
        T = int(lens.sum())
        cu_q = np.concatenate([[0], np.cumsum(lens)])
        cu_k = np.concatenate([[0], np.cumsum(lens + cached)])
        paged = bool(cached.any())
        slot_map = np.concatenate([kv_index.slot_mapping(t, bs, int(c), int(c + l)) for t, c, l in zip(tables, cached, lens)])
        runner = self.runner if slots is not None else None
        # one int32 plan: slot_mapping (i64) | token ids | positions | cu_q | cu_k | last rows | dest rows | block tables
        stride = max(len(t) for t in tables) if (paged or runner is not None) else 0
        if runner is not None:
            stride = runner.max_blocks
        seg = [2 * T, T, T, n + 1, n + 1, n, n, n * stride]
        off = np.concatenate([[0], np.cumsum(seg)])
        host = torch.empty(int(off[-1]), dtype=torch.int32, pin_memory=True)
        hn = host.numpy()
        hn[off[0]:off[1]] = slot_map.view(np.int32)
        hn[off[1]:off[2]] = np.concatenate(ids)
        hn[off[2]:off[3]] = np.concatenate([np.arange(c, c + l) for c, l in zip(cached, lens)])
        hn[off[3]:off[4]] = cu_q
        hn[off[4]:off[5]] = cu_k
        hn[off[5]:off[6]] = cu_q[1:] - 1
        hn[off[6]:off[7]] = slots if slots is not None else 0
        bt = hn[off[7]:off[8]].reshape(n, stride) if stride else None
        if bt is not None:
            bt[:] = 0
            for i, t in enumerate(tables):
                bt[i, :min(len(t), stride)] = t[:stride]
        plan = host.to(dev, non_blocking=True)
        ptr = lambda k: plan.data_ptr() + 4 * int(off[k])
        if runner is not None and bt is not None:   # the rows' block tables, for the decode steps that follow
            rows = plan[off[6]:off[7]].long()
            runner.block_tables.index_copy_(0, rows, plan[off[7]:off[8]].view(n, stride))
            for s, t in zip(slots, tables):
                runner.tables[s] = list(t)
        p = _Prefill()
        p.n_seqs, p.total_tokens, p.max_q_len, p.max_kv_len = n, T, int(lens.max()), int((lens + cached).max())
        p.paged, p.lm_rows, p.block_table_stride, p.num_blocks = int(paged), int(lm_rows), stride, self.num_cache_blocks
        p.slot_mapping, p.token_ids, p.positions, p.cu_seqlens_q, p.cu_seqlens_k, p.last_rows = (ptr(k) for k in range(6))
        p.block_tables = ptr(7) if paged else None
        _point(p, self.buf)
        logits = None
        if lm_rows:
            logits = torch.empty(n if lm_rows == 1 else T, cfg.vocab, dtype=self.dt, device=dev)
            p.logits, p.out_token = logits.data_ptr(), self._out.data_ptr()
        if runner is not None:
            p.dest_rows = ptr(6)
            p.runner_token_ids, p.runner_context_lens = runner.meta["token_ids"].data_ptr(), runner.context_lens.data_ptr()
        return p, logits, plan


class LlamaPrefill(PromptPrefill):
    """Prompt processing through `mrs_llama_prefill_step` (include/mrs_b200_model.h), the reference's prompt forward
    (`models/llama.rs` Block::forward with seq_len > 1) over the packed rows of one or many sequences:
    embedding -> per layer RMSNorm, wgmma dequant-GEMMs (grouped QKV, gate|up with the GLU epilogue), RoPE, var-len
    causal prompt attention over the fresh q/k/v (the reference's flash-attn call, paged_attention.rs:1413-1475) and the
    KV scatter into the paged HND cache, o_proj, add+RMSNorm, down, add+RMSNorm -> lm_head on each sequence's last row
    (`extract_logits`) -> argmax.  A sequence with cached rows (prefix-cache hit, or a later chunk of a chunked prompt)
    has its new K/V scattered first and attends over the cache (`prefill_attention_paged`).
    `forward` is the one-sequence call; TTFT of BASELINE config 3 is its time on a 4096-token prompt.  `forward_batch`
    runs up to 256 sequences in one step and can hand them to a decode runner's rows on the device."""
    STEP = "mrs_llama_prefill_step"

    def __init__(self, weights: "LlamaWeights", max_tokens=4096, runner: "LlamaRunner" = None, pdl=True):
        """max_tokens: new rows per call (all sequences together); the scratch for them is allocated here.
        runner: write prompts' K/V into this decode runner's paged cache (sequence 0's block table by default), so a
        generation is prefill -> `runner.reset(T)` -> decode-graph replays, or `forward_batch(slots=...)` ->
        decode-graph replays."""
        from . import ops, paged_attn, quant  # noqa: F401  (fail early when the extension is missing)
        if weights.tp_size != 1:
            raise NotImplementedError("LlamaPrefill runs single-GPU")
        self._init_caches(weights, max_tokens, runner)
        cfg, dev, dt = self.cfg, self.dev, self.dt
        T, H = self.max_tokens, cfg.hidden
        nq, nkv = cfg.n_heads * cfg.head_dim, cfg.n_kv_heads * cfg.head_dim
        a = lambda *s: torch.empty(*s, dtype=dt, device=dev)
        self.buf = dict(x=a(T, H), x2=a(T, H), h=a(T, H), q=a(T, nq), k=a(T, nkv), v=a(T, nkv), attn_out=a(T, nq),
                        act=a(T, cfg.inter), h_last=a(MAX_PREFILL_SEQS, H),
                        gate_up=a(2, T, cfg.inter) if T > PREFILL_GROUPED_MAX_ROWS else None,
                        argmax_scratch=torch.zeros(16 * MAX_PREFILL_SEQS + 16, dtype=torch.uint8, device=dev),
                        q8_scratch=torch.empty(MMVQ_MAX_BATCH * (-(-H // 512) * 16) * 36, dtype=torch.uint8, device=dev))
        self._layers, self.step_struct = _model_step(weights, self.k_cache, self.v_cache, pdl, cfg.n_heads, cfg.n_kv_heads)


def check_drafts(drafts, batch, draft_len, vocab):
    """drafts as int32 [batch, draft_len] (a [B][k] list or a CPU tensor); ValueError on a wrong shape or an id outside
    the vocabulary."""
    t = drafts if torch.is_tensor(drafts) else torch.as_tensor(np.asarray(drafts, dtype=np.int64))
    if t.device.type != "cpu" or tuple(t.shape) != (batch, draft_len):
        raise ValueError(f"drafts must be a host [{batch}][{draft_len}] array, got {tuple(t.shape)} on {t.device}")
    if t.dtype.is_floating_point or t.dtype == torch.bool:
        raise ValueError(f"draft ids must be integers, got {t.dtype}")
    if t.numel() and (int(t.min()) < 0 or int(t.max()) >= vocab):
        raise ValueError(f"draft ids must lie in [0, {vocab})")
    return t if t.dtype == torch.int32 else t.to(torch.int32)


def check_verifier_args(runner, draft_len):
    """ValueError unless `runner` can run verify steps of `draft_len` drafts (see LlamaVerifier).  A verify step takes
    the linear route of the runner's plain step: up to 8 sequences the GEMV chain, which holds B * (k + 1) <= 8 rows;
    9..256 sequences the GEMM chain, which takes any k."""
    k = int(draft_len)
    if not 1 <= k <= 7:
        raise ValueError(f"draft_len must be 1..7, got {draft_len}")
    if runner.B <= MMVQ_MAX_BATCH and runner.B * (k + 1) > MMVQ_MAX_BATCH:
        raise ValueError(f"batch x (draft_len + 1) = {runner.B} x {k + 1} exceeds the 8 rows of one verify step")
    if runner.w.tp_size != 1 or runner._peer is not None or runner._ar_cb is not None:
        raise ValueError("speculative verification runs single-GPU (no tensor parallelism)")
    if runner.cfg.head_dim not in (64, 128):
        raise ValueError(f"verify attention supports head_dim 64 / 128, got {runner.cfg.head_dim}")
    if runner.dt not in (torch.float16, torch.bfloat16):
        raise ValueError(f"verify steps run in f16 / bf16, got {runner.dt}")
    if not runner.step_struct.fused_attention:
        raise ValueError("verify steps need the runner's fused attention path")
    if runner.max_ctx < k + 1:
        raise ValueError(f"the runner's context ({runner.max_ctx}) is shorter than one verify step ({k + 1} rows)")
    return k


class SpecVerifier:
    """Greedy speculative decoding on a decode runner's sequences (REF mistralrs-core/src/speculative/): each verify step
    feeds q = k + 1 rows per sequence — the anchor (the token the runner would process next) and k caller-proposed
    drafts — through the model's verify step in one pass over the weights, and accepts drafts on the device
    (mrs_spec_accept).  This base holds what does not depend on the model: the B*q-row metadata over the runner's tables,
    the accepted / emitted results and their pinned staging, the anchor hand-over, the advance, graph capture and
    replay.  A subclass checks its arguments first, then calls this constructor, allocates its scratch (`buf`), points
    its step struct (`step_struct`) and names its C entry (`STEP`), which forward() calls as
    STEP(step, q, context_lens, accepted, emitted, stream).

    Shares the runner's weights, KV caches, block tables, context_lens and error_flag, so verify steps and plain
    `runner.step()` calls can be mixed; owns the B*q-row metadata and scratch.  The anchor moves explicitly:
    `sync_from_runner()` takes it from runner.meta["token_ids"], `sync_to_runner()` hands the next one back.  Rows a
    step rejected stay in the cache past the context and are overwritten later (never read)."""
    STEP = None

    def __init__(self, runner, k):
        """k: the checked draft length"""
        B, q = runner.B, k + 1
        self.r, self.k, self.q, self.B, self.dev, self.vocab = runner, k, q, B, runner.dev, runner.cfg.vocab
        self.meta = runner.decode_meta(q)
        self.results = torch.zeros(B + B * q, dtype=torch.int32, device=self.dev)   # accepted [B] then emitted [B*q]
        self._results_h = torch.zeros(B + B * q, dtype=torch.int32).pin_memory()     # one D2H copy per step
        self._drafts_h = torch.zeros(B, k, dtype=torch.int32).pin_memory()
        self._h2d_done = torch.cuda.Event()
        self.graph = None

    def sync_from_runner(self):
        """anchor of every sequence <- runner.meta["token_ids"]"""
        self.meta["token_ids"].view(self.B, self.q)[:, 0].copy_(self.r.meta["token_ids"])

    def sync_to_runner(self):
        """runner.meta["token_ids"] <- the anchor the last verify step left (the token to process next)"""
        self.r.meta["token_ids"].copy_(self.meta["token_ids"].view(self.B, self.q)[:, 0])

    def set_drafts(self, drafts):
        """drafts: [B][k] ids (list or host tensor) -> rows 1..k of every sequence (one pinned H2D copy)."""
        t = check_drafts(drafts, self.B, self.k, self.vocab)
        if not t.is_pinned():
            self._h2d_done.synchronize()              # the previous copy out of the staging buffer has finished
            self._drafts_h.copy_(t)
            t = self._drafts_h
        self.meta["token_ids"].view(self.B, self.q)[:, 1:].copy_(t, non_blocking=True)
        self._h2d_done.record()

    def advance(self):
        """enqueue the advance of every sequence by q rows (the metadata of the next verify step)"""
        self.r._advance(self.meta, self.q)

    def forward(self):
        """enqueue the verify step on the advanced metadata: the layer stack over the B*q rows, then the acceptance"""
        res = self.results
        rc = getattr(lib(), self.STEP)(ctypes.byref(self.step_struct), ctypes.c_int(self.q),
                                       ctypes.c_void_p(self.r.context_lens.data_ptr()), ctypes.c_void_p(res.data_ptr()),
                                       ctypes.c_void_p(res.data_ptr() + 4 * self.B), self.r._stream())
        if rc != 0:
            raise RuntimeError(f"{self.STEP} failed: cudaError {rc}")

    def step(self):
        """one verify step on the current anchors and drafts (eager): advance by q rows, verify, accept."""
        self.advance()
        self.forward()

    def capture(self):
        """capture step() as a CUDA graph.  The warm-up step outside the capture only writes cache rows past every
        context; the lengths, the error flag and the anchors are restored."""
        r = self.r
        saved = (r.context_lens.clone(), r.error_flag.clone(), self.meta["token_ids"].clone())
        self.step()
        r.context_lens.copy_(saved[0]); r.error_flag.copy_(saved[1]); self.meta["token_ids"].copy_(saved[2])
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.step()
        self.graph = g
        return g

    def replay(self):
        self.graph.replay()

    def accepted(self):
        """[B] device int32: drafts accepted by the last step (-1: the sequence ran out of context and was frozen)"""
        return self.results[:self.B]

    def emitted(self):
        """[B, q] device int32: the tokens the last step produced (accepted + 1 per sequence), -1 beyond them"""
        return self.results[self.B:].view(self.B, self.q)

    def logits(self):
        """[B*q, vocab]: the target's logits after each fed row"""
        return self.buf["logits"]

    def fetch(self):
        """(accepted [B], emitted [B][q]) on the host after one D2H copy"""
        self._results_h.copy_(self.results, non_blocking=True)
        torch.cuda.current_stream(self.dev).synchronize()
        h = self._results_h.tolist()
        return h[:self.B], [h[self.B + b * self.q:self.B + (b + 1) * self.q] for b in range(self.B)]


class LlamaVerifier(SpecVerifier):
    """Speculative decoding on a LlamaRunner's sequences through mrs_llama_verify_step (see SpecVerifier).  Verify
    steps take the runner's linear route: the GEMV chain for 1..8 sequences (B * q <= 8), the dequant-GEMM chain for
    9..256 (B * q up to 2048 rows), so plain and verify steps share their numerics."""
    STEP = "mrs_llama_verify_step"

    def __init__(self, runner: LlamaRunner, draft_len: int):
        k = check_verifier_args(runner, draft_len)
        super().__init__(runner, k)
        r, cfg, dev, dt = runner, runner.cfg, runner.dev, runner.dt
        B, q = self.B, self.q
        R = B * q
        z = lambda *s, d=torch.int32: torch.zeros(*s, dtype=d, device=dev)
        a = lambda *s: torch.zeros(*s, dtype=dt, device=dev)
        H, D, n_heads, n_kv = cfg.hidden, cfg.head_dim, r.n_heads, r.n_kv
        nsub = -(-(n_heads // n_kv) * q // 16)
        self.buf = dict(x=a(R, H), x2=a(R, H), q=a(R, n_heads * D), k=a(R, n_kv * D), v=a(R, n_kv * D),
                        attn_out=a(R, n_heads * D), act=a(R, cfg.inter), logits=a(R, cfg.vocab),
                        tmp_v=a(r.padded_tiles, q * n_heads, D),
                        tmp_s=torch.zeros(r.padded_tiles, q * n_heads, dtype=torch.float32, device=dev),
                        out_token=z(R), attn_counters=z(B * n_kv * nsub),
                        argmax_scratch=torch.zeros(16 * R + 16, dtype=torch.uint8, device=dev),
                        h=a(R, H))                    # the GEMM route's normed activations (not the runner's [B, H])
        s = _Step.from_buffer_copy(runner.step_struct)   # weights, caches, shapes, pdl: the runner's
        _point(s, self.meta, self.buf)
        self.step_struct = s


def speculative_generate(verifier: SpecVerifier, first_tokens, n_tokens, propose):
    """Greedy speculative generation: every sequence b starts from first_tokens[b] (processed at position
    runner.context_lens[b]) and runs until it has produced n_tokens tokens.  propose(history) -> k draft ids, where
    history is the sequence's tokens so far (first token included).  Per step: one pinned H2D copy of the drafts, one
    graph replay, one D2H copy of accepted / emitted.  Returns (token streams [B][n_tokens], accepted counts per step
    [steps][B]); the runner's token_ids hold the next anchors afterwards."""
    v = verifier
    if len(first_tokens) != v.B:
        raise ValueError(f"need {v.B} first tokens, got {len(first_tokens)}")
    v.r.set_tokens(list(first_tokens))
    v.sync_from_runner()
    if v.graph is None:
        v.capture()
    hist = [[int(t)] for t in first_tokens]
    streams = [[] for _ in range(v.B)]
    steps = []
    while min(len(s) for s in streams) < n_tokens:
        v.set_drafts([[int(t) for t in propose(h)] for h in hist])
        v.replay()
        acc, em = v.fetch()
        if min(acc) < 0:
            raise RuntimeError("speculative_generate: a sequence ran past its allocated context")
        for b in range(v.B):
            toks = em[b][:acc[b] + 1]
            streams[b] += toks
            hist[b] += toks
        steps.append(acc)
    v.sync_to_runner()
    return [s[:n_tokens] for s in streams], steps
