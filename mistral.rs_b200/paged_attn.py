"""Host-side mirror of `mistralrs-paged-attn`'s CUDA backend functions
(REF: mistralrs-paged-attn/src/cuda/backend/{paged_attention,flashinfer,mod}.rs): same names,
argument meaning and error behaviour; each is argument checking + one call through the C ABI
with raw device pointers and the current stream.

Cache layouts (both the reference's):
  vLLM   key_cache [NB, KVH, D/x, BS, x] (x = 16 / elt size), value_cache [NB, KVH, D, BS]
  HND    key_cache / value_cache [NB, KVH, BS, D]   (FlashInfer path)
"""
import ctypes

import torch

from . import lib

_DT_CODE = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}
_TAG = {torch.float16: "f16", torch.bfloat16: "bf16", torch.float32: "f32"}
_SUPPORTED_HEAD_SIZES = (64, 80, 96, 112, 128, 192, 256)      # backend/paged_attention.rs:251-261
PARTITION_SIZE = 512  # backend/paged_attention.rs:302
FLASHINFER_DECODE_ENV = "MISTRALRS_FLASHINFER_DECODE"


def _env_flag(name, default):
    """REF mistralrs-core/src/perf_flags.rs:9-22"""
    import os
    v = os.environ.get(name)
    if v in ("1", "true", "TRUE", "yes", "on"):
        return True
    if v in ("0", "false", "FALSE", "no", "off"):
        return False
    return default


def flashinfer_decode_enabled():
    return _env_flag(FLASHINFER_DECODE_ENV, True)


def supports_flashinfer_group_size(q_heads, kv_heads):
    """REF mistralrs-core/src/flashinfer/mod.rs:266-273 (the GQA group sizes the decode kernel is instantiated for)"""
    return kv_heads != 0 and q_heads % kv_heads == 0 and q_heads // kv_heads in (1, 2, 3, 4, 6, 8, 16)


def flashinfer_supports_layer(q_heads, kv_heads, k_head_dim, v_head_dim):
    """Which decode backend a layer gets (REF flashinfer/mod.rs:257-264 `supports_layer`): the HND / CSR path
    (`flashinfer_decode`) when this holds, the vLLM-layout `paged_attention` otherwise or when
    MISTRALRS_FLASHINFER_DECODE=0."""
    return (flashinfer_decode_enabled() and k_head_dim == v_head_dim and k_head_dim in (64, 128, 256, 512)
            and supports_flashinfer_group_size(q_heads, kv_heads))


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _cache_dtype_code(t):
    if t.dtype in _DT_CODE:
        return _DT_CODE[t.dtype]
    if t.dtype == torch.float8_e4m3fn:
        return 3
    raise ValueError(f"unsupported cache dtype {t.dtype}")


def _dense_heads(t, name):
    # backend/mod.rs:28-63 `cache_input_layout`: heads must be dense, row stride free
    if t.dim() != 3 or t.stride(2) != 1 or t.stride(1) != t.shape[2]:
        raise ValueError(f"{name} must be [tokens, heads, head_size] with dense heads")
    return t.stride(0)


def reshape_and_cache(key, value, k_scale, v_scale, key_cache, value_cache, slot_mapping):
    """Scatter new K/V rows into the vLLM-layout cache (backend/paged_attention.rs:694-735)."""
    if key.dtype != value.dtype or key_cache.dtype != value_cache.dtype:
        raise ValueError("reshape_and_cache expects matching key/value and cache dtypes")
    if slot_mapping.dtype != torch.int64:
        raise ValueError("slot_mapping must be i64")
    T, H, D = key.shape
    nb, kvh, dx, bs, x = key_cache.shape
    if (kvh, dx * x) != (H, D) or tuple(value_cache.shape) != (nb, kvh, D, bs):
        raise ValueError(f"cache shape {tuple(key_cache.shape)}/{tuple(value_cache.shape)} incompatible with key {tuple(key.shape)}")
    ks, vs = _dense_heads(key, "key"), _dense_heads(value, "value")
    lib().reshape_and_cache(_p(key), _p(value), _p(key_cache), _p(value_cache), _p(slot_mapping),
                            ctypes.c_int(T), ctypes.c_int(H), ctypes.c_int(D), ctypes.c_int(bs), ctypes.c_int(x),
                            ctypes.c_int(ks), ctypes.c_int(vs), _stream(key.device),
                            ctypes.c_uint32(_DT_CODE[key.dtype]), ctypes.c_uint32(_cache_dtype_code(key_cache)),
                            _p(k_scale), _p(v_scale))


def reshape_and_cache_flashinfer(key, value, key_cache, value_cache, slot_mapping, k_scale=1.0, v_scale=1.0):
    """Scatter into the HND cache (backend/flashinfer.rs:71-…)."""
    if slot_mapping.dtype != torch.int64:
        raise ValueError("slot_mapping must be i64")
    T, H, D = key.shape
    nb, kvh, bs, d = key_cache.shape
    if (kvh, d) != (H, D) or value_cache.shape != key_cache.shape:
        raise ValueError("reshape_and_cache_flashinfer cache shape incompatible with key")
    ks, vs = _dense_heads(key, "key"), _dense_heads(value, "value")
    lib().reshape_and_cache_flashinfer(_p(key), _p(value), _p(key_cache), _p(value_cache), _p(slot_mapping),
                                       ctypes.c_int(T), ctypes.c_int(H), ctypes.c_int(D), ctypes.c_int(bs),
                                       ctypes.c_int(ks), ctypes.c_int(vs), ctypes.c_float(k_scale),
                                       ctypes.c_float(v_scale), ctypes.c_uint32(_DT_CODE[key.dtype]),
                                       ctypes.c_uint32(_cache_dtype_code(key_cache)), _stream(key.device))


_V2_SCRATCH = {}


def paged_attention(q, k_scale, v_scale, key_cache, value_cache, block_tables, context_lens, alibi_slopes,
                    max_context_len, softmax_scale, softcapping=1.0, sinks=None):
    """Decode attention over the vLLM-layout cache (backend/paged_attention.rs:453-483).
    q [S, H, D]; block_tables [S, max_blocks] i32/u32; context_lens [S]."""
    if q.dtype not in _TAG:
        raise ValueError(f"paged_attention: unsupported dtype {q.dtype}")
    S, H, D = q.shape
    nb, kvh, dx, bs, x = key_cache.shape
    if D not in _SUPPORTED_HEAD_SIZES:
        raise ValueError(f"`head_size` must be one of {_SUPPORTED_HEAD_SIZES}, got {D}")
    if dx * x != D or tuple(value_cache.shape) != (nb, kvh, D, bs):
        raise ValueError("paged_attention: cache shape incompatible with query")
    if block_tables.shape[0] != S or context_lens.shape[0] != S:
        raise ValueError("paged_attention: block_tables/context_lens batch mismatch")
    max_blocks = block_tables.shape[1]
    out = torch.empty(S, H, D, dtype=q.dtype, device=q.device)
    eff = min(max_blocks * bs, max_context_len)
    max_parts = (eff + PARTITION_SIZE - 1) // PARTITION_SIZE
    use_v1 = (max_parts == 1 or S * H > 512) and PARTITION_SIZE % bs == 0  # paged_attention.rs:302-307
    common = (_p(key_cache), _p(value_cache), _p(alibi_slopes), ctypes.c_int(kvh), ctypes.c_float(softmax_scale),
              ctypes.c_float(softcapping), _p(block_tables), _p(context_lens), ctypes.c_int(bs),
              ctypes.c_int(eff), ctypes.c_int(S), ctypes.c_int(H), ctypes.c_int(D),  # effective_max_context_len (paged_attention.rs:299-301)
              ctypes.c_int(max_blocks), ctypes.c_int(q.stride(0)), ctypes.c_int(key_cache.stride(0)),
              ctypes.c_int(key_cache.stride(1)), _stream(q.device), ctypes.c_uint32(_cache_dtype_code(key_cache)),
              _p(k_scale), _p(v_scale), _p(sinks))
    if use_v1:
        getattr(lib(), f"paged_attention_v1_{_TAG[q.dtype]}")(_p(out), _p(q), *common)
    else:
        key = (q.device.index, S, H, max_parts, D, q.dtype)
        if key not in _V2_SCRATCH:  # per-device grow-only slot in the reference
            _V2_SCRATCH[key] = (torch.empty(S, H, max_parts, D, dtype=q.dtype, device=q.device),
                                torch.empty(S, H, max_parts, dtype=torch.float32, device=q.device),
                                torch.empty(S, H, max_parts, dtype=torch.float32, device=q.device))
        tmp_out, exp_sums, max_logits = _V2_SCRATCH[key]
        getattr(lib(), f"paged_attention_v2_{_TAG[q.dtype]}")(_p(out), _p(exp_sums), _p(max_logits), _p(tmp_out),
                                                               _p(q), *common)
    return out


def flashinfer_decode(query, key_cache, value_cache, paged_kv_indptr, paged_kv_indices, paged_kv_last_page_len,
                      request_indices, kv_tile_indices, o_indptr, kv_chunk_size, block_valid_mask, sm_scale,
                      window_left=None, logits_soft_cap=None, scratch=None, k_scale=1.0, v_scale=1.0):
    """Decode attention over the HND cache with CSR page lists and split-KV tiles
    (backend/flashinfer.rs:241-…)."""
    for name, t in (("paged_kv_indptr", paged_kv_indptr), ("paged_kv_indices", paged_kv_indices),
                    ("paged_kv_last_page_len", paged_kv_last_page_len), ("request_indices", request_indices),
                    ("kv_tile_indices", kv_tile_indices), ("o_indptr", o_indptr), ("kv_chunk_size", kv_chunk_size)):
        if t.dtype != torch.int32:
            raise ValueError(f"flashinfer_decode expects {name} to be i32")
    if block_valid_mask.dtype != torch.uint8:
        raise ValueError("flashinfer_decode expects block_valid_mask to be u8")
    B, H, D = query.shape
    nb, kvh, page, d = key_cache.shape
    if value_cache.shape != key_cache.shape or d != D:
        raise ValueError("flashinfer_decode cache shape incompatible with query")
    padded = request_indices.shape[0]
    if (paged_kv_indptr.shape[0] != B + 1 or paged_kv_last_page_len.shape[0] != B or padded < B
            or kv_tile_indices.shape[0] != padded or o_indptr.shape[0] != B + 1 or kv_chunk_size.shape[0] != 1
            or block_valid_mask.shape[0] != padded):
        raise ValueError("flashinfer_decode metadata shapes are invalid")
    split = padded > B
    tmp_v = tmp_s = None
    if split:
        if scratch is None:
            scratch = (torch.empty(padded, H, D, dtype=query.dtype, device=query.device),
                       torch.empty(padded, H, dtype=torch.float32, device=query.device))
        tmp_v, tmp_s = scratch
        if tmp_v.dtype != query.dtype or tmp_s.dtype != torch.float32 or tmp_v.shape[0] < padded:
            raise ValueError("flashinfer_decode scratch dtypes are invalid")
    out = torch.empty(B, H, D, dtype=query.dtype, device=query.device)
    rc = lib().flashinfer_decode(_p(query), _p(key_cache), _p(value_cache), _p(paged_kv_indptr), _p(paged_kv_indices),
                                 _p(paged_kv_last_page_len), _p(request_indices), _p(kv_tile_indices), _p(o_indptr),
                                 _p(kv_chunk_size), _p(block_valid_mask), _p(out), _p(tmp_v), _p(tmp_s),
                                 ctypes.c_int(B), ctypes.c_int(padded), ctypes.c_int(H), ctypes.c_int(kvh),
                                 ctypes.c_int(D), ctypes.c_int(page), ctypes.c_int(query.stride(0)),
                                 ctypes.c_int(query.stride(1)), ctypes.c_float(sm_scale),
                                 ctypes.c_int(-1 if window_left is None else int(window_left)),
                                 ctypes.c_float(0.0 if logits_soft_cap is None else float(logits_soft_cap)),
                                 ctypes.c_float(k_scale), ctypes.c_float(v_scale),
                                 ctypes.c_uint32(_DT_CODE[query.dtype]), ctypes.c_uint32(_cache_dtype_code(key_cache)),
                                 _stream(query.device))
    if rc != 0:
        raise RuntimeError(f"flashinfer_decode failed with cudaError {rc}")
    return out


def gather_kv_cache_flashinfer(key_cache, value_cache, block_table, cu_seq_lens, num_tokens, out_dtype,
                               k_scale=1.0, v_scale=1.0):
    nb, kvh, bs, D = key_cache.shape
    k_out = torch.empty(num_tokens, kvh, D, dtype=out_dtype, device=key_cache.device)
    v_out = torch.empty_like(k_out)
    lib().gather_kv_cache_flashinfer(_p(key_cache), _p(value_cache), _p(k_out), _p(v_out), _p(block_table),
                                     _p(cu_seq_lens), ctypes.c_int(num_tokens), ctypes.c_int(cu_seq_lens.shape[0] - 1),
                                     ctypes.c_int(bs), ctypes.c_int(block_table.stride(0)), ctypes.c_int(kvh),
                                     ctypes.c_int(D), ctypes.c_uint32(_DT_CODE[out_dtype]),
                                     ctypes.c_uint32(_cache_dtype_code(key_cache)), ctypes.c_float(k_scale),
                                     ctypes.c_float(v_scale), _stream(key_cache.device))
    return k_out, v_out


def gather_kv_cache(key_cache, value_cache, k_scale, v_scale, block_table, cu_seq_lens, num_tokens, out_dtype):
    nb, kvh, dx, bs, x = key_cache.shape
    D = dx * x
    k_out = torch.empty(num_tokens, kvh, D, dtype=out_dtype, device=key_cache.device)
    v_out = torch.empty_like(k_out)
    lib().gather_kv_cache(_p(key_cache), _p(value_cache), _p(k_out), _p(v_out), _p(k_scale), _p(v_scale),
                          _p(block_table), _p(cu_seq_lens), ctypes.c_int(num_tokens),
                          ctypes.c_int(cu_seq_lens.shape[0] - 1), ctypes.c_int(bs), ctypes.c_int(block_table.stride(0)),
                          ctypes.c_int(kvh), ctypes.c_int(D), ctypes.c_int(x), _stream(key_cache.device),
                          ctypes.c_uint32(_DT_CODE[out_dtype]), ctypes.c_uint32(_cache_dtype_code(key_cache)))
    return k_out, v_out


def copy_blocks(key_caches, value_caches, block_mapping):
    """Copy-on-write block copies across all layers (backend/mod.rs `copy_blocks`).
    block_mapping: list of (src, dst)."""
    if not block_mapping:
        return
    dev = key_caches[0].device
    kptr = torch.tensor([t.data_ptr() for t in key_caches], dtype=torch.int64, device=dev)
    vptr = torch.tensor([t.data_ptr() for t in value_caches], dtype=torch.int64, device=dev)
    bm = torch.tensor(block_mapping, dtype=torch.int64, device=dev).reshape(-1)
    es = key_caches[0].element_size()
    tag = {1: "u8", 2: "bf16", 4: "f32"}[es]
    getattr(lib(), f"copy_blocks_{tag}")(_p(kptr), _p(vptr), _p(bm), ctypes.c_int(len(key_caches)),
                                         ctypes.c_int(len(block_mapping)),
                                         ctypes.c_int(key_caches[0][0].numel()), ctypes.c_int(value_caches[0][0].numel()),
                                         ctypes.c_int64(torch.cuda.current_stream(dev).cuda_stream))
    return kptr, vptr, bm  # keep alive until the stream has consumed them


def swap_blocks(src: torch.Tensor, dst: torch.Tensor, block_mapping):
    """`swap_blocks` (backend/cache.rs:194): copy cache blocks src[s] -> dst[d] for every (s, d) in
    `block_mapping` (dict or list of pairs).  Either side may be a CUDA tensor or a (pinned) host
    tensor — swap-out / swap-in; both on CUDA must be the same device, as in the reference."""
    pairs = list(block_mapping.items()) if isinstance(block_mapping, dict) else list(block_mapping)
    if not pairs:
        return
    if src.dtype != dst.dtype or src.shape[1:] != dst.shape[1:]:
        raise ValueError("swap_blocks: src and dst must share dtype and block geometry")
    if src.is_cuda and dst.is_cuda and src.device != dst.device:
        raise ValueError(f"Tensors must be on the same device to copy, got {src.device} (src) and {dst.device} (dst).")
    if not (src.is_cuda or dst.is_cuda):
        raise ValueError("swap_blocks: at least one side must be a CUDA tensor")
    if not (src.is_contiguous() and dst.is_contiguous()):
        raise ValueError("swap_blocks: caches must be contiguous")
    dev = src.device if src.is_cuda else dst.device
    block_bytes = src[0].numel() * src.element_size()
    flat = (ctypes.c_int64 * (2 * len(pairs)))(*[int(x) for p in pairs for x in p])
    if max(p[0] for p in pairs) >= src.shape[0] or max(p[1] for p in pairs) >= dst.shape[0] or min(min(p) for p in pairs) < 0:
        raise IndexError("swap_blocks: block number out of range")
    rc = lib().mrs_swap_blocks(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), ctypes.c_int64(block_bytes),
                               flat, ctypes.c_int64(len(pairs)), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    if rc != 0:
        raise RuntimeError(f"mrs_swap_blocks failed with cudaError {rc}")


def kv_scale_update(key: torch.Tensor, value: torch.Tensor, k_scales: torch.Tensor, v_scales: torch.Tensor):
    """`kv_scale_update` (backend/scale_update.rs:114): k_scales[0] = max(k_scales[0], absmax(key)/240),
    same for value; one f32 scalar each, updated in place on the device."""
    if key.dtype != value.dtype or key.numel() != value.numel():
        raise ValueError("kv_scale_update: key and value must share dtype and element count")
    if k_scales.dtype != torch.float32 or v_scales.dtype != torch.float32:
        raise ValueError("kv_scale_update: scales must be f32")
    tag = {torch.float32: "f32", torch.float16: "f16", torch.bfloat16: "bf16"}.get(key.dtype)
    if tag is None:
        raise ValueError("Invalid dtype for kv scale update!")
    key, value = key.contiguous(), value.contiguous()
    getattr(lib(), f"update_kv_scales_{tag}")(_p(key), _p(value), ctypes.c_long(key.numel()), _p(k_scales), _p(v_scales),
                                              ctypes.c_int64(torch.cuda.current_stream(key.device).cuda_stream))


def prefill_attention(q, k, v, softmax_scale, causal=True, cu_seqlens=None, max_seqlen=None, window_left=None,
                      softcap=None):
    """Prompt attention over fresh q/k/v (the reference's flash-attn call on a fresh prompt,
    paged_attention.rs:1413-1475; `flash_attn_varlen` signature when cu_seqlens is given).
    q [T, H, D], k/v [T, KVH, D] (last dim contiguous, heads dense), f16/bf16 -> out [T, H, D]."""
    if q.dtype not in _TAG:
        raise ValueError(f"prefill_attention: unsupported dtype {q.dtype}")
    T, H, D = q.shape
    KVH = k.shape[1]
    if D not in (64, 128):
        raise ValueError("prefill_attention: head_dim must be 64 or 128")
    if k.shape != v.shape or k.shape[0] != T or k.shape[2] != D or H % KVH:
        raise ValueError("prefill_attention: q/k/v shapes do not agree")
    for t, name in ((q, "q"), (k, "k"), (v, "v")):
        if t.stride(2) != 1 or t.stride(1) != D:
            raise ValueError(f"prefill_attention: {name} must have dense heads")
    out = torch.empty(T, H, D, dtype=q.dtype, device=q.device)
    batch = 0 if cu_seqlens is None else cu_seqlens.numel() - 1
    rc = lib().mrs_prefill_attention(_p(q), _p(k), _p(v), _p(out), _p(cu_seqlens), ctypes.c_int(batch), ctypes.c_int(T),
                                     ctypes.c_int(max_seqlen or T), ctypes.c_int(H), ctypes.c_int(KVH), ctypes.c_int(D),
                                     ctypes.c_int64(q.stride(0)), ctypes.c_int64(k.stride(0)), ctypes.c_int64(out.stride(0)),
                                     ctypes.c_float(softmax_scale), ctypes.c_int(int(causal)),
                                     ctypes.c_int(-1 if window_left is None else window_left),
                                     ctypes.c_float(0.0 if softcap is None else softcap),
                                     ctypes.c_uint32({torch.float16: 0, torch.bfloat16: 1}[q.dtype]), _stream(q.device))
    if rc != 0:
        raise RuntimeError(f"mrs_prefill_attention failed with cudaError {rc}")
    return out


PREFILL_PAGE_SIZES = (8, 16, 32)   # the reference's allowed block sizes


def prefill_attention_paged(q, key_cache, value_cache, block_table, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                            softmax_scale, causal=True, window_left=None, softcap=None):
    """Prompt attention of new query tokens over K/V already in the HND page cache (the reference's
    `flash_attn_varlen_paged_windowed`, paged_attention.rs:1357-1411): prefix-cache hits and chunked prompts.
    q [total_q, H, D] (heads dense); key_cache / value_cache [num_blocks, KVH, page, D] in q's dtype, holding the new
    tokens' K/V already; block_table [batch, max_pages] i32; cu_seqlens_q / cu_seqlens_k [batch + 1] i32, cumulative.
    Query i of sequence b sits at position kv_len_b - q_len_b + i (causal mask aligned bottom-right) -> out [total_q, H, D]."""
    if q.dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"prefill_attention_paged: unsupported dtype {q.dtype}")
    if key_cache.dtype != q.dtype or value_cache.dtype != q.dtype:
        raise ValueError(f"prefill_attention_paged: cache dtype {key_cache.dtype}/{value_cache.dtype} must equal q's {q.dtype}")
    if q.dim() != 3 or q.stride(2) != 1 or q.stride(1) != q.shape[2]:
        raise ValueError("prefill_attention_paged: q must be [tokens, heads, head_dim] with dense heads")
    T, H, D = q.shape
    if key_cache.dim() != 4 or value_cache.shape != key_cache.shape or not (key_cache.is_contiguous() and value_cache.is_contiguous()):
        raise ValueError("prefill_attention_paged: caches must be contiguous [num_blocks, kv_heads, page, head_dim] of one shape")
    nb, KVH, page, d = key_cache.shape
    if D not in (64, 128) or d != D:
        raise ValueError(f"prefill_attention_paged: head_dim must be 64 or 128 and match the cache, got {D} / {d}")
    if page not in PREFILL_PAGE_SIZES:
        raise ValueError(f"prefill_attention_paged: page size must be one of {PREFILL_PAGE_SIZES}, got {page}")
    if KVH == 0 or H % KVH:
        raise ValueError(f"prefill_attention_paged: {H} query heads do not divide into {KVH} KV heads")
    if block_table.dtype != torch.int32 or block_table.dim() != 2 or block_table.stride(1) != 1:
        raise ValueError("prefill_attention_paged: block_table must be a 2-D i32 tensor with contiguous rows")
    batch = cu_seqlens_q.numel() - 1
    for name, t in (("cu_seqlens_q", cu_seqlens_q), ("cu_seqlens_k", cu_seqlens_k)):
        if t.dtype != torch.int32 or t.dim() != 1 or t.numel() != batch + 1 or not t.is_contiguous():
            raise ValueError(f"prefill_attention_paged: {name} must be a contiguous i32 vector of batch + 1 entries")
    if block_table.shape[0] != batch:
        raise ValueError(f"prefill_attention_paged: block_table has {block_table.shape[0]} rows for {batch} sequences")
    if max_seqlen_k > block_table.shape[1] * page:
        raise ValueError("prefill_attention_paged: max_seqlen_k exceeds the block table's capacity")
    out = torch.empty(T, H, D, dtype=q.dtype, device=q.device)
    rc = lib().mrs_prefill_attention_paged(_p(q), _p(key_cache), _p(value_cache), _p(out), _p(block_table),
                                           ctypes.c_int(block_table.stride(0)), _p(cu_seqlens_q), _p(cu_seqlens_k),
                                           ctypes.c_int(batch), ctypes.c_int(T), ctypes.c_int(int(max_seqlen_q)),
                                           ctypes.c_int(int(max_seqlen_k)), ctypes.c_int(nb), ctypes.c_int(H), ctypes.c_int(KVH),
                                           ctypes.c_int(D), ctypes.c_int(page), ctypes.c_int64(q.stride(0)),
                                           ctypes.c_int64(out.stride(0)), ctypes.c_float(softmax_scale), ctypes.c_int(int(causal)),
                                           ctypes.c_int(-1 if window_left is None else int(window_left)),
                                           ctypes.c_float(0.0 if softcap is None else float(softcap)),
                                           ctypes.c_uint32(_DT_CODE[q.dtype]), _stream(q.device))
    if rc != 0:
        raise RuntimeError(f"mrs_prefill_attention_paged failed with cudaError {rc}")
    return out
