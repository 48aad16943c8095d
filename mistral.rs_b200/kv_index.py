"""ctypes front-end of the C++ host layer (host/kv_index.hpp): BlockPool, slot mapping, the
FlashInfer CSR page table and the split-KV decode tile plan — the integer metadata the
reference's scheduler side produces (REF: block_pool.rs, inputs_processor.rs:896-923,
flashinfer/metadata.rs).  Pure host code; no GPU needed."""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
HOST_LIB_PATH = os.path.join(_HERE, "libmrs_b200_host.so")
_lib = None
PAD_SLOT_ID = -1


def host_lib():
    global _lib
    if _lib is None:
        if not os.path.exists(HOST_LIB_PATH):
            raise RuntimeError(f"{HOST_LIB_PATH} missing: run __graft_entry__.build()")
        L = ctypes.CDLL(HOST_LIB_PATH)
        L.mrs_block_pool_new.restype = ctypes.c_void_p
        L.mrs_block_pool_new_cached.restype = ctypes.c_void_p
        L.mrs_block_pool_usage.restype = ctypes.c_double
        for f in ("null_block_id", "num_free_blocks", "ref_cnt", "num_cached_blocks", "num_block_hashes", "computed_blocks"):
            getattr(L, f"mrs_block_pool_{f}").restype = ctypes.c_int64
        L.mrs_block_hashes.restype = ctypes.c_int64
        L.mrs_sample_topk_packed_batch.restype = ctypes.c_int64
        L.mrs_ggml_quantize.restype = ctypes.c_int64
        L.mrs_kv_manager_new.restype = ctypes.c_void_p
        L.mrs_kv_manager_pool.restype = ctypes.c_void_p
        L.mrs_kv_manager_usage.restype = ctypes.c_double
        for f in ("num_free_blocks", "num_usable_blocks", "get_computed_blocks", "allocate_slots", "num_blocks", "num_cached_blocks",
                  "decode_step"):
            getattr(L, f"mrs_kv_manager_{f}").restype = ctypes.c_int64
        L.mrs_decode_split_pages.restype = ctypes.c_int64
        L.mrs_make_decode_tiles.restype = ctypes.c_int64
        for f in ("prompt_chunk_size", "build_prompt_chunk_plan", "next_prompt_chunk_group"):
            getattr(L, f"mrs_{f}").restype = ctypes.c_int64
        _lib = L
    return _lib


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)


def compute_block_hashes(tokens, block_size, extra_keys=(), prev=()):
    """Chained hashes of the full blocks of `tokens` (REF block_hash.rs:232-263; with `prev`, only the blocks
    after those already hashed are computed, :270-300)."""
    t, e, pv = _u32(tokens), _u64(list(extra_keys)), _u64(list(prev))
    out = np.empty(max(t.size // block_size, 1), dtype=np.uint64)
    n = host_lib().mrs_block_hashes(ctypes.c_void_p(t.ctypes.data), ctypes.c_int64(t.size), ctypes.c_int64(block_size),
                                    ctypes.c_void_p(e.ctypes.data), ctypes.c_int64(e.size),
                                    ctypes.c_void_p(pv.ctypes.data), ctypes.c_int64(pv.size), ctypes.c_void_p(out.ctypes.data))
    if n < 0:
        raise ValueError("block_size must be positive")
    return [int(v) for v in out[:n]]


def hash_block_tokens(parent, tokens, extra_keys=()):
    """One link of the chain: hash of a block given the previous block's hash (None for the first)."""
    t = _u32(tokens)
    if parent is None:
        return compute_block_hashes(t, t.size, extra_keys)[0]
    both = np.concatenate([t, t])                        # block 1 of a two-block run whose block 0 hash is `parent`
    return compute_block_hashes(both, t.size, extra_keys, prev=[parent])[1]


class BlockPool:
    def __init__(self, num_gpu_blocks, enable_caching=False, hash_block_size=16):
        self._h = ctypes.c_void_p(host_lib().mrs_block_pool_new_cached(ctypes.c_int64(num_gpu_blocks), ctypes.c_int32(int(enable_caching)),
                                                                       ctypes.c_int64(hash_block_size)))
        if not self._h:
            raise ValueError("Must have at least 1 GPU block")
        self.enable_caching, self.hash_block_size = bool(enable_caching), hash_block_size

    def usage(self):
        return host_lib().mrs_block_pool_usage(self._h)

    def num_cached_blocks(self):
        return host_lib().mrs_block_pool_num_cached_blocks(self._h)

    def num_block_hashes(self, block_id):
        return host_lib().mrs_block_pool_num_block_hashes(self._h, ctypes.c_int64(block_id))

    def get_cached_block(self, block_hash, group_ids):
        g = _u32(group_ids)
        out = np.empty(max(g.size, 1), dtype=np.int64)
        ok = host_lib().mrs_block_pool_get_cached_block(self._h, ctypes.c_uint64(block_hash), ctypes.c_void_p(g.ctypes.data),
                                                       ctypes.c_int64(g.size), ctypes.c_void_p(out.ctypes.data))
        return [int(v) for v in out[:g.size]] if ok else None

    def cache_full_blocks(self, block_ids, block_hashes, num_cached_blocks, num_full_blocks, kv_cache_group_id=0):
        a, h = _i64(block_ids), _u64(block_hashes)
        rc = host_lib().mrs_block_pool_cache_full_blocks(self._h, ctypes.c_void_p(a.ctypes.data), ctypes.c_int64(a.size),
                                                         ctypes.c_void_p(h.ctypes.data), ctypes.c_int64(h.size),
                                                         ctypes.c_int64(num_cached_blocks), ctypes.c_int64(num_full_blocks),
                                                         ctypes.c_uint32(kv_cache_group_id))
        if rc != 0:
            raise ValueError(f"Not enough block hashes ({h.size}) for {num_full_blocks} full blocks")

    def reset_prefix_cache(self):
        return bool(host_lib().mrs_block_pool_reset_prefix_cache(self._h))

    def computed_blocks(self, block_hashes, num_tokens, block_size, group_ids=(0,)):
        """Longest cached prefix of a request as block ids (REF kv_cache_manager.rs:129-174): the caller touches them
        and starts prefill at len(result) * block_size."""
        h, g = _u64(block_hashes), _u32(group_ids)
        out = np.empty(max(h.size, 1), dtype=np.int64)
        n = host_lib().mrs_block_pool_computed_blocks(self._h, ctypes.c_void_p(h.ctypes.data), ctypes.c_int64(h.size),
                                                      ctypes.c_int64(num_tokens), ctypes.c_int64(block_size),
                                                      ctypes.c_void_p(g.ctypes.data), ctypes.c_int64(g.size), ctypes.c_void_p(out.ctypes.data))
        return [int(v) for v in out[:n]]

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            try:
                _lib.mrs_block_pool_free(self._h)
            except Exception:
                pass
            self._h = None

    def null_block_id(self):
        return host_lib().mrs_block_pool_null_block_id(self._h)

    def num_free_blocks(self):
        return host_lib().mrs_block_pool_num_free_blocks(self._h)

    def block_ref_cnt(self, block_id):
        return host_lib().mrs_block_pool_ref_cnt(self._h, ctypes.c_int64(block_id))

    def get_new_blocks(self, num):
        out = np.empty(max(num, 1), dtype=np.int64)
        ok = host_lib().mrs_block_pool_get_new_blocks(self._h, ctypes.c_int64(num), ctypes.c_void_p(out.ctypes.data))
        return [int(v) for v in out[:num]] if ok else None

    def free_blocks(self, ordered_block_ids):
        a = _i64(ordered_block_ids)
        host_lib().mrs_block_pool_free_blocks(self._h, ctypes.c_void_p(a.ctypes.data), ctypes.c_int64(a.size))

    def touch(self, block_ids):
        a = _i64(block_ids)
        host_lib().mrs_block_pool_touch(self._h, ctypes.c_void_p(a.ctypes.data), ctypes.c_int64(a.size))


class ComputedBlocks:
    def __init__(self, block_ids, num_computed_tokens):
        self.block_ids, self.num_computed_tokens = block_ids, num_computed_tokens


class KVCacheManager:
    """Per-request block tables over a BlockPool (C++ host/kv_cache_manager.hpp; REF kv_cache_manager.rs:62-435):
    same method names and results as the reference's manager."""

    def __init__(self, num_gpu_blocks, block_size, enable_caching, kv_cache_group_ids=(0,)):
        g = _u32(list(kv_cache_group_ids))
        self._h = ctypes.c_void_p(host_lib().mrs_kv_manager_new(ctypes.c_int64(num_gpu_blocks), ctypes.c_int64(block_size),
                                                                ctypes.c_int32(int(enable_caching)), ctypes.c_void_p(g.ctypes.data),
                                                                ctypes.c_int64(g.size)))
        if not self._h:
            raise ValueError("Must have at least 1 GPU block and a positive block size")
        self.block_size, self.enable_caching = block_size, bool(enable_caching)

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            try:
                _lib.mrs_kv_manager_free(self._h)
            except Exception:
                pass
            self._h = None

    def _rid(self, request_id):
        return ctypes.c_uint64(request_id)

    def num_free_blocks(self):
        return host_lib().mrs_kv_manager_num_free_blocks(self._h)

    def num_usable_blocks(self):
        return host_lib().mrs_kv_manager_num_usable_blocks(self._h)

    def usage(self):
        return host_lib().mrs_kv_manager_usage(self._h)

    def caching_enabled(self):
        return self.enable_caching

    def get_computed_blocks(self, block_hashes, num_tokens):
        h = _u64(block_hashes)
        out = np.empty(max(h.size, 1), dtype=np.int64)
        n = host_lib().mrs_kv_manager_get_computed_blocks(self._h, ctypes.c_void_p(h.ctypes.data), ctypes.c_int64(h.size),
                                                          ctypes.c_int64(num_tokens), ctypes.c_void_p(out.ctypes.data))
        return ComputedBlocks([int(v) for v in out[:n]], n * self.block_size)

    def allocate_slots(self, request_id, num_tokens, computed_blocks=()):
        c = _i64(list(computed_blocks))
        out = np.empty(-(-num_tokens // self.block_size) + 1, dtype=np.int64)
        n = host_lib().mrs_kv_manager_allocate_slots(self._h, self._rid(request_id), ctypes.c_int64(num_tokens),
                                                     ctypes.c_void_p(c.ctypes.data), ctypes.c_int64(c.size), ctypes.c_void_p(out.ctypes.data))
        return None if n < 0 else [int(v) for v in out[:n]]

    def free(self, request_id):
        host_lib().mrs_kv_manager_release(self._h, self._rid(request_id))

    def trim_request_to_num_tokens(self, request_id, num_tokens):
        host_lib().mrs_kv_manager_trim(self._h, self._rid(request_id), ctypes.c_int64(num_tokens))

    def cache_blocks(self, request_id, block_hashes, num_computed_tokens):
        h = _u64(block_hashes)
        if host_lib().mrs_kv_manager_cache_blocks(self._h, self._rid(request_id), ctypes.c_void_p(h.ctypes.data), ctypes.c_int64(h.size),
                                                  ctypes.c_int64(num_computed_tokens)) != 0:
            raise ValueError("Not enough block hashes for the full blocks")

    def has_request(self, request_id):
        return bool(host_lib().mrs_kv_manager_has_request(self._h, self._rid(request_id)))

    def num_blocks_for_request(self, request_id):
        return host_lib().mrs_kv_manager_num_blocks(self._h, self._rid(request_id))

    def num_cached_blocks(self, request_id):
        return host_lib().mrs_kv_manager_num_cached_blocks(self._h, self._rid(request_id))

    def reset_prefix_cache(self):
        return bool(host_lib().mrs_kv_manager_reset_prefix_cache(self._h))

    def get_block_ids(self, request_id):
        n = self.num_blocks_for_request(request_id)
        if not self.has_request(request_id):
            return None
        t = self.get_block_table(request_id, n)
        return [int(v) for v in t]

    def get_slot_mapping(self, request_id, start_token, num_tokens):
        out = np.empty(max(num_tokens, 1), dtype=np.int64)
        rc = host_lib().mrs_kv_manager_slot_mapping(self._h, self._rid(request_id), ctypes.c_int64(start_token), ctypes.c_int64(num_tokens),
                                                    ctypes.c_void_p(out.ctypes.data))
        return None if rc != 0 else out[:num_tokens]

    def get_block_table(self, request_id, max_blocks):
        out = np.empty(max(max_blocks, 1), dtype=np.int32)
        rc = host_lib().mrs_kv_manager_block_table(self._h, self._rid(request_id), ctypes.c_int64(max_blocks), ctypes.c_void_p(out.ctypes.data))
        return None if rc != 0 else out[:max_blocks]

    def decode_step(self, request_ids, context_lens, max_blocks, tables=None, slots=None):
        """Grow every request to context_lens[b] tokens and write its table row + last-token slot into `tables`
        ([batch, max_blocks] int32) / `slots` ([batch] int64) — numpy arrays, e.g. views of pinned staging tensors."""
        r, c = _u64(list(request_ids)), _i64(list(context_lens))
        if tables is None:
            tables = np.zeros((r.size, max_blocks), dtype=np.int32)
        if slots is None:
            slots = np.zeros(r.size, dtype=np.int64)
        assert tables.dtype == np.int32 and tables.flags.c_contiguous and tables.shape == (r.size, max_blocks)
        assert slots.dtype == np.int64 and slots.flags.c_contiguous and slots.shape == (r.size,)
        bad = host_lib().mrs_kv_manager_decode_step(self._h, ctypes.c_void_p(r.ctypes.data), ctypes.c_void_p(c.ctypes.data),
                                                    ctypes.c_int64(r.size), ctypes.c_int64(max_blocks),
                                                    ctypes.c_void_p(tables.ctypes.data), ctypes.c_void_p(slots.ctypes.data))
        if bad >= 0:
            raise MemoryError(f"request {int(r[bad])} (batch index {bad}) is unknown or the pool cannot grow it")
        return tables, slots


def slot_mapping(table, block_size, start, end):
    t = _i64(table)
    out = np.empty(max(end - start, 0), dtype=np.int64)
    rc = host_lib().mrs_slot_mapping(ctypes.c_void_p(t.ctypes.data), ctypes.c_int64(t.size), ctypes.c_int64(block_size),
                                     ctypes.c_int64(start), ctypes.c_int64(end), ctypes.c_void_p(out.ctypes.data))
    if rc != 0:
        raise IndexError("Block table is too small (prompt)!")
    return out


def make_paged_kv_tensors(tables, context_lens, block_size, padded_indices_len):
    batch = len(tables)
    max_blocks = max((len(t) for t in tables), default=0)
    dense = np.zeros((batch, max(max_blocks, 1)), dtype=np.int64)
    for b, t in enumerate(tables):
        dense[b, :len(t)] = t
    cl = _i64(context_lens)
    for b, t in enumerate(tables):
        if -(-int(cl[b]) // block_size) > len(t):
            raise IndexError("paged kv block table is too small")
    indptr = np.empty(batch + 1, dtype=np.int32)
    indices = np.empty(max(padded_indices_len, 1), dtype=np.int32)
    last = np.empty(max(batch, 1), dtype=np.int32)
    rc = host_lib().mrs_make_paged_kv(ctypes.c_void_p(dense.ctypes.data), ctypes.c_int64(batch),
                                      ctypes.c_int64(dense.shape[1]), ctypes.c_void_p(cl.ctypes.data),
                                      ctypes.c_int64(block_size), ctypes.c_int64(padded_indices_len),
                                      ctypes.c_void_p(indptr.ctypes.data), ctypes.c_void_p(indices.ctypes.data),
                                      ctypes.c_void_p(last.ctypes.data))
    if rc != 0:
        raise IndexError("paged kv indices exceed padded length")
    return indptr, indices[:padded_indices_len], last[:batch]


def decode_split_pages(block_size, batch_size, num_kv_heads, max_context_len, sm_count=132):
    return int(host_lib().mrs_decode_split_pages(ctypes.c_int64(block_size), ctypes.c_int64(batch_size),
                                                 ctypes.c_int64(num_kv_heads), ctypes.c_int64(sm_count),
                                                 ctypes.c_int64(max_context_len)))


def make_paged_kv_decode_tensors(tables, context_lens, block_size, split_pages, padded_tiles_len):
    """split_pages None -> no split.  Returns (request_indices, kv_tile_indices, o_indptr,
    kv_chunk_size, block_valid_mask) exactly like metadata.rs:152-216."""
    batch = len(tables)
    tl = _i64([len(t) for t in tables])
    cl = _i64(context_lens)
    req = np.empty(max(padded_tiles_len, 1), dtype=np.int32)
    tile = np.empty(max(padded_tiles_len, 1), dtype=np.int32)
    o_indptr = np.empty(batch + 1, dtype=np.int32)
    chunk = np.empty(1, dtype=np.int32)
    mask = np.empty(max(padded_tiles_len, 1), dtype=np.uint8)
    n = host_lib().mrs_make_decode_tiles(ctypes.c_void_p(tl.ctypes.data), ctypes.c_void_p(cl.ctypes.data),
                                         ctypes.c_int64(batch), ctypes.c_int64(block_size),
                                         ctypes.c_int64(split_pages or 0), ctypes.c_int64(padded_tiles_len),
                                         ctypes.c_void_p(req.ctypes.data), ctypes.c_void_p(tile.ctypes.data),
                                         ctypes.c_void_p(o_indptr.ctypes.data), ctypes.c_void_p(chunk.ctypes.data),
                                         ctypes.c_void_p(mask.ctypes.data))
    if n < 0:
        raise IndexError("paged kv decode tiles exceed padded length / table too small")
    return req[:padded_tiles_len], tile[:padded_tiles_len], o_indptr, chunk, mask[:padded_tiles_len]


# ---- prompt chunk plan (host/prompt_chunks.hpp; REF pipeline/prompt_chunks.rs for text prompts) ----
def prompt_chunk_size(batch, budget):
    """Each of `batch` scheduled prompts' share of a step's token budget: max(1, budget // batch)."""
    r = host_lib().mrs_prompt_chunk_size(ctypes.c_int64(int(batch)), ctypes.c_int64(int(budget)))
    if r < 0:
        raise ValueError(f"prompt_chunk_size: need batch, budget >= 0, got {batch}, {budget}")
    return int(r)


def build_prompt_chunk_plan(total_len, prefix_len, chunk_size, block_align=None):
    """[(start, end)] chunks of rows [prefix_len, total_len), each at most chunk_size; with block_align a chunk that
    would end inside a block ends at that block's start when it stays non-empty."""
    args = [int(total_len), int(prefix_len), int(chunk_size), int(block_align or 0)]
    f = host_lib().mrs_build_prompt_chunk_plan
    n = f(*[ctypes.c_int64(a) for a in args], None, ctypes.c_int64(0))
    if n < 0:
        raise ValueError(f"build_prompt_chunk_plan: bad arguments {args}")
    out = np.empty(max(1, 2 * n), dtype=np.int64)
    f(*[ctypes.c_int64(a) for a in args], ctypes.c_void_p(out.ctypes.data), ctypes.c_int64(n))
    return [(int(out[2 * i]), int(out[2 * i + 1])) for i in range(n)]


def next_prompt_chunk_group(plan_indices, plans, require_uniform_query_len=False):
    """(members, is_final) of the next prompt step, or None when no sequence has a chunk left.  plan_indices[i] is the
    index of sequence i's next chunk in plans[i] (a list of (start, end)).  The first sequence with a chunk left sets
    finality and query length; members are the sequences whose next chunk has the same finality (and, with
    require_uniform_query_len, the same length)."""
    n = len(plans)
    if len(plan_indices) != n:
        raise ValueError(f"next_prompt_chunk_group: {len(plan_indices)} indices for {n} plans")
    idx = _i64([int(i) for i in plan_indices] or [0])
    offs = _i64(np.cumsum([0] + [len(p) for p in plans]))
    flat = _i64([v for p in plans for c in p for v in c] or [0])
    members = np.empty(max(1, n), dtype=np.int64)
    fin = ctypes.c_int32(0)
    r = host_lib().mrs_next_prompt_chunk_group(ctypes.c_void_p(idx.ctypes.data), ctypes.c_void_p(offs.ctypes.data),
                                               ctypes.c_void_p(flat.ctypes.data), ctypes.c_int64(n),
                                               ctypes.c_int32(int(bool(require_uniform_query_len))),
                                               ctypes.c_void_p(members.ctypes.data), ctypes.byref(fin))
    if r < 0:
        raise ValueError("next_prompt_chunk_group: bad arguments")
    if r == 0:
        return None
    return [int(m) for m in members[:r]], bool(fin.value)
