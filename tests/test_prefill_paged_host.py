"""prefill_attention_paged and LlamaPrefill.forward(cached=...) reject bad input before anything is launched: these
run without a GPU, on CPU tensors that no kernel could take."""
import pytest
import torch

from mistralrs_b200 import model as M, paged_attn


def _args(cache_dtype=torch.bfloat16, table_dtype=torch.int32, page=16, D=128, KVH=2, table=None):
    q = torch.zeros(5, 8, D, dtype=torch.bfloat16)
    kc = torch.zeros(4, KVH, page, D, dtype=cache_dtype)
    bt = torch.zeros(1, 4, dtype=table_dtype) if table is None else table
    cu_q = torch.tensor([0, 5], dtype=torch.int32)
    cu_k = torch.tensor([0, 20], dtype=torch.int32)
    return (q, kc, kc.clone(), bt, cu_q, cu_k, 5, 20, 0.125)


@pytest.mark.parametrize("kw,match", [
    (dict(cache_dtype=torch.float8_e4m3fn), "cache dtype"),
    (dict(cache_dtype=torch.float16), "cache dtype"),
    (dict(table_dtype=torch.int64), "block_table"),
    (dict(table=torch.zeros(4, dtype=torch.int32)), "block_table"),
    (dict(table=torch.zeros(2, 4, dtype=torch.int32)), "rows for 1 sequences"),
    (dict(page=24), "page size"),
    (dict(D=96), "head_dim"),
    (dict(KVH=3), "KV heads"),
])
def test_wrapper_rejects_bad_input(kw, match):
    with pytest.raises(ValueError, match=match):
        paged_attn.prefill_attention_paged(*_args(**kw))


def test_wrapper_rejects_table_too_short():
    q, kc, vc, bt, cu_q, cu_k, mq, _, scale = _args()
    with pytest.raises(ValueError, match="capacity"):
        paged_attn.prefill_attention_paged(q, kc, vc, bt, cu_q, cu_k, mq, 4 * 16 + 1, scale)


def _prefill(max_tokens=64):
    """A LlamaPrefill with its host-side state only (no weights, no device cache): enough to reach the checks."""
    pre = M.LlamaPrefill.__new__(M.LlamaPrefill)
    pre.cfg = M.LlamaConfig.tiny_test()
    pre.w, pre.dev, pre.dt = None, torch.device("cpu"), torch.bfloat16
    pre.max_tokens = max_tokens
    pre.table = list(range(1, -(-max_tokens // pre.cfg.block_size) + 1))
    return pre


@pytest.mark.parametrize("cached,n,table", [
    (60, 5, None),                 # past the prefill's own table (64 tokens)
    (30, 3, [1, 2]),               # past a caller's table of 2 blocks
    (510, 3, list(range(40))),     # past max_pos (512)
    (-1, 3, None),
    (0, 1, [1, 2]),                # one token with nothing cached
    (10, 0, None),
])
def test_llama_prefill_rejects_out_of_range(cached, n, table):
    with pytest.raises(ValueError):
        _prefill().forward(list(range(n)), cached=cached, table=table)
