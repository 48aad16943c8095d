"""Argument checks of GptqRunner and mrs_gptq_decode_step (no GPU): a batch the decode step cannot take is rejected
before anything is allocated, and a step struct it cannot run before any launch."""
import ctypes
import types

import pytest

from mistralrs_b200 import gptq_model as G
from mistralrs_b200 import lib


def test_gptq_runner_rejects_bad_batch():
    # the stub weights have no device state at all: reaching an allocation would fail differently
    w = types.SimpleNamespace(cfg=G.GptqConfig.tiny_test())
    for batch in (0, 257, -1, 2.0, True, "4", None):
        with pytest.raises(ValueError, match="batch must be"):
            G.GptqRunner(w, batch=batch)


def test_gptq_decode_step_rejects_bad_arguments():
    """mrs_gptq_decode_step returns cudaErrorInvalidValue before any launch; every case differs from a well-formed
    two-layer batch-16 step in one field (the device pointers are never dereferenced)"""
    bufs = (ctypes.c_int32 * 64)()
    p = lambda i: ctypes.addressof(bufs) + 4 * i
    layers = (G._Layer * 2)()
    act_order = (G._Layer * 2)()
    act_order[1].perm_o = p(16)                   # an act-order o_proj without the attn_perm scratch

    def call(**fields):
        s = G._Step()
        s.batch, s.n_layers, s.head_dim, s.cache_layout, s.act_dtype, s.hidden = 16, 2, 128, 1, 1, 4096
        s.layers = ctypes.cast(layers, ctypes.POINTER(G._Layer))
        s.token_ids, s.out_token = p(0), p(8)
        for n, v in fields.items():
            setattr(s, n, v)
        return lib().mrs_gptq_decode_step(ctypes.byref(s), None)

    bad = [dict(layers=None), dict(n_layers=0), dict(batch=0), dict(batch=257), dict(act_dtype=2), dict(hidden=4092),
           dict(cache_layout=2), dict(layers=ctypes.cast(act_order, ctypes.POINTER(G._Layer)))]
    for kw in bad:
        assert call(**kw) == 1, kw
