"""Argument checks of GptqRunner (no GPU): a batch the decode step cannot take is rejected before anything is
allocated."""
import types

import pytest

from mistralrs_b200 import gptq_model as G


def test_gptq_runner_rejects_bad_batch():
    # the stub weights have no device state at all: reaching an allocation would fail differently
    w = types.SimpleNamespace(cfg=G.GptqConfig.tiny_test())
    for batch in (0, 257, -1, 2.0, True, "4", None):
        with pytest.raises(ValueError, match="batch must be"):
            G.GptqRunner(w, batch=batch)
