"""bench.py on the GPU, on truncated models: the default (config 2) line prints one JSON result line with and without
--dump-outputs, and two runs with the same arguments dump the same arrays; configs 3 and 4 time exactly --steps
steps and dump their outputs too."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench(*extra, layers="2"):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "2", "--warmup", "1", "--layers", layers,
                        "--no-extras", "--no-cpu-baseline", "--no-validate", *extra], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout[-2000:]
    line = json.loads(lines[0])
    assert line["steps"] == 2 and line["value"] > 0
    return line


def test_bench_line_and_dumped_outputs(cuda, tmp_path):
    _bench()
    dirs = [tmp_path / "a", tmp_path / "b"]
    for d in dirs:
        _bench("--dump-outputs", str(d))
    names = sorted(os.listdir(dirs[0]))
    assert names == ["last_logits.npy", "prompt_logits.npy", "token_ids.npy"]
    assert sum(os.path.getsize(dirs[0] / n) for n in names) <= 64 << 20
    for n in names:
        a, b = np.load(dirs[0] / n), np.load(dirs[1] / n)
        assert a.dtype in (np.float32, np.float64) and np.isfinite(a).all()
        assert np.array_equal(a, b), n


@pytest.mark.parametrize("config,block,names", [("3", "prefill", ["first_token.npy", "prefill_logits.npy"]),
                                                ("4", "config4", ["last_logits.npy", "token_ids.npy"])])
def test_bench_configs_3_4_steps_and_dump(cuda, tmp_path, config, block, names):
    line = _bench("--config", config, "--dump-outputs", str(tmp_path), layers="1")
    assert line[block]["steps"] == 2 and line[block]["warmup"] == 1
    assert sorted(os.listdir(tmp_path)) == names
    for n in names:
        a = np.load(tmp_path / n)
        assert a.dtype in (np.float32, np.float64) and a.size > 0 and np.isfinite(a).all()
