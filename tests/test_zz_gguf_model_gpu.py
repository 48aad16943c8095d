"""GGUF file -> device-resident blocks -> decode, end to end: a llama-architecture GGUF written
with gguf-py is loaded through the C++ reader (`gguf_file.GgufArchive`, `LlamaWeights.from_gguf`)
and decoded by the C++ layer stack; logits are compared with the CPU oracle model running on the
bytes read back from the same file.  GGUF llama files use the interleaved RoPE pairing, which the
fused attention kernel applies in registers (`pdl` bit 1 of mrs_paged_decode_fused)."""
import numpy as np
import pytest
import torch

from gguf_util import write_llama_gguf
from oracle.model import OracleLlama
from mistralrs_b200 import gguf_file, model as M

pytestmark = pytest.mark.gpu


def test_gguf_llama_decode_matches_oracle(cuda, tmp_path):
    cfg0 = M.LlamaConfig.tiny_test(quant="q4_k_m", n_layers=3)
    path = str(tmp_path / "tiny.gguf")
    write_llama_gguf(path, cfg0, extra_meta=False)
    with gguf_file.GgufArchive(path) as ar:
        w = M.LlamaWeights.from_gguf(ar, cuda, keep_host=True)
    cfg = w.cfg
    assert cfg.rope_neox is False and cfg.n_layers == 3
    types = {(l, n): w.layers[l][n][1] for l in range(cfg.n_layers) for n in M.LlamaWeights.GGUF_NAMES}
    types[(0, "token_embd")], types[(0, "output")] = w.tok_embd[1], w.output[1]
    run = M.LlamaRunner(w, batch=2, max_ctx=64)
    cos, sin = M.rope_tables(cfg)
    ref = OracleLlama(cfg, w.host, lambda c, name, layer: types[(layer if name not in ("token_embd", "output") else 0, name)],
                      cos, sin, "bf16")
    toks = [5, 731]
    run.set_tokens(toks)
    for pos in range(4):
        run.step()
        torch.cuda.synchronize()
        got = run.logits().float().cpu().numpy()
        want = ref.step(toks, pos)
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 4.1 * 2.0 ** -7, (pos, err)     # bf16 logits: isolated 1-3 ulp flips, as in test_model_gpu
        toks = np.argmax(want, axis=1).tolist()
        run.set_tokens(toks)


def test_uqff_llama_decode_matches_oracle(cuda, tmp_path):
    # UQFF artifact (safetensors shards + residual + config.json) -> from_uqff -> fused decode path
    from gguf_util import write_llama_uqff
    from mistralrs_b200 import uqff_file
    cfg0 = M.LlamaConfig.tiny_test(quant="q4_k_m", n_layers=3)
    d = str(tmp_path / "art")
    write_llama_uqff(d, cfg0, n_shards=2)
    with uqff_file.UqffArchive(d) as ar:
        w = M.LlamaWeights.from_uqff(ar, cuda, keep_host=True)
    cfg = w.cfg
    assert cfg.rope_neox is True
    types = {(l, n): w.layers[l][n][1] for l in range(cfg.n_layers) for n in M.LlamaWeights.GGUF_NAMES}
    types[(0, "token_embd")], types[(0, "output")] = w.tok_embd[1], w.output[1]
    run = M.LlamaRunner(w, batch=2, max_ctx=64)
    cos, sin = M.rope_tables(cfg)
    ref = OracleLlama(cfg, w.host, lambda c, name, layer: types[(layer if name not in ("token_embd", "output") else 0, name)],
                      cos, sin, "bf16")
    toks = [5, 731]
    run.set_tokens(toks)
    for pos in range(4):
        run.step()
        torch.cuda.synchronize()
        got = run.logits().float().cpu().numpy()
        want = ref.step(toks, pos)
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 4.1 * 2.0 ** -7, (pos, err)
        toks = np.argmax(want, axis=1).tolist()
        run.set_tokens(toks)


def test_prefill_composition_matches_oracle(cuda):
    # prompt processing through mmq (wgmma dequant-GEMM) + rope + KV scatter + causal attention via
    # the paged decode kernel, against the oracle stepping token by token with EXACT linears
    cfg = M.LlamaConfig.tiny_test(quant="q4_k_m", n_layers=2)
    w = M.LlamaWeights(cfg, cuda, keep_host=True)            # bf16 (f16 overflows on the synthetic 2-layer model)
    pre = M.LlamaPrefill(w, max_tokens=64)
    toks = [(131 * i + 7) % cfg.vocab for i in range(37)]
    got = pre.forward(toks, all_logits=True).float().cpu().numpy()
    cos, sin = M.rope_tables(cfg)
    ref = OracleLlama(cfg, w.host, M.tensor_type, cos, sin, "bf16", exact_gemm=True)
    want = np.stack([ref.step([t], pos)[0] for pos, t in enumerate(toks)])
    scale = np.abs(want).max()
    err = np.abs(got - want).max() / scale
    print(f"prefill composition vs exact-GEMM oracle: max err {err:.3e} of the logit scale")
    # bf16 per-tensor rounding on both sides + bf16-rounded weights in the MMA; for scale: the oracle's
    # own exact-vs-Q8_1 variants differ by 0.7 % on this model
    assert err <= 2e-2, err
    last = pre.forward(toks).float().cpu().numpy()          # decode-GEMV lm_head on the last row: Q8_1 numerics
    assert np.abs(last - want[-1]).max() / scale <= 3e-2
