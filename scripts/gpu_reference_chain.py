"""GPU reference arm: the UNMODIFIED reference kernels (oracle/_ref/*.so, compiled from the reference sources by
oracle/build_ref.sh with the reference's own flags) chained per decoder layer the way mistral.rs chains them
(REF mistralrs-core/src/models/llama.rs:243-260 Block::forward, core/src/ops.rs:5036,5081 qkv_projections /
quantized_ffn -> mistralrs-quant/src/gguf/fast_mmvq.rs:299,472,682), captured in one CUDA graph per token like
the reference's `pipeline/cuda_graph.rs`:

    add_rms_norm -> quantize_q8_1 -> mmvq fused_qkv (same ggml type) | 3 x plain -> rotary_embedding_positions
    -> reshape_and_cache_flashinfer -> flashinfer_decode (reference split-KV policy + its merge)
    -> quantize_q8_1 -> mmvq plain (o_proj) -> add_rms_norm -> quantize_q8_1 -> mmvq fused_glu
    -> quantize_q8_1 -> mmvq plain (down_proj)                                          [13-15 launches / layer]
    ... final add_rms_norm -> quantize_q8_1 -> mmvq plain (lm_head) -> argmax

This is "the recompiled Ampere-class kernel path on the same GPU" (BASELINE.md §1), not our product: bench.py
reports it as `gpu_reference` next to `value`.  Only the KV-index advance, the embedding gather and the argmax
are ours (plumbing the reference does on the host / in candle)."""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class RefChain:
    def __init__(self, weights, M, batch=1, max_ctx=400):
        import oracle
        from mistralrs_b200 import kv_index, lib
        self.libs = {n: oracle.ref_lib(n) for n in ("mmvq", "rotary", "rmsnorm", "flashinfer")}
        missing = [n for n, l in self.libs.items() if l is None]
        if missing:
            raise RuntimeError(f"reference builds missing under oracle/_ref: {missing}")
        self.libs["flashinfer"].flashinfer_decode.restype = ctypes.c_int32
        self.w, self.M, self.cfg = weights, M, weights.cfg
        cfg, dev, dt = weights.cfg, weights.device, weights.dtype
        assert dt == torch.bfloat16 and weights.tp_size == 1
        # our runner only as the owner of KV cache / block tables / index metadata (reference split policy)
        self.run = M.LlamaRunner(weights, batch=batch, max_ctx=max_ctx, pdl=False, fused_attention=False, split_policy="reference")
        self.B = batch
        H = cfg.hidden
        kmax = max(H, cfg.inter, cfg.n_heads * cfg.head_dim)
        kp = (kmax + 511) // 512 * 512
        self.q8 = torch.empty(batch * kp // 32 * 36, dtype=torch.uint8, device=dev)
        a = lambda *s: torch.zeros(*s, dtype=dt, device=dev)
        self.h, self.o, self.zero = a(batch, H), a(batch, H), a(batch, H)
        self.kv_index, self.lib = kv_index, lib

    def _st(self):
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def _quant(self, x, K):
        kp = (K + 511) // 512 * 512
        self.libs["mmvq"].launch_mmvq_gguf_quantize_q8_1_bf16(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(self.q8.data_ptr()), K, kp, self.B, self._st())
        return kp // 32

    def _plain(self, wt, out, K, stride):
        t, ty, rows, cols = wt
        getattr(self.libs["mmvq"], f"launch_mmvq_gguf_{ty}_bf16_plain")(ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(self.q8.data_ptr()),
                                                                      ctypes.c_void_p(out.data_ptr()), K, rows, stride, rows, self.B, self._st())

    def _add_norm(self, x, res, w, res_dst, norm_dst):
        self.libs["rmsnorm"].add_rms_norm_bf16(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(res.data_ptr()), ctypes.c_void_p(w.data_ptr()),
                                               ctypes.c_void_p(res_dst.data_ptr()), ctypes.c_void_p(norm_dst.data_ptr()), self.B, self.cfg.hidden,
                                               ctypes.c_float(self.cfg.rms_eps), ctypes.c_int64(torch.cuda.current_stream().cuda_stream))

    def forward(self):
        """one token for the batch: expects run.advance() to have produced the index metadata"""
        cfg, w, r, B = self.cfg, self.w, self.run, self.B
        H, D, NH, KVH = cfg.hidden, cfg.head_dim, cfg.n_heads, cfg.n_kv_heads
        nq, nkv = NH * D, KVH * D
        P = lambda t: ctypes.c_void_p(t.data_ptr())
        m, b = r.meta, r.buf
        t, ty, rows, cols = w.tok_embd
        from mistralrs_b200 import GGML
        rc = self.lib().mrs_embedding_gather(ctypes.c_int32(GGML[ty]), P(t), ctypes.c_int32(cols), P(m["token_ids"]), ctypes.c_int32(B), P(b["x"]),
                                             ctypes.c_int32(1), self._st())
        assert rc == 0
        x, x2 = b["x"], b["x2"]
        self._add_norm(x, self.zero, w.layers[0]["attn_norm"], x, self.h)          # x + 0 ; h = norm(x)
        mm = self.libs["mmvq"]
        for l, L in enumerate(w.layers):
            s = self._quant(self.h, H)
            tq, tk, tv = L["attn_q"], L["attn_k"], L["attn_v"]
            if tq[1] == tk[1] == tv[1]:
                getattr(mm, f"launch_mmvq_gguf_{tq[1]}_bf16_fused_qkv")(P(tq[0]), P(tk[0]), P(tv[0]), P(self.q8), P(b["q"]), P(b["k"]), P(b["v"]),
                                                                        H, nq, nkv, nkv, s, B, self._st())
            else:    # REF fast_mmvq.rs fused_qkv: dtype mismatch -> three plain launches
                self._plain(tq, b["q"], H, s); self._plain(tk, b["k"], H, s); self._plain(tv, b["v"], H, s)
            self.libs["rotary"].rotary_embedding_positions(P(b["q"]), P(b["k"]), P(w.rope_cos), P(w.rope_sin), P(m["positions"]), 1, D,
                                                           ctypes.c_int64(B), D // 2, 0, NH, KVH, ctypes.c_int64(nq), ctypes.c_int64(nkv),
                                                           ctypes.c_uint32(1), ctypes.c_int64(torch.cuda.current_stream().cuda_stream))
            fi = self.libs["flashinfer"]
            fi.reshape_and_cache_flashinfer(P(b["k"]), P(b["v"]), P(r.k_cache[l]), P(r.v_cache[l]), P(m["slot_mapping"]), B, KVH, D, cfg.block_size,
                                            nkv, nkv, ctypes.c_float(1.0), ctypes.c_float(1.0), ctypes.c_uint32(1), ctypes.c_uint32(1), self._st())
            split = r.padded_tiles > B
            rc = fi.flashinfer_decode(P(b["q"]), P(r.k_cache[l]), P(r.v_cache[l]), P(m["kv_indptr"]), P(m["kv_indices"]), P(m["kv_last_page_len"]),
                                      P(m["request_indices"]), P(m["kv_tile_indices"]), P(m["o_indptr"]), P(m["kv_chunk_size"]),
                                      P(m["block_valid_mask"]), P(b["attn_out"]), P(b["tmp_v"]) if split else ctypes.c_void_p(0),
                                      P(b["tmp_s"]) if split else ctypes.c_void_p(0), B, r.padded_tiles, NH, KVH, D, cfg.block_size, nq, D,
                                      ctypes.c_float(D ** -0.5), -1, ctypes.c_float(0.0), ctypes.c_float(1.0), ctypes.c_float(1.0),
                                      ctypes.c_uint32(1), ctypes.c_uint32(1), self._st())
            assert rc == 0, rc
            s = self._quant(b["attn_out"], nq)
            self._plain(L["attn_output"], self.o, nq, s)
            self._add_norm(self.o, x, L["ffn_norm"], x2, self.h)                                 # x2 = o + x ; h = norm(x2)
            s = self._quant(self.h, H)
            tg, tu = L["ffn_gate"], L["ffn_up"]
            getattr(mm, f"launch_mmvq_gguf_{tg[1]}_bf16_fused_glu")(P(tg[0]), P(tu[0]), P(self.q8), P(b["act"]), H, tg[2], s, tg[2], B, 0, self._st())
            s = self._quant(b["act"], cfg.inter)
            self._plain(L["ffn_down"], self.o, cfg.inter, s)
            nxt = w.layers[l + 1]["attn_norm"] if l + 1 < cfg.n_layers else w.output_norm
            self._add_norm(self.o, x2, nxt, x, self.h)                                           # x = down + x2 ; h = next norm(x)
        s = self._quant(self.h, H)
        self._plain(w.output, b["logits"], H, s)
        rc = self.lib().mrs_argmax(P(b["logits"]), B, cfg.vocab, 1, P(b["out_token"]), P(b["argmax_scratch"]), 0, self._st())
        assert rc == 0

    def step(self):
        self.run.advance()
        self.forward()

    def capture(self):
        self.step(); self.run.reset()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph(keep_graph=True)
        with torch.cuda.graph(g):
            self.step()
        self.run.reset()
        self.graph = g
        return g


if __name__ == "__main__":
    import __graft_entry__ as g
    g.load_package()
    from mistralrs_b200 import model as M
    dev = torch.device("cuda:0")
    cfg = M.LlamaConfig.llama3_8b()
    if len(sys.argv) > 1:
        cfg.n_layers = int(sys.argv[1])
    w = M.LlamaWeights(cfg, dev)
    ref = RefChain(w, M)
    ours = M.LlamaRunner(w, batch=1, max_ctx=400, pdl=True)
    # same weights, same token stream: the two chains must agree (same arithmetic, different kernels)
    ref.run.set_tokens([1131]); ours.set_tokens([1131])
    for i in range(4):
        ref.step(); ours.step()
        torch.cuda.synchronize()
        a, b = ref.run.logits().float(), ours.logits().float()
        print(f"step {i}: reference-kernel chain vs ours: max |dlogit| / scale = {((a - b).abs().max() / a.abs().max()).item():.3e}, "
              f"tokens {int(ref.run.meta['token_ids'][0])} / {int(ours.meta['token_ids'][0])}", flush=True)
        ours.set_tokens(ref.run.meta["token_ids"].cpu().tolist())
    gr = ref.capture()
    ref.run.reset(256)
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    ref.run.reset(256)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(30):
        gr.replay()
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / 30 * 1e3
    print(f"reference-kernel chain: {us:.1f} us/token -> {1e6 / us:.1f} tok/s ({cfg.n_layers} layers)")
