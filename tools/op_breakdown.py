"""Per-op cost of a Llama-3-8B decoder layer at batch 1 / 32: each op kind alone in a CUDA graph over 8 distinct
layers' weights (HBM-streamed), PDL on.  Compare with the 5-op layer time of tools/layer_sweep.py."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bee2bee_b200 import ops
from bee2bee_b200.models.config import resolve_config
from bee2bee_b200.models.native import NativePiece, BatchMeta
from bee2bee_b200.models.weights import init_random

cfg = resolve_config("llama-3-8b")
NL = 8
dev = torch.device("cuda:0")
C = ops.native(); C.init_kernels(0)
t = init_random(cfg, range(NL), False, False, device=dev, dtype=torch.bfloat16)
H, F, Q, KV = cfg.hidden_size, cfg.ffn_size, cfg.q_dim, cfg.kv_dim
wbytes = {"qkv": (Q + 2 * KV) * H * 2, "attn": 0, "o": H * Q * 2, "gu": 2 * F * H * 2, "down": H * F * 2}
for B in (1, 32):
    piece = NativePiece(cfg, range(NL), False, False, t, dev, max_tokens=64, max_seqs=64, num_pages=B + 2)
    i32 = torch.int32
    m = BatchMeta(ids=torch.zeros(B, device=dev, dtype=i32), positions=torch.full((B,), 50, device=dev, dtype=i32),
                  slots=torch.arange(B, device=dev, dtype=i32) * 64 + 64 + 50, q_start=torch.arange(B, device=dev, dtype=i32),
                  q_len=torch.ones(B, device=dev, dtype=i32), kv_len=torch.full((B,), 51, device=dev, dtype=i32),
                  block_table=(torch.arange(B, device=dev, dtype=i32) + 1)[:, None].contiguous(), n_tokens=B, n_seqs=B, max_q=1)
    x = torch.randn(64, H, device=dev).bfloat16()[:B]
    x2, xn, c, eps = piece.xb[:B], piece.xa[:B], cfg, cfg.norm_eps
    a, hmid = piece.attn_buf[:B], piece.h_buf[:B]

    def op(kind, l):
        p = f"l{l}."
        if kind == "qkv":
            ops.gemm(piece.w[p + "wqkv"], x, norm_from_x=True, epi=ops.EPI_QKV_ROPE, eps=eps, q_out=piece.q_buf,
                     k_cache=piece.k_cache[l], v_cache=piece.v_cache[l], positions=m.positions, slots=m.slots,
                     n_q_heads=c.n_heads, n_kv_heads=c.n_kv_heads, head_dim=c.head_dim, rope_theta=c.rope_theta,
                     q_scale=c.softmax_scale)
        elif kind == "attn":
            ops.attention(piece.q_buf, piece.k_cache[l], piece.v_cache[l], piece.attn_buf, m.block_table, m.q_start, m.q_len,
                          m.kv_len, max_q=1, n_q=c.n_heads, n_kv=c.n_kv_heads, head_dim=c.head_dim, window=0, softcap=0.0,
                          splits=1, ws=piece.attn_ws)
        elif kind == "o":
            ops.gemm(piece.w[p + "wo"], a, out=x2, epi=ops.EPI_RESIDUAL, residual=x)
        elif kind == "gu":
            ops.gemm(piece.w[p + "wgu"], x2, out=hmid, epi=ops.EPI_GLU, norm_from_x=True, eps=eps)
        elif kind == "down":
            ops.gemm(piece.w[p + "w_down"], hmid, out=xn, epi=ops.EPI_RESIDUAL, residual=x2)

    tot = 0.0
    for kind in ("qkv", "attn", "o", "gu", "down", "layer"):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            def body():
                for _ in range(4):
                    for l in range(NL):
                        if kind == "layer":
                            for k2 in ("qkv", "attn", "o", "gu", "down"):
                                op(k2, l)
                        else:
                            op(kind, l)
            body(); s.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                body()
            g.replay(); s.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for _ in range(5):
                g.replay()
            e1.record(s); s.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / (5 * 4 * NL)
        if kind != "layer":
            tot += us
            ideal = wbytes[kind] / 3.35e6       # H100 SXM data-sheet HBM3 bandwidth
            print(f"B={B:2d} {kind:5s}: {us:6.1f} us   (weights at data-sheet HBM bw: {ideal:5.1f} us, overhead {us - ideal:5.1f})", flush=True)
        else:
            print(f"B={B:2d} layer: {us:6.1f} us   (sum of isolated ops {tot:6.1f}; HBM floor {sum(wbytes.values()) / 3.35e6:5.1f})", flush=True)
    del piece
