"""L2 weight-prefetch sweep: one Llama-3-8B decoder layer (5 launches) x 32 inside a CUDA graph, 8 distinct
layers' weights cycled (3.5 GB >> L2).  `pf` = k-blocks each GEMM CTA prefetches into L2 behind its smem ring;
mode 0 = TMA prefetch up front + rolling, 1 = TMA up front only, 2 = LSU prefetch.global.L2 by the epilogue warps."""
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
shapes = {"qkv": (Q + 2 * KV, H), "o": (H, Q), "gu": (2 * F, H), "down": (H, F)}
wb = sum(a * b * 2 for a, b in shapes.values())
NCU = os.environ.get("NCU") == "1"
for B in [int(b) for b in os.environ.get("B", "32").split(",")]:
    piece = NativePiece(cfg, range(NL), False, False, t, dev, max_tokens=64, max_seqs=64, num_pages=B + 2)
    i32 = torch.int32
    meta = BatchMeta(ids=torch.zeros(B, device=dev, dtype=i32), positions=torch.full((B,), 20, device=dev, dtype=i32),
                     slots=torch.arange(B, device=dev, dtype=i32) * 64 + 64 + 20, q_start=torch.arange(B, device=dev, dtype=i32),
                     q_len=torch.ones(B, device=dev, dtype=i32), kv_len=torch.full((B,), 21, device=dev, dtype=i32),
                     block_table=(torch.arange(B, device=dev, dtype=i32) + 1)[:, None].contiguous(), n_tokens=B, n_seqs=B, max_q=1)
    x = torch.randn(64, cfg.hidden_size, device=dev).bfloat16()
    if NCU:
        for pf in (0, 16, 1024 + 16, 2048 + 16):
            ops.L2_PREFETCH = pf
            for _ in range(2):
                piece.forward(meta, x_in=x)
            torch.cuda.synchronize()
        sys.exit(0)
    for stages in (0, 4, 3, 2):
        ops.GEMM_STAGES = stages
        for pf in (0, 8, 32, 64):
            ops.L2_PREFETCH = 1024 + pf
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                piece.forward(meta, x_in=x)
                s.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    for _ in range(4):
                        piece.forward(meta, x_in=x)
                g.replay(); s.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(s)
                for _ in range(5):
                    g.replay()
                e1.record(s); s.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / (5 * 4 * NL)
            print(f"B={B} stages={stages} pf(upfront)={pf:3d}: {us:7.1f} us/layer  ({wb / us / 1e3:6.0f} GB/s, data-sheet floor {wb / 3.35e6:5.1f} us)", flush=True)
    del piece
