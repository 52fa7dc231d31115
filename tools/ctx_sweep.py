"""Decode attention over long contexts (B sequences x 1 query token, GQA 32:8, d = 128, paged KV): the CUDA-core
kernel (with and without split-KV) against the tensor-core flash kernel driven with one-token query blocks.
Reports microseconds per call, the KV bytes streamed and the fraction of the data-sheet HBM bandwidth; numerics of the
tensor-core path are checked against the fp32 reference at every context length."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from bee2bee_b200 import ops
from test_kernels_gpu import _attn_ref, bf

HBM = 3.35e12        # H100 SXM data-sheet HBM3 bandwidth
nq, nkv, hd = 32, 8, 128
for B in (32, 4):
    for ctx in (64, 512, 2048, 8192):
        pages_per = (ctx + 63) // 64 + 1
        total_pages = B * pages_per + 1
        g = torch.Generator(device="cuda").manual_seed(0)
        kc = torch.randn(total_pages, ops.PAGE, nkv, hd, device="cuda", generator=g).to(torch.bfloat16)
        vc = torch.randn(total_pages, ops.PAGE, nkv, hd, device="cuda", generator=g).to(torch.bfloat16)
        bt = (torch.randperm(total_pages - 1, device="cuda", generator=g).int() + 1)[:B * pages_per].view(B, pages_per).contiguous()
        q = bf(B, nq * hd, scale=0.3)
        out = torch.zeros_like(q)
        qs = torch.arange(B, device="cuda", dtype=torch.int32)
        ql = torch.ones(B, device="cuda", dtype=torch.int32)
        kvl = torch.full((B,), ctx, device="cuda", dtype=torch.int32)
        ws = torch.zeros(B * nkv * 16 * 4 * (hd + 2), device="cuda", dtype=torch.float32)
        kv_bytes = B * ctx * nkv * hd * 2 * 2
        ref = _attn_ref(q, kc, vc, bt, [1] * B, [ctx] * B, nq, nkv, hd, 0, 0.0) if ctx <= 2048 or B <= 4 else None
        auto = max(1, min(16, ops.NUM_SMS // (B * nkv)))
        for name, tc_min_q, splits in (("cuda-core, 1 split", 0, 1), (f"cuda-core, {max(auto, 2)} splits", 0, max(auto, 2)),
                                       ("cuda-core, 16 splits", 0, 16), ("tensor-core flash, 1-token blocks", 1, 1),
                                       (f"tensor-core flash, {max(auto, 2)} splits", 1, max(auto, 2)), ("tensor-core flash, 16 splits", 1, 16)):
            ops.set_attn_tc_min_q(2)
            f = lambda: ops.attention(q, kc, vc, out, bt, qs, ql, kvl, max_q=1, n_q=nq, n_kv=nkv, head_dim=hd, window=0,
                                      softcap=0.0, splits=splits, ws=ws, use_tc=1 if tc_min_q else 0)
            try:
                out.zero_(); f(); torch.cuda.synchronize()
            except Exception as e:
                print(f"B={B} ctx={ctx} {name}: FAILED {e}"); continue
            err = f" max_err {(out.float() - ref).abs().max().item():.4f}" if ref is not None else ""
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10): f()
            e1.record(); torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 100
            print(f"B={B:2d} ctx={ctx:5d} {name:32s}: {us:8.1f} us  {kv_bytes / us / 1e3:7.0f} GB/s ({kv_bytes / us * 1e6 / HBM:4.2f} of data-sheet HBM){err}", flush=True)
        del kc, vc
ops.set_attn_tc_min_q(2)
