"""Quick numerical probe of the wgmma GEMM across tile/split configurations (prints, never asserts)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bee2bee_b200 import ops

torch.manual_seed(0)
def run(m, n, k, bn=0, splitk=1, **kw):
    w = (torch.randn(n, k, device="cuda") * 0.05).bfloat16()
    x = torch.randn(m, k, device="cuda").bfloat16()
    try:
        out = ops.gemm(w, x, bn=bn, splitk=splitk, **kw)
        torch.cuda.synchronize()
        ref = x.float() @ w.float().t()
        err = (out.float() - ref).abs().max().item()
        print(f"m={m} n={n} k={k} bn={bn} splitk={splitk}: max_err={err:.4f} ref_max={ref.abs().max().item():.3f} "
              f"finite={bool(torch.isfinite(out.float()).all())}", flush=True)
        if err > 0.1:
            bad = ((out.float() - ref).abs() > 0.1)
            print("   bad rows(tokens):", bad.any(1).nonzero().flatten()[:8].tolist(), "bad cols(features):",
                  bad.any(0).nonzero().flatten()[:16].tolist(), "out[0,:4]", out[0, :4].tolist(), "ref[0,:4]", ref[0, :4].tolist())
    except Exception as e:
        print(f"m={m} n={n} k={k} bn={bn} splitk={splitk}: EXC {e!r}"[:300], flush=True)
        raise

print(torch.cuda.get_device_name(0), flush=True)
ops.native().init_kernels(0)
run(16, 128, 64, bn=16)
run(16, 128, 128, bn=16)
run(1, 256, 256)
run(16, 256, 1024, bn=16)
for bn in (16, 32, 64, 128, 256):
    run(bn, 256, 512, bn=bn)
run(5, 384, 2048, splitk=2)
run(5, 384, 2048, splitk=4)
run(31, 384, 2048, splitk=8)
run(300, 384, 512)
# timing: llama-3-8b decode shapes at batch 32 / 1
for (m, n, k, sk) in [(32, 6144, 4096, 3), (32, 4096, 4096, 4), (32, 28672, 4096, 1), (32, 4096, 14336, 7),
                      (32, 128256, 4096, 1), (1, 6144, 4096, 3), (1, 28672, 4096, 1), (1, 4096, 14336, 8)]:
    w = (torch.randn(n, k, device="cuda") * 0.02).bfloat16()
    x = torch.randn(m, k, device="cuda").bfloat16()
    out = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
    flush = torch.empty(200 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for it in range(6):
        flush.fill_(it)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); ops.gemm(w, x, out=out, splitk=sk); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    t = min(ts[2:])
    tcub = []
    for it in range(6):
        flush.fill_(it)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); y = x @ w.t(); e1.record(); torch.cuda.synchronize()
        tcub.append(e0.elapsed_time(e1))
    gb = (n * k * 2) / 1e9
    print(f"shape m={m} n={n} k={k} splitk={sk}: ours {t*1e3:.1f} us ({gb/t*1e3:.0f} GB/s)   cuBLAS {min(tcub[2:])*1e3:.1f} us "
          f"({gb/min(tcub[2:])*1e3:.0f} GB/s)", flush=True)
