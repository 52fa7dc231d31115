"""First-light check + timing of the tensor-core prefill attention against an fp32 reference."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from bee2bee_b200 import ops
from test_kernels_gpu import _paged_setup, _attn_ref, bf

def run(hd, nq, nkv, q_lens, kv_lens, window=0, softcap=0.0, tc=True, check=True, iters=0):
    kc, vc, bt = _paged_setup(kv_lens, nkv, hd)
    q = bf(sum(q_lens), nq * hd, scale=0.3)
    out = torch.zeros_like(q)
    qs = torch.tensor([sum(q_lens[:i]) for i in range(len(q_lens))], device="cuda", dtype=torch.int32)
    ql = torch.tensor(q_lens, device="cuda", dtype=torch.int32)
    kvl = torch.tensor(kv_lens, device="cuda", dtype=torch.int32)
    ops.set_attn_tc_min_q(16 if tc else 0)
    f = lambda: ops.attention(q, kc, vc, out, bt, qs, ql, kvl, max_q=max(q_lens), n_q=nq, n_kv=nkv, head_dim=hd,
                              window=window, softcap=softcap)
    f(); torch.cuda.synchronize()
    msg = f"hd={hd} nq={nq} nkv={nkv} q={q_lens} kv={kv_lens} w={window} cap={softcap} tc={tc}:"
    if check:
        ref = _attn_ref(q, kc, vc, bt, q_lens, kv_lens, nq, nkv, hd, window, softcap)
        err = (out.float() - ref).abs()
        msg += f" max_err {err.max().item():.4f} mean_err {err.mean().item():.5f} ref_rms {ref.pow(2).mean().sqrt().item():.3f}"
    if iters:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters): f()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        flops = 0
        for a, b in zip(q_lens, kv_lens):
            # causal: query i sees (b - a + i + 1) keys (ignoring the window)
            keys = sum(min(b - a + i + 1, window if window > 0 else 1 << 30) for i in range(a))
            flops += 4 * keys * hd * nq
        msg += f"  {ms*1e3:.1f} us  {flops/ms/1e9:.1f} TFLOP/s"
    print(msg, flush=True)

if __name__ == "__main__":
    run(128, 8, 2, [70, 1, 33, 16], [70, 9, 100, 16])
    run(128, 32, 8, [1000, 257, 640], [1000, 900, 640])
    run(128, 32, 8, [1000, 257, 640], [1000, 900, 640], window=300)
    run(256, 8, 4, [1000, 257], [1000, 900], softcap=50.0)
    run(64, 12, 12, [500, 257], [500, 900])
    for T in (1024, 4096):
        run(128, 32, 8, [T], [T], check=False, iters=10)
        run(128, 32, 8, [T], [T], check=False, iters=3, tc=False)
    run(256, 8, 4, [4096], [4096], check=False, iters=10, softcap=50.0)
    run(256, 8, 4, [4096], [4096], check=False, iters=10, softcap=50.0, window=4096)
