"""Per-CTA timeline of the GEMMs of consecutive decoder layers inside one CUDA graph (PDL chain, HBM-streamed
weights): where do the kernel boundaries lose time?  Stamps (%globaltimer, 256 ns ticks): 0 CTA entry, 1 set-up done,
2 producer: ring filled + producer released (pdl_wait / flag passed), 3 first MMA issued, 4 last MMA committed,
5 accumulator visible to the epilogue warps, 6 epilogue stores done, 7 CTA exit.

Per boundary between consecutive GEMMs it also prints the gap from the last exit of kernel n to the first MMA of kernel
n+1, and how many of kernel n+1's CTAs had finished set-up and issued their weight prefetch (stamp 1) before that last
exit: the weight stream that overlaps the boundary."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bee2bee_b200 import ops
from bee2bee_b200.models.config import resolve_config
from bee2bee_b200.models.native import NativePiece, BatchMeta
from bee2bee_b200.models.weights import init_random

cfg = resolve_config("llama-3-8b")
NL = 8
B = int(os.environ.get("B", "32"))
dev = torch.device("cuda:0")
C = ops.native(); C.init_kernels(0)
t = init_random(cfg, range(NL), False, False, device=dev, dtype=torch.bfloat16)
piece = NativePiece(cfg, range(NL), False, False, t, dev, max_tokens=64, max_seqs=64, num_pages=B + 2)
i32 = torch.int32
meta = BatchMeta(ids=torch.zeros(B, device=dev, dtype=i32), positions=torch.full((B,), 20, device=dev, dtype=i32),
                 slots=torch.arange(B, device=dev, dtype=i32) * 64 + 64 + 20, q_start=torch.arange(B, device=dev, dtype=i32),
                 q_len=torch.ones(B, device=dev, dtype=i32), kv_len=torch.full((B,), 21, device=dev, dtype=i32),
                 block_table=(torch.arange(B, device=dev, dtype=i32) + 1)[:, None].contiguous(), n_tokens=B, n_seqs=B, max_q=1)
x = torch.randn(64, cfg.hidden_size, device=dev).bfloat16()
names = {ops.EPI_QKV_ROPE: "qkv", ops.EPI_RESIDUAL: "o/down", ops.EPI_GLU: "gate/up", ops.EPI_PLAIN: "plain"}
s = torch.cuda.Stream()
with torch.cuda.stream(s):
    piece.forward(meta, x_in=x); s.synchronize()
    buf = torch.zeros(8 * 4096 * NL, device=dev, dtype=torch.int64)
    ops.TIMELINE = {"buf": buf, "off": 0, "log": []}
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        piece.forward(meta, x_in=x)
    log = ops.TIMELINE["log"]
    ops.TIMELINE = None
    for _ in range(3):
        g.replay()
    s.synchronize()
h = buf.cpu()
# report layers 3..5 (steady state), times relative to the first stamp of layer 3's QKV
per_layer = 4
first = log[3 * per_layer]
t0 = int(h[first[4]: first[4] + first[5] * 8].view(-1, 8)[:, 0].min())
print(f"B={B}; columns: min / median / max over the CTAs of a kernel, microseconds since layer 3 began")
print(f"{'kernel':10s} {'ctas':>5s} | {'entry':>17s} | {'setup':>17s} | {'released':>17s} | {'1st mma':>17s} | {'last mma':>17s} | {'epi done':>17s} | {'exit':>17s}")
rows = []
for (epi, n_out, k, sk, off, n) in log[3 * per_layer: 6 * per_layer]:
    v = (h[off: off + n * 8].view(n, 8).double() - t0) / 1e3
    def col(i):
        c = v[:, i]
        c = c[c > -1e6]
        return f"{c.min():5.1f} {c.median():5.1f} {c.max():5.1f}"
    nm = names.get(epi, "?") + (f"/{sk}" if sk > 1 else "")
    rows.append((nm, v))
    print(f"{nm:10s} {n:5d} | {col(0)} | {col(1)} | {col(2)} | {col(3)} | {col(4)} | {col(6)} | {col(7)}")
print()
print("boundary             | last exit -> 1st mma (us) | CTAs of n+1 with prefetch issued before the last exit of n")
for (na, va), (nb, vb) in zip(rows, rows[1:]):
    def live(c):
        return c[c > -1e6]
    last_exit = live(va[:, 7]).max()
    first_mma = live(vb[:, 3]).min()
    setup = live(vb[:, 1])
    early = int((setup < last_exit).sum())
    print(f"{na:>9s} -> {nb:9s} | {first_mma - last_exit:25.2f} | {early:4d} / {len(setup)}")
