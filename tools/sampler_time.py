"""Time ``sample`` at B=32, V=128256 (Llama-3 vocabulary), T=0.7, repetition penalty 1.15, for these settings:
off (top_p 0.95), top_k=50, top_k=50 with top_p=0.95, min_p=0.05; off with a count table (what the engine runs when a
request sets no penalty: the table is only written); presence and frequency penalties 0.5 over a count table with a
few hundred distinct ids per row, alone and with top_k=50; off with the logit-bias tables (every row's entry count 0:
what the engine runs for a request without logit_bias); a 1024-entry logit bias per row (distinct random ids, biases
in [-2, 2]).  The settings run in one process and alternate round by
round, so clock and neighbour load drift hit all of them alike.  Prints the card and its power limit."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bee2bee_b200 import ops

B, V, ITERS, ROUNDS = 32, 128256, 50, 6
dev = "cuda"
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
except OSError:
    power = "unknown"
print(f"card: {torch.cuda.get_device_name()}  power limit: {power or 'unknown'}")

torch.manual_seed(0)
logits = torch.randn(B, V, device=dev) * 4.0
out = torch.zeros(B, device=dev, dtype=torch.int32)
seen = torch.zeros(B, (V + 31) // 32, device=dev, dtype=torch.int32)
seen[:, :64] = 0x01010101                       # some ids already in the context
t = torch.full((B,), 0.7, device=dev)
rp = torch.full((B,), 1.15, device=dev)
seeds = torch.arange(B, device=dev, dtype=torch.int32)
step = torch.zeros(1, device=dev, dtype=torch.int32)
# a generation history: 400 distinct ids per row, each generated 1 to 12 times
counts = ops.counts_table(B, V, dev)
gen = torch.Generator(device="cpu").manual_seed(1)
for b in range(B):
    ids = torch.randperm(V, generator=gen)[:400]
    counts[b, ids.to(dev)] = torch.randint(1, 13, (400,), generator=gen, dtype=torch.int16).to(dev)
bias_ids, bias_vals = ops.logit_bias_table(B, 1024, dev)
for b in range(B):
    bias_ids[b] = torch.randperm(V, generator=gen)[:1024].to(dev, torch.int32)
    bias_vals[b] = (torch.rand(1024, generator=gen) * 4.0 - 2.0).to(dev)


def full(v, dtype=torch.float32):
    return torch.full((B,), v, device=dev, dtype=dtype)


rows = {
    "off (top_p 0.95)": dict(top_p=full(0.95)),
    "top_k=50": dict(top_p=full(1.0), top_k=full(50, torch.int32), min_p=full(0.0)),
    "top_k=50 top_p=0.95": dict(top_p=full(0.95), top_k=full(50, torch.int32), min_p=full(0.0)),
    "min_p=0.05": dict(top_p=full(1.0), top_k=full(0, torch.int32), min_p=full(0.05)),
    "off + count table": dict(top_p=full(0.95), counts=counts, presence=full(0.0), frequency=full(0.0)),
    "p=0.5 f=0.5": dict(top_p=full(0.95), counts=counts, presence=full(0.5), frequency=full(0.5)),
    "p=0.5 f=0.5 top_k=50": dict(top_p=full(0.95), top_k=full(50, torch.int32), min_p=full(0.0), counts=counts,
                                 presence=full(0.5), frequency=full(0.5)),
    "off + bias tables": dict(top_p=full(0.95), bias_ids=bias_ids, bias_vals=bias_vals, bias_n=full(0, torch.int32)),
    "logit_bias 1024": dict(top_p=full(0.95), bias_ids=bias_ids, bias_vals=bias_vals, bias_n=full(1024, torch.int32)),
}


def call(kw):
    ops.sample(logits, out, seen=seen, temperature=t, rep_penalty=rp, seeds=seeds, step=step, **kw)


for kw in rows.values():
    for _ in range(5):
        call(kw)
torch.cuda.synchronize()
times = {name: [] for name in rows}
for _ in range(ROUNDS):
    for name, kw in rows.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(ITERS):
            call(kw)
        e1.record()
        torch.cuda.synchronize()
        times[name].append(e0.elapsed_time(e1) * 1e3 / ITERS)
for name, ts in times.items():
    ts = sorted(ts)
    print(f"sampler B={B} V={V} {name:24s}: median {ts[len(ts) // 2]:.1f} us  (min {ts[0]:.1f}, max {ts[-1]:.1f}, "
          f"{ROUNDS} rounds x {ITERS} launches)")
