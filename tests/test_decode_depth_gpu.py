"""A decode GEMM that asks for the default ring depth may run a shallower ring when that fits its whole grid in one
wave (Llama-3-8B down-projection at 17..32 tokens: 256 CTAs in clusters of 8).  The depth changes neither the k-block
order nor any sum, so a default-depth launch must write exactly the bytes of a launch with an explicit depth, and
leave the sentinel rows beyond the last token untouched.  Llama-3-8B shapes (lm_head with a 32768-row vocabulary) at
T = 1, 8, 31, 32, 64 with the split-K the model's launcher picks."""
import functools
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bee2bee_b200 import ops  # noqa: E402

pytestmark = pytest.mark.gpu

H, FFN, VOCAB = 4096, 14336, 32768
TOKENS = (1, 8, 31, 32, 64)
KINDS = {  # kind: (rows of W, K, epilogue)
    "o": (H, H, ops.EPI_RESIDUAL),
    "gate_up": (2 * FFN, H, ops.EPI_GLU),
    "down": (H, FFN, ops.EPI_RESIDUAL),
    "lm_head": (VOCAB, H, ops.EPI_PLAIN),
}
SENTINEL = -31.0      # exact in bf16 and fp32, and far from any output of these inputs


def _rand(shape, seed, scale):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


@functools.lru_cache(maxsize=None)
def _weight(kind):
    n, k, _ = KINDS[kind]
    return _rand((n, k), 200 + list(KINDS).index(kind), 0.02)


def run(kind, t, stages):
    n, k, epi = KINDS[kind]
    x = _rand((64, k), 7, 1.0)[:t].contiguous()
    width = n // 2 if epi == ops.EPI_GLU else n
    fp32 = kind == "lm_head"
    out = torch.full((64, width), SENTINEL, device="cuda", dtype=torch.float32 if fp32 else torch.bfloat16)
    kw = dict(epi=epi, out=out[:t], out_fp32=fp32, stages=stages)
    if epi == ops.EPI_RESIDUAL:
        kw.update(residual=_rand((64, n), 9, 1.0)[:t])
    if kind in ("gate_up", "lm_head"):
        kw.update(norm_from_x=True, eps=1e-5)
    ops.gemm(_weight(kind), x, **kw)
    torch.cuda.synchronize()
    return out


CASES = [(kind, t) for kind in KINDS for t in TOKENS]


@pytest.mark.parametrize("kind,t", CASES, ids=[f"{k}-T{t}" for k, t in CASES])
def test_default_depth_bytes_equal_explicit_depth(kind, t):
    bn = ops.pick_bn(t)
    deepest = ops.native().gemm_resolve(bn, KINDS[kind][2], KINDS[kind][1], 0, 0, 1)[0]
    got = run(kind, t, 0)
    assert bool((got[t:].float() == SENTINEL).all()), f"rows beyond T={t} were written"
    for st in sorted({deepest, 3}):
        ref = run(kind, t, st)
        assert torch.equal(got.view(torch.uint8), ref.view(torch.uint8)), f"default depth differs from {st} stages"
