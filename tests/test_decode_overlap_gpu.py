"""Decode GEMMs with the fused RMSNorm of their input (``norm_from_x``) must give the same bytes however the per-token
1/rms is scheduled inside the kernel.

Llama-3-8B QKV, gate/up and lm_head shapes run at T = 1 .. 64 tokens with split-K 1/2/4/8, and as flag-waiting piece
heads.  The SHA-256 of every output buffer is compared with hashes recorded on an H100 from the kernel that computed
1/rms in a prologue before its main loop (``tests/golden/decode_overlap_gemm.json``).

Regenerate the hashes (only from a build whose outputs are known good):

    python tests/test_decode_overlap_gpu.py --write
"""
import functools
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bee2bee_b200 import ops  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decode_overlap_gemm.json")
H, NQ, NKV, HD, FFN, VOCAB = 4096, 32, 8, 128, 14336, 128256
EPS = 1e-5
TOKENS = (1, 8, 31, 32, 64)
SPLITS = (1, 2, 4, 8)
SHAPES = {"qkv": (NQ + 2 * NKV) * HD, "gate_up": 2 * FFN, "lm_head": VOCAB}


def _rand(shape, seed, scale):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


@functools.lru_cache(maxsize=None)
def _weight(kind):
    return _rand((SHAPES[kind], H), {"qkv": 11, "gate_up": 12, "lm_head": 13}[kind], 0.02)


def _x(t):
    # rows of different magnitude, so every token has its own 1/rms
    x = _rand((64, H), 21, 1.0).float() * torch.linspace(0.25, 4.0, 64, device="cuda")[:, None]
    return x.to(torch.bfloat16)[:t].contiguous()


def run_case(kind, t, splitk, flag):
    """one GEMM; returns {buffer name: sha256 of its bytes}"""
    w, x = _weight(kind), _x(t)
    kw = dict(norm_from_x=True, eps=EPS, splitk=splitk)
    if flag:
        # piece head: wait until flag >= epoch + 1 (already true, so the wait passes at once)
        sync = torch.tensor([1, 0], device="cuda", dtype=torch.int32)
        kw.update(wait_flag=sync.data_ptr(), wait_epoch=sync.data_ptr() + 4)
    if kind == "qkv":
        pages = 3
        kc = torch.full((pages, ops.PAGE, NKV, HD), 7.0, device="cuda", dtype=torch.bfloat16)
        vc = kc.clone()
        q_out = torch.full((t, NQ * HD), 7.0, device="cuda", dtype=torch.bfloat16)
        pos = torch.arange(t, device="cuda", dtype=torch.int32) * 3 + 5
        slots = torch.arange(t, device="cuda", dtype=torch.int32) * 2 + 1
        ops.gemm(w, x, epi=ops.EPI_QKV_ROPE, q_out=q_out, k_cache=kc, v_cache=vc, positions=pos, slots=slots,
                 n_q_heads=NQ, n_kv_heads=NKV, head_dim=HD, rope_theta=500000.0, q_scale=HD ** -0.5, **kw)
        bufs = {"q": q_out, "k_cache": kc, "v_cache": vc}
    elif kind == "gate_up":
        bufs = {"out": ops.gemm(w, x, epi=ops.EPI_GLU, **kw)}
    else:
        bufs = {"out": ops.gemm(w, x, epi=ops.EPI_PLAIN, out_fp32=True, bn=ops.pick_bn(t), **kw)}
    torch.cuda.synchronize()
    return {name: hashlib.sha256(b.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
            for name, b in bufs.items()}


CASES = [(kind, t, sk, False) for kind in SHAPES for t in TOKENS for sk in SPLITS] + \
        [(kind, t, 0, True) for kind in ("qkv", "gate_up") for t in (8, 32)]


def case_id(kind, t, sk, flag):
    return f"{kind}-T{t}-" + ("flag" if flag else f"sk{sk}")


@functools.lru_cache(maxsize=None)
def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("kind,t,sk,flag", [pytest.param(*c, id=case_id(*c)) for c in CASES])
def test_norm_from_x_bytes_match_golden(kind, t, sk, flag):
    want = _golden()[case_id(kind, t, sk, flag)]
    got = run_case(kind, t, sk, flag)
    assert got == want, f"{case_id(kind, t, sk, flag)}: output bytes differ from the recorded hashes"
    assert run_case(kind, t, sk, flag) == got, "repeat call gave different bytes"


if __name__ == "__main__":
    assert "--write" in sys.argv, __doc__
    table = {case_id(*c): run_case(*c) for c in CASES}
    os.makedirs(os.path.dirname(GOLDEN), exist_ok=True)
    with open(GOLDEN, "w") as f:
        json.dump(table, f, indent=1, sort_keys=True)
    print(f"wrote {len(table)} cases to {GOLDEN}")
