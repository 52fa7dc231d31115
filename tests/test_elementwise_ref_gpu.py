"""The ``elementwise.cu`` kernels against a plain fp64 reference, with poison tails and sentinel rows.

Semantics (what each reference function below computes):
  * ``rmsnorm``: out = bf16(x rs (g + plus_one) + residual), rs = 1 / sqrt(mean(x^2) + eps); ``rstd_out`` = rs (fp32);
    ``ops.rstd`` writes rs alone.
  * ``layernorm``: out = bf16((x - mean) rs g + b), rs = 1 / sqrt(mean((x - mean)^2) + eps).
  * ``embed``: out = bf16(bf16(E[clamp(id, 0, vocab - 1)] * scale) + P[position]), every product and sum in fp32: the
    scaled embedding is rounded to bf16 before the position row is added (HF), and ``scale`` is used as given (the
    model passes embed_scale already rounded to bf16).
  * ``kv_append``: q_out = bf16(q * q_scale) (fp32 product); K / V copied to the cache row of the token's slot; slot -1
    writes nothing.
  * ``add``: out = bf16(a + b) (fp32 sum).
  * ``quant_fp8_rows``: s = max(amax / 448, FLT_MIN) (1 for an all-zero row), q = e4m3_satfinite(x / s), scale_out =
    s, times rs when ``with_rms``.  The FLT_MIN floor matters under ``--use_fast_math``: there amax / 448 of a row whose
    amax is below 448 FLT_MIN (about 5e-36) flushes to 0, 1 / s becomes inf and a zero element quantises to NaN.
  * ``decode_advance`` / ``set_decode_state`` / ``fetch_window``: integer bookkeeping, compared with host models.

embed, kv_append and add are exact: their bytes must equal the reference.  The norms and the quantiser run fp32 sums
(and, under ``--use_fast_math``, div.approx / rsqrt.approx / rcp.approx), so their result before the final rounding may
differ from the fp64 value.  Each such output must lie between the roundings of ref - d and ref + d (rounding is
monotone, so this admits a different code only where ref lies within d of a rounding boundary), where
  * rmsnorm:    d = C_NORM 2^-23 (|x rs (g + plus_one)| + |residual|)
  * layernorm:  d = C_NORM 2^-23 ((|x| + |mean|) rs |g| + |b|)      (the row mean cancels in x - mean)
  * quant_fp8:  d = C_Q 2^-23 |x / s|                                (e4m3 code of the value)
and fp32 results must satisfy |got - ref| <= C_RSTD 2^-23 |ref| (``rstd_out``, ``ops.rstd``, ``scale_out``).
These constants were measured with the tests below on one NVIDIA H100 80GB HBM3 (SXM) at its 700 W power limit, and
set with at least 4x margin:
    measured  c_norm = 0.323 (layernorm h=1600)   c_rstd = 0.866 (scale_out, h=256, with_rms)   c_q = 0
    set       C_NORM = 2                          C_RSTD = 4                                    C_Q = 8
(c_q = 0: every e4m3 byte equalled the rounding of the fp64 x / s.  C_Q is the instruction bound instead: div.approx
for amax / 448 (2 ulp), rcp.approx for 1 / s (1 ulp) and the product (1/2 ulp) move x / s by at most 3.5 ulp, about
3.5 2^-23 relative; C_Q doubles that.)  ``pytest -s`` prints the ``MEASURED`` table: the smallest constant each test
would have passed with.  The reference-level mutants move an output by 74x (eps x 10) to 1.7e4x (row mean dropped)
the widest deviation the bound admits; without the FLT_MIN floor the subnormal-scale row is not finite.

Poison and sentinels: inputs are the leading rows of buffers whose tail rows hold poison; outputs are the leading
rows of buffers prefilled with a sentinel that the rows behind them must keep; the KV caches carry a guard row in
front of slot 0, which a store to slot -1 would hit.  The CPU tests at the top pin the reference against
``torch_ref`` and show that each reference-level mutant (eps x 10, plus_one dropped, gamma dropped, the row mean
dropped, no FLT_MIN floor) moves an output past the bound at the inputs used here."""
from __future__ import annotations

import math
from collections import defaultdict

import pytest
import torch

gpu = pytest.mark.gpu

C_NORM = 2.0
C_RSTD = 4.0
C_Q = 8.0
U23 = 2.0 ** -23
FLT_MIN = 2.0 ** -126
SENT16 = 0x7FA5            # bf16 NaN pattern no kernel store produces
SENT8 = 0x7F               # e4m3 NaN
POISON = 16384.0
PAGE = 64

MEASURED: dict = defaultdict(float)     # constant -> smallest value each output would have passed with


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if MEASURED:
        print("\nMEASURED (smallest constant that passes):")
        for k in sorted(MEASURED):
            print(f"  {k:<40s} {MEASURED[k]:.3g}")


# ------------------------------------------------------------------------------------------ references
def rmsnorm_ref64(x, g, eps, plus_one=False, residual=None, mut=None):
    """(y64 before rounding, rs64, per-element error unit)"""
    x64 = x.double()
    e = eps * 10 if mut == "eps_x10" else eps
    rs = 1.0 / torch.sqrt(x64.pow(2).mean(-1, keepdim=True) + e)
    g64 = torch.ones_like(g.double()) if mut == "no_gamma" else g.double()
    if plus_one and mut != "drop_plus_one":
        g64 = g64 + 1.0
    y = x64 * rs * g64
    unit = y.abs()
    if residual is not None:
        y = y + residual.double()
        unit = unit + residual.double().abs()
    return y, rs.squeeze(-1), unit * U23


def layernorm_ref64(x, g, b, eps, mut=None):
    x64 = x.double()
    mean = x64.mean(-1, keepdim=True)
    if mut == "no_mean":
        mean = torch.zeros_like(mean)
    rs = 1.0 / torch.sqrt((x64 - mean).pow(2).mean(-1, keepdim=True) + eps)
    y = (x64 - mean) * rs * g.double() + b.double()
    unit = ((x64.abs() + mean.abs()) * rs * g.double().abs() + b.double().abs()) * U23
    return y, unit


def quant_fp8_ref64(x, eps, with_rms, mut=None):
    """(x / s in fp64, scale_out in fp64)"""
    x64 = x.double()
    amax = x64.abs().amax(-1)
    s = amax / 448.0
    if mut == "ftz_no_floor":
        s = torch.where(s < FLT_MIN, torch.zeros_like(s), s)       # fast-math division flushes a subnormal to 0
    else:
        s = s.clamp_min(FLT_MIN)
    s = torch.where(amax > 0, s, torch.ones_like(s))
    v = x64 / s[:, None]
    sc = s * (1.0 / torch.sqrt(x64.pow(2).mean(-1) + eps)) if with_rms else s
    return v, sc


def to_bf16(v64):
    return v64.float().to(torch.bfloat16)


def to_e4m3(v64):
    return v64.float().clamp(-448.0, 448.0).to(torch.float8_e4m3fn)


def interval_check(got, ref64, d, rnd, name):
    """got (rounded) must lie between rnd(ref - d) and rnd(ref + d); records the smallest constant that passes: where
    got differs from rnd(ref) (one code apart), the distance from ref to the midpoint of the two codes"""
    g = got.double().cpu()
    ref64, d = ref64.cpu(), d.cpu()
    lo, hi = rnd(ref64 - d).double(), rnd(ref64 + d).double()
    r = rnd(ref64).double()
    diff = g != r
    if diff.any():
        need = ((r[diff] + g[diff]) / 2 - ref64[diff]).abs() / (d[diff] / _const(name)).clamp_min(1e-300)
        MEASURED[name] = max(MEASURED[name], need.max().item())
    bad = ~((g >= lo) & (g <= hi))
    assert not bad.any(), (f"{name}: {int(bad.sum())} outputs outside the bound, first at {bad.nonzero()[0].tolist()}: "
                           f"got {g[bad][0].item()!r}, ref {ref64[bad][0].item()!r}")


def _const(name):
    return {"c_norm": C_NORM, "c_q": C_Q}[name.split(" ")[0]]


def rel_check(got, ref64, name):
    err = (got.double().cpu() - ref64.cpu()).abs() / (ref64.cpu().abs() * U23)
    MEASURED[name] = max(MEASURED[name], err.max().item())
    assert err.max().item() <= C_RSTD, f"{name}: relative error {err.max().item():.3g} x 2^-23 > C_RSTD"


# ------------------------------------------------------------------------------------------ inputs (CPU, seeded)
EPS_RMS = 1e-6
EPS_LN = 1e-5


def norm_rows(T, h, seed):
    """T rows: Llama-magnitude activations, one outlier row, one row whose mean square is about eps (so eps moves rs
    by ~30 %), one all-zero row"""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(T, h, generator=gen) * 3.0
    x[1] = torch.randn(h, generator=gen)
    x[1, h // 2] = 900.0
    x[2] = torch.randn(h, generator=gen) * math.sqrt(EPS_RMS)
    x[3] = 0.0
    return x.to(torch.bfloat16)


def spread_gamma(h, seed):
    """norm weights over [0.25, 2] (a wrong or missing gamma is O(1))"""
    gen = torch.Generator().manual_seed(seed)
    return (0.25 + 1.75 * torch.rand(h, generator=gen)).to(torch.bfloat16)


def padded(x, tail=2, fill=POISON):
    """x as the leading rows of a buffer whose ``tail`` trailing rows hold poison"""
    buf = torch.full((x.shape[0] + tail, *x.shape[1:]), fill, dtype=x.dtype, device=x.device)
    buf[: x.shape[0]] = x
    return buf


def sentinel_bf16(rows, h, device="cuda"):
    return torch.full((rows, h), SENT16, dtype=torch.int16, device=device).view(torch.bfloat16)


def is_sentinel16(t):
    return bool((t.contiguous().view(torch.int16) == SENT16).all())


# ------------------------------------------------------------------------------------------ CPU tests
def bf16_tol(y, unit):
    """the widest deviation the interval check admits: C_NORM units plus one bf16 ulp (2^-7 |y| at most)"""
    return (C_NORM * unit + y.abs() * 2.0 ** -7).clamp_min(1e-30)


def test_ref64_matches_torch_oracle():
    from bee2bee_b200.models import torch_ref
    x, g = norm_rows(8, 256, 0), spread_gamma(256, 1)
    r = torch.randn(8, 256, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16)
    for plus_one in (False, True):
        y, _, _ = rmsnorm_ref64(x, g, EPS_RMS, plus_one, r)
        want = torch_ref.rms_norm(x.float(), g.float(), EPS_RMS, plus_one) + r.float()
        assert torch.allclose(y.float(), want, rtol=1e-5, atol=1e-5)
    b = spread_gamma(256, 3)
    y, _ = layernorm_ref64(x + 100, g, b, EPS_LN)
    want = torch_ref.layer_norm((x + 100).float(), g.float(), b.float(), EPS_LN)
    assert torch.allclose(y.float(), want, rtol=1e-3, atol=1e-3)


@pytest.mark.parametrize("mut", ["eps_x10", "drop_plus_one", "no_gamma"])
def test_rmsnorm_mutant_is_exposed(mut):
    """at the inputs of the GPU test the mutant moves some output far past the bound (>= 20x)"""
    x, g = norm_rows(6, 2304, 5), spread_gamma(2304, 6)
    y, _, unit = rmsnorm_ref64(x, g - 1, EPS_RMS, True)
    ym, _, _ = rmsnorm_ref64(x, g - 1, EPS_RMS, True, mut=mut)
    margin = ((ym - y).abs() / bf16_tol(y, unit)).max().item()
    print(f"MUTANT {mut}: {margin:.3g}x the bound")
    assert margin >= 20


def test_layernorm_and_quant_mutants_are_exposed():
    x = layernorm_rows(4, 768, 7)
    g, b = spread_gamma(768, 8), spread_gamma(768, 9)
    y, unit = layernorm_ref64(x, g, b, EPS_LN)
    ym, _ = layernorm_ref64(x, g, b, EPS_LN, mut="no_mean")
    margin = ((ym - y).abs() / bf16_tol(y, unit)).max().item()
    print(f"MUTANT no_mean: {margin:.3g}x the bound")
    assert margin >= 20
    xq = quant_rows(4, 256, 10)
    v, _ = quant_fp8_ref64(xq, EPS_RMS, False)
    vm, _ = quant_fp8_ref64(xq, EPS_RMS, False, mut="ftz_no_floor")
    assert torch.isfinite(v).all() and v.abs().max() <= 448
    assert not torch.isfinite(vm[2]).all()       # s = 0: inf for the nonzero elements, NaN for the zero one


# ------------------------------------------------------------------------------------------ rmsnorm
@gpu
@pytest.mark.parametrize("h", [8, 2304, 4096, 8192])
@pytest.mark.parametrize("plus_one", [False, True])
@pytest.mark.parametrize("with_residual", [False, True])
def test_rmsnorm_matches_ref64(h, plus_one, with_residual):
    """both block sizes (256 / 512 threads), a row loop with a remainder (2304 = 288 x 8), residual, plus_one (the
    gamma stored as w - 1), rstd_out; the rows behind the outputs keep their sentinels"""
    from bee2bee_b200 import ops
    T = 7
    x = norm_rows(T, h, h)
    g = spread_gamma(h, h + 1)
    g_arg = (g.float() - 1.0).to(torch.bfloat16) if plus_one else g
    res = (torch.randn(T, h, generator=torch.Generator().manual_seed(h + 2)) * 4).to(torch.bfloat16) if with_residual else None
    xb = padded(x).cuda()
    rb = padded(res).cuda() if res is not None else None
    out = sentinel_bf16(T + 1, h)
    rstd = torch.full((T + 1,), float("nan"), device="cuda")
    ops.rmsnorm(xb[:T], g_arg.cuda(), out=out[:T], residual=rb[:T] if rb is not None else None, eps=EPS_RMS,
                plus_one=plus_one, rstd_out=rstd[:T])
    torch.cuda.synchronize()
    y, rs, unit = rmsnorm_ref64(x, g_arg, EPS_RMS, plus_one, res)
    interval_check(out[:T], y, C_NORM * unit, to_bf16, f"c_norm rmsnorm h={h}")
    rel_check(rstd[:T], rs, f"c_rstd rmsnorm h={h}")
    assert is_sentinel16(out[T]) and torch.isnan(rstd[T])
    r2 = ops.rstd(xb[:T], EPS_RMS)
    rel_check(r2, rs, f"c_rstd ops.rstd h={h}")


# ------------------------------------------------------------------------------------------ layernorm
def layernorm_rows(T, h, seed):
    """GPT-2 magnitudes, one row with a large mean (|mean| / std ~ 100)"""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(T, h, generator=gen) * 2.0
    x[0] = 100.0 + torch.randn(h, generator=gen)
    x[1, 3] = 60.0
    return x.to(torch.bfloat16)


@gpu
@pytest.mark.parametrize("h", [128, 768, 1600])
def test_layernorm_matches_ref64(h):
    from bee2bee_b200 import ops
    T = 5
    x = layernorm_rows(T, h, h)
    g = spread_gamma(h, h + 1)
    b = ((torch.rand(h, generator=torch.Generator().manual_seed(h + 2)) - 0.5) * 4).to(torch.bfloat16)
    xb = padded(x).cuda()
    out = sentinel_bf16(T + 1, h)
    ops.layernorm(xb[:T], g.cuda(), b.cuda(), out=out[:T], eps=EPS_LN)
    torch.cuda.synchronize()
    y, unit = layernorm_ref64(x, g, b, EPS_LN)
    interval_check(out[:T], y, C_NORM * unit, to_bf16, f"c_norm layernorm h={h}")
    assert is_sentinel16(out[T])


# ------------------------------------------------------------------------------------------ embed
@gpu
@pytest.mark.parametrize("h", [64, 2304])
@pytest.mark.parametrize("scale", [1.0, "bf16_sqrt", "raw_sqrt"])
@pytest.mark.parametrize("with_pos", [False, True])
def test_embed_matches_ref(h, scale, with_pos):
    """ids below 0 and at or above vocab are clamped; the position table; the scale is used as given, the scaled row
    is rounded to bf16 before the position row is added"""
    from bee2bee_b200 import ops
    vocab, n_pos = 100, 40
    if scale == "bf16_sqrt":
        scale = float(torch.tensor(math.sqrt(h), dtype=torch.bfloat16))
    elif scale == "raw_sqrt":
        scale = math.sqrt(h) * 1.01
    gen = torch.Generator().manual_seed(h)
    table = (torch.randn(vocab, h, generator=gen) * 0.05).to(torch.bfloat16)
    ptab = torch.randn(n_pos, h, generator=gen).to(torch.bfloat16)
    ids = torch.tensor([-5, -1, 0, 3, vocab - 1, vocab, vocab + 100, 57], dtype=torch.int32)
    pos = torch.tensor([0, 1, 2, 39, 17, 38, 5, 20], dtype=torch.int32)
    T = ids.numel()
    out = sentinel_bf16(T + 1, h)
    ops.embed(ids.cuda(), padded(table).cuda()[:vocab], out[:T], pos_table=padded(ptab).cuda()[:n_pos] if with_pos else None,
              positions=pos.cuda() if with_pos else None, scale=scale)
    torch.cuda.synchronize()
    e = table[ids.clamp(0, vocab - 1).long()].double()
    if scale != 1.0 or with_pos:
        e = to_bf16(e * torch.tensor(scale, dtype=torch.float32).double())      # fp32 product, then bf16
        p = ptab[pos.long()].double() if with_pos else torch.zeros_like(e, dtype=torch.float64)
        e = to_bf16(e.double() + p)
    else:
        e = e.to(torch.bfloat16)
    assert torch.equal(out[:T].cpu().view(torch.int16), e.view(torch.int16))
    assert is_sentinel16(out[T])


# ------------------------------------------------------------------------------------------ kv_append / add
@gpu
@pytest.mark.parametrize("n_heads,hd", [(2, 64), (12, 64)])
def test_kv_append_matches_ref(n_heads, hd):
    """q scaled in fp32 then rounded, K / V copied bit for bit to their slots; slot -1 leaves the cache (and the guard
    row in front of slot 0) untouched, and so do all unnamed slots"""
    from bee2bee_b200 import ops
    q_dim = kv_dim = n_heads * hd
    T, n_slots = 6, 3 * PAGE
    slots = torch.tensor([0, 65, -1, 191, 64, -1], dtype=torch.int32)
    qkv = torch.randn(T, q_dim + 2 * kv_dim, generator=torch.Generator().manual_seed(n_heads)).to(torch.bfloat16)
    q_scale = hd ** -0.5 * 1.03
    kbuf, vbuf = sentinel_bf16(1 + n_slots, kv_dim), sentinel_bf16(1 + n_slots, kv_dim)
    qbuf = sentinel_bf16(T + 1, q_dim)
    ops.kv_append(padded(qkv).cuda()[:T], qbuf, kbuf[1:], vbuf[1:], slots.cuda(), q_dim, kv_dim, q_scale)
    torch.cuda.synchronize()
    q_ref = to_bf16(qkv[:, :q_dim].double() * torch.tensor(q_scale, dtype=torch.float32).double())
    assert torch.equal(qbuf[:T].cpu().view(torch.int16), q_ref.view(torch.int16))
    assert is_sentinel16(qbuf[T])
    k_exp, v_exp = sentinel_bf16(1 + n_slots, kv_dim, "cpu"), sentinel_bf16(1 + n_slots, kv_dim, "cpu")
    for t, s in enumerate(slots.tolist()):
        if s >= 0:
            k_exp[1 + s] = qkv[t, q_dim:q_dim + kv_dim]
            v_exp[1 + s] = qkv[t, q_dim + kv_dim:]
    assert torch.equal(kbuf.cpu().view(torch.int16), k_exp.view(torch.int16))
    assert torch.equal(vbuf.cpu().view(torch.int16), v_exp.view(torch.int16))


@gpu
@pytest.mark.parametrize("n", [8, 2304 * 3, 8 * 1000 + 8])
def test_add_matches_ref(n):
    from bee2bee_b200 import ops
    gen = torch.Generator().manual_seed(n)
    a = (torch.randn(n, generator=gen) * 10).to(torch.bfloat16)
    b = (torch.randn(n, generator=gen) * 0.01).to(torch.bfloat16)
    out = sentinel_bf16(1, n + 8).view(-1)
    ops.add(a.cuda(), b.cuda(), out[:n])
    torch.cuda.synchronize()
    assert torch.equal(out[:n].cpu().view(torch.int16), to_bf16(a.double() + b.double()).view(torch.int16))
    assert is_sentinel16(out[n:])


# ------------------------------------------------------------------------------------------ quant_fp8_rows
def quant_rows(T, h, seed):
    """random rows, an all-zero row, a row whose amax / 448 is an fp32 subnormal (amax = 2^-120), one outlier row"""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(T, h, generator=gen) * 2.0
    x[1] = 0.0
    sign = torch.where(torch.rand(h, generator=gen) < 0.5, -1.0, 1.0)
    x[2] = sign * (1.0 + torch.rand(h, generator=gen)) * 2.0 ** -121          # normal values, none below FLT_MIN
    x[2, 5] = 2.0 ** -120
    x[2, 6] = 0.0
    x[3, 7] = -3000.0
    return x.to(torch.bfloat16)


@gpu
@pytest.mark.parametrize("h", [256, 4096])
@pytest.mark.parametrize("with_rms", [False, True])
def test_quant_fp8_rows_matches_ref64(h, with_rms):
    """every e4m3 byte within the bound of x / s, no NaN byte, scales within C_RSTD; the zero row gives s = 1 and the
    subnormal row s = FLT_MIN"""
    from bee2bee_b200 import ops
    T = 6
    x = quant_rows(T, h, h)
    q = torch.full((T + 1, h), SENT8, dtype=torch.uint8, device="cuda")
    sc = torch.full((T + 1,), float("nan"), device="cuda")
    ops.quant_fp8_rows(padded(x).cuda()[:T], EPS_RMS, with_rms, out=q.view(torch.float8_e4m3fn)[:T], scale_out=sc[:T])
    torch.cuda.synchronize()
    qb = q[:T].cpu()
    assert not ((qb & 0x7F) == 0x7F).any(), "NaN e4m3 bytes"
    v, s_ref = quant_fp8_ref64(x, EPS_RMS, with_rms)
    interval_check(qb.view(torch.float8_e4m3fn), v, C_Q * U23 * v.abs(), to_e4m3, f"c_q h={h} rms={int(with_rms)}")
    rel_check(sc[:T], s_ref, f"c_rstd quant_fp8 scale h={h} rms={int(with_rms)}")
    assert (q[T] == SENT8).all() and torch.isnan(sc[T])


# ------------------------------------------------------------------------------------------ bookkeeping kernels
@gpu
def test_decode_advance_at_the_last_page():
    """positions / kv_len advance for rows with q_len > 0; the slot is the block-table page of the new position, -1
    once the position passes the last page; rows with q_len = 0 keep positions and kv_len and get slot -1"""
    from bee2bee_b200 import ops
    n, mp = 6, 3
    bt = (torch.arange(n * mp, dtype=torch.int32).view(n, mp) * 7 + 2)
    pos = torch.tensor([0, 63, 127, 191, 190, 50], dtype=torch.int32)
    q_len = torch.tensor([1, 1, 1, 1, 1, 0], dtype=torch.int32)
    kv = pos + 1
    slots = torch.full((n,), 12345, dtype=torch.int32)
    dp, dk, ds = pos.cuda(), kv.cuda(), slots.cuda()
    ops.native().decode_advance(dp, dk, ds, q_len.cuda(), bt.cuda())
    want_pos, want_kv, want_slots = pos.clone(), kv.clone(), []
    for i in range(n):
        if q_len[i] <= 0:
            want_slots.append(-1)
            continue
        p = int(pos[i]) + 1
        want_pos[i], want_kv[i] = p, p + 1
        want_slots.append(int(bt[i, p // PAGE]) * PAGE + p % PAGE if p // PAGE < mp else -1)
    assert dp.cpu().tolist() == want_pos.tolist() and dk.cpu().tolist() == want_kv.tolist()
    assert ds.cpu().tolist() == want_slots
    assert want_slots[3] == -1 and want_slots[4] == int(bt[4, 2]) * PAGE + 63      # the edge of the last page


@gpu
def test_set_decode_state_skips_rows():
    """row_map < 0 skips a chunk sequence; every batch row not named keeps its state"""
    from bee2bee_b200 import ops
    B = 8
    positions = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    kv_len = torch.full((B,), -8, dtype=torch.int32, device="cuda")
    q_len = torch.full((B,), -9, dtype=torch.int32, device="cuda")
    row_map = torch.tensor([5, -1, 0, -3, 7], dtype=torch.int32, device="cuda")
    kvlen = torch.tensor([10, 99, 64, 98, 1], dtype=torch.int32, device="cuda")
    ops.native().set_decode_state(positions, kv_len, q_len, row_map.data_ptr(), kvlen.data_ptr(), row_map.numel())
    wp, wk, wq = [-7] * B, [-8] * B, [-9] * B
    for b, n in zip(row_map.tolist(), kvlen.tolist()):
        if b >= 0:
            wp[b], wk[b], wq[b] = n - 1, n, 1
    assert positions.cpu().tolist() == wp and kv_len.cpu().tolist() == wk and q_len.cpu().tolist() == wq


@gpu
@pytest.mark.parametrize("width", [1, 5, 16])
def test_fetch_window_wraps_the_ring(width):
    """out[b, j] = history[b, (cursor[b] + j) % stride], cursors placed so that cursor + width wraps the ring; no flag
    waits; the row behind the output keeps its sentinel"""
    from bee2bee_b200 import ops
    rows, stride = 4, 16
    hist = torch.arange(rows * stride, dtype=torch.int32).view(rows, stride) * 3 + 1
    cursors = torch.tensor([0, stride - 1, stride - width // 2 - 1, 7], dtype=torch.int32)
    dh, dc = hist.cuda(), cursors.cuda()
    out = torch.full((rows + 1, width), -99, dtype=torch.int32, device="cuda")
    ops.native().fetch_window(dh.data_ptr(), stride, dc.data_ptr(), rows, width, out.data_ptr(), 0, 0, 0)
    torch.cuda.synchronize()
    want = torch.stack([hist[b, (torch.arange(width) + cursors[b]) % stride] for b in range(rows)])
    assert torch.equal(out[:rows].cpu(), want)
    assert (out[rows] == -99).all()


# ------------------------------------------------------------------------------------------ host-side refusals
def _bad_call(what):
    """(callable, output tensor that must stay untouched) of one refused call"""
    from bee2bee_b200 import ops
    C = ops.native()
    T, h = 4, 256
    x = torch.ones(T, h, dtype=torch.bfloat16, device="cuda")
    g = torch.ones(h, dtype=torch.bfloat16, device="cuda")
    out = sentinel_bf16(T, h)
    if what == "rmsnorm_gamma_len":
        return lambda: C.rmsnorm(x, g[:128], None, out, None, 1e-5, False), out
    if what == "rmsnorm_out_shape":
        return lambda: C.rmsnorm(x, g, None, out[:T - 1], None, 1e-5, False), out
    if what == "rmsnorm_residual_shape":
        return lambda: C.rmsnorm(x, g, x[:T - 1], out, None, 1e-5, False), out
    if what == "rmsnorm_gamma_fp32":
        return lambda: C.rmsnorm(x, g.float(), None, out, None, 1e-5, False), out
    if what == "rmsnorm_rstd_small":
        r = torch.full((T,), float("nan"), device="cuda")
        return lambda: C.rmsnorm(x, x, None, None, r[:T - 1], 1e-5, False), r
    if what == "layernorm_beta_len":
        return lambda: C.layernorm(x, g, g[:h - 8], out, 1e-5), out
    if what == "layernorm_out_fp32":
        o = torch.full((T, h), float("nan"), device="cuda")
        return lambda: C.layernorm(x, g, g, o, 1e-5), o
    if what == "embed_pos_without_positions":
        ids = torch.zeros(T, dtype=torch.int32, device="cuda")
        return lambda: C.embed(ids.data_ptr(), x, x, None, out, 1.0, 0, 0, 0, 0), out
    if what == "embed_pos_table_width":
        ids = torch.zeros(T, dtype=torch.int32, device="cuda")
        return lambda: C.embed(ids.data_ptr(), x, x[:, :128].contiguous(), ids, out, 1.0, 0, 0, 0, 0), out
    if what == "embed_positions_strided":
        ids = torch.zeros(T, dtype=torch.int32, device="cuda")
        pos = torch.zeros(2 * T, dtype=torch.int32, device="cuda")[::2]
        return lambda: C.embed(ids.data_ptr(), x, x, pos, out, 1.0, 0, 0, 0, 0), out
    if what == "embed_out_width":
        ids = torch.zeros(T, dtype=torch.int32, device="cuda")
        o = sentinel_bf16(T, h + 8)
        return lambda: C.embed(ids.data_ptr(), x, None, None, o.view(-1)[: T * h + 8], 1.0, 0, 0, 0, 0), o
    if what.startswith("kv_append"):
        q_dim = kv_dim = 64
        qkv = torch.ones(T, q_dim + 2 * kv_dim, dtype=torch.bfloat16, device="cuda")
        q = sentinel_bf16(T, q_dim)
        kc, vc = sentinel_bf16(PAGE, kv_dim), sentinel_bf16(PAGE, kv_dim)
        slots = torch.arange(T, dtype=torch.int32, device="cuda")
        if what == "kv_append_qkv_width":
            return lambda: C.kv_append(qkv, q, kc, vc, slots, q_dim, 2 * kv_dim, 1.0), kc
        if what == "kv_append_q_out_small":
            return lambda: C.kv_append(qkv, q[:T - 1], kc, vc, slots, q_dim, kv_dim, 1.0), kc
        if what == "kv_append_slots_int64":
            return lambda: C.kv_append(qkv, q, kc, vc, slots.long(), q_dim, kv_dim, 1.0), kc
        if what == "kv_append_slots_strided":
            strided = torch.arange(2 * T, dtype=torch.int32, device="cuda")[::2]
            return lambda: C.kv_append(qkv, q, kc, vc, strided, q_dim, kv_dim, 1.0), kc
        if what == "kv_append_cache_sizes":
            return lambda: C.kv_append(qkv, q, kc, vc[:PAGE - 1], slots, q_dim, kv_dim, 1.0), kc
    if what == "add_b_numel":
        return lambda: C.add(x, x[:T - 1], out), out
    if what == "add_out_numel":
        return lambda: C.add(x, x, out[:T - 1]), out
    raise AssertionError(what)


REFUSALS = ["rmsnorm_gamma_len", "rmsnorm_out_shape", "rmsnorm_residual_shape", "rmsnorm_gamma_fp32",
            "rmsnorm_rstd_small", "layernorm_beta_len", "layernorm_out_fp32", "embed_pos_without_positions",
            "embed_pos_table_width", "embed_positions_strided", "embed_out_width", "kv_append_qkv_width",
            "kv_append_q_out_small", "kv_append_slots_int64", "kv_append_slots_strided", "kv_append_cache_sizes",
            "add_b_numel", "add_out_numel"]


@gpu
@pytest.mark.parametrize("what", REFUSALS)
def test_refused_launches(what):
    """operands of the wrong size or dtype raise before any launch and leave the output untouched"""
    call, watched = _bad_call(what)
    before = watched.clone()
    with pytest.raises(RuntimeError):
        call()
    torch.cuda.synchronize()
    assert torch.equal(watched.view(torch.uint8), before.view(torch.uint8))
