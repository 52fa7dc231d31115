"""The wgmma GEMM (``gemm_tc_kernel<BN, EPI, QM>``) and every fused epilogue against a plain fp64 reference.

Random inputs under an fp32 tolerance cannot see one dropped 16-element MMA k-step or one mis-scaled MX block.  The
exact-sum probes here can: x from {-2..2} (MX: +-1), w integers in [-wmax, wmax] (wmax <= 15, exact in bf16 and
e4m3), fp8 ``w_scale`` / ``rstd`` powers of two, MX scale bytes in 124..130 (weights) and 124..127 (activations), bias
and residual on a 1/4 grid.  ``wmax`` is chosen so that sum_k |x_k w_k| * scale < 2^12 for every output (asserted), so
every partial sum, in any order, is an integer multiple of 2^-6 below 2^12: exact in the fp32 accumulator and in the
narrower accumulator Hopper's fp8 MMA is reported to have (~13-14 bits; DeepSeek-V3 section 3.3.2; not measured here).
Every (token, k-block) gets its own nonzero positions, every weight row its own dense random integers, so a dropped or
doubled k-block / k-step / swizzle chunk, a wrong row or token column, or a wrong scale changes an output.  PLAIN and
RESIDUAL outputs (and QKV without rotary) must then equal the reference rounded to the output dtype bit for bit.

``gemm_ref64`` states the semantics of ``ops.gemm``: a = (X W^T) * rs[t] * w_scale[n] + bias[n] with
  * rs = 1/rms of the raw input rows when ``norm_from_x`` is set (this wins over ``rstd`` when both are passed),
    otherwise ``rstd`` (1 when absent); MX multiplies in rsqrt(sumsq / K + eps) when ``sumsq`` is passed;
  * X and W dequantised exactly (MX: the UE8M0 scale of every 32-K block, read through the chunk layout);
  * PLAIN a (bf16 / fp32), GELU gelu_tanh(a), RESIDUAL a + residual (also to ``out2``), GLU act(a_gate) * u with the
    rows of each 128-row tile [gate 0..63 | up 0..63] and u = acc_up * rs * w_scale[up row] (no bias on u),
    QKV_ROPE rotate-half RoPE on pair-interleaved rows (row 2j = x_j, 2j+1 = x_{j+D/2}), theta = pos * rope_theta^(-2j/D),
    q * q_scale, K / V to the cache row of the token's slot (slot -1: no write).

Error model where the result cannot be exact (bounds per output element, on top of ulp(ref) of the output dtype and
2^-22 |ref| for the fp32 epilogue arithmetic):
  * transcendental epilogues: ``--use_fast_math`` turns tanhf into MUFU.TANH and the SiLU exp / division into
    approximations; the error of act(a) is bounded by C_FN 2^-23 |a| (times |u| for GLU): the absolute form also
    covers the cancellation in 1 + tanh and x / (1 + e^-x) at large negative arguments;
  * RoPE: fast-math exp2f / log2f for inv_freq and __sincosf: |d theta| <= C_THETA 2^-22 (1 + |theta|), times the pair
    norm (and q_scale);
  * rsqrtf and fast division for 1/rms (``norm_from_x``, MX ``sumsq``): C_RS 2^-23 |acc * scale|;
  * realistic random inputs (Llama magnitudes, K up to 14336): C_ACC[QM] 2^-23 sum_k |x_k w_k| * scale.
C_ACC, C_THETA, C_FN and C_RS were measured with the tests below on one NVIDIA H100 80GB HBM3 (SXM) at its 700 W power
limit, and set with at least 4x margin:
    measured  c_acc[0] = 4.7   c_acc[1] = 3.3e3   c_acc[2] = 41.5   c_theta = 1.46   c_fn = 5.4   c_rs = 0
    set       C_ACC[0] = 24    C_ACC[1] = 16384   C_ACC[2] = 192    C_THETA = 8      C_FN = 32    C_RS = 4
(c_rs = 0: across the ``norm_from_x`` and MX ``sumsq`` cases, fp32 outputs included, every 1/rms error stayed inside
the 2^-22 |ref| term; C_RS keeps a few rsqrt.approx / div.approx ulps on top.)  The per-row fp8
path (QM 1) is ~700x worse than bf16: it accumulates all of K in the wgmma accumulator.  MX moves every 32-K partial
into fp32 registers, but each partial is itself summed in the fp8 MMA's accumulator, so it lands ~9x above bf16.  Every GPU test prints a ``MEASURED`` table of max(|err| / bound) per
(QM, epilogue) and the measured constants (``pytest -s``).

Poison and sentinels: X and W are the leading rows of buffers whose tail rows hold large poison; outputs go through
``ld_out`` > width into buffers prefilled with a NaN sentinel that rows >= m_tok and columns >= width keep; the KV cache
and q buffer are prefilled too, and unnamed slots and slot -1 keep the sentinel.  Every call runs twice and must give
identical bytes.  The CPU tests at the top pin the reference against the torch oracle and the ops helpers, prove the
probe sums order-independent, and show that every reference-level mutant is exposed."""
from __future__ import annotations

import math
import zlib
from collections import defaultdict

import pytest
import torch

gpu = pytest.mark.gpu

EPI_PLAIN, EPI_RESIDUAL, EPI_GLU, EPI_QKV_ROPE, EPI_GELU = 0, 1, 2, 3, 4
EPI_NAMES = {EPI_PLAIN: "plain", EPI_RESIDUAL: "residual", EPI_GLU: "glu", EPI_QKV_ROPE: "qkv", EPI_GELU: "gelu"}
BNS = (16, 32, 64, 128, 256)
DEFAULT_STAGES = {16: 5, 32: 5, 64: 4, 128: 6, 256: 4}     # GemmCfg<BN>::kStages
BKE = {0: 64, 1: 128, 2: 128}                               # K elements per 128-byte k-block
INSTANTIATIONS = [(bn, epi, qm) for bn in BNS for epi in EPI_NAMES for qm in (0, 1, 2) if not (qm == 2 and bn == 16)]
SUM_LIMIT = 4096                                            # every probe output: sum |x w| * scale < 2^12
POSITIONS = (0, 1, 63, 64, 4095, 8191, 32767, 131071)
QKV_HEADS = ((64, 2, 2), (128, 2, 1))                       # (head_dim, n_q_heads, n_kv_heads)
EPS = 1e-5

C_ACC = {0: 24.0, 1: 16384.0, 2: 192.0}
C_THETA = 8.0
C_FN = 32.0
C_RS = 4.0

SENT16 = 0x7FA5            # bf16 NaN pattern no kernel store produces
SENT32 = 0x7FC0DEAD
POISON = 16384.0           # bf16 poison rows of X / W (fp8: 448)

MEASURED: dict = defaultdict(float)     # (QM, epilogue) -> max |err| / bound
C_MEASURED: dict = defaultdict(float)   # constant -> max |err| / (its unit), the value the constant must exceed


# --------------------------------------------------------------------------- operands
def _bytes_to_scale(b):
    return torch.exp2(b.double() - 127.0)


def sf_chunks(sf, bn):
    """[rows, K/32] UE8M0 bytes of activations -> the GEMM's chunk layout for token tile ``bn`` (inverse of
    ``ops.mx_unchunk``); rows of the padded last tile hold ``pad`` bytes"""
    rows, nb = sf.shape
    halves = 2 if bn > 128 else 1
    tiles = (rows + bn - 1) // bn
    full = torch.full((tiles * bn, nb), 140, dtype=torch.uint8, device=sf.device)   # poison scale 2^13 past m_tok
    full[:rows] = sf
    pad = torch.full((tiles, halves * 128, nb), 140, dtype=torch.uint8, device=sf.device)
    pad[:, :bn] = full.view(tiles, bn, nb)
    v = pad.view(tiles, halves, 4, 32, nb // 4, 4)                  # tile, half, r/32, r%32, kc, j
    return v.permute(0, 4, 1, 3, 2, 5).contiguous().view(-1)       # tile, kc, half, r%32, r/32, j


def probe_x(qm, m, k, g):
    """probe activations [m, K]: ``npk`` nonzeros (+-1..+-xmag) in every (token, k-block), each in its own 16-byte
    swizzle chunk c = (t + 3 kb + 2 p) % 8 (p < npk) at a random offset inside the chunk.  Every token therefore hits
    all 8 chunks -- and so all 4 MMA k-steps and, for MX, all 4 scale blocks -- of the k-block row within any two
    (npk 4, 3 is odd) or eight (npk 1, 2) consecutive k-blocks; ``test_probe_positions_cover_every_target`` checks it
    per case.  Returns (x fp32, npk, xmag)."""
    dev = g.device
    bke = BKE[qm]
    nkb = k // bke
    npk = 4 if nkb <= 8 else (2 if nkb <= 32 else 1)
    xmag = 1 if qm == 2 else 2
    ce = bke // 8                                                    # elements per 16-byte chunk
    t = torch.arange(m, device=dev)[:, None, None]
    kb = torch.arange(nkb, device=dev)[None, :, None]
    p = torch.arange(npk, device=dev)[None, None, :]
    pos = ((t + 3 * kb + 2 * p) % 8) * ce + torch.randint(0, ce, (m, nkb, npk), generator=g, device=dev)
    sign = torch.randint(0, 2, (m, nkb, npk), generator=g, device=dev) * 2 - 1
    vals = (torch.randint(1, xmag + 1, (m, nkb, npk), generator=g, device=dev) * sign).float()
    x = torch.zeros(m, nkb, bke, device=dev).scatter_(-1, pos, vals).view(m, k)
    return x, npk, xmag


class Operands:
    """W [n_out, K] and X [m, K] as the kernel reads them (bf16 / e4m3 / e4m3 + UE8M0 chunks), each the leading rows of
    a buffer whose tail rows hold poison, with the per-row / per-token scales and the exact fp64 dequantised values.
    kind "probe": the exact-sum inputs of the module docstring; "random": Llama-magnitude inputs (needs the extension
    for fp8 / MX quantisation)."""

    def __init__(self, qm, m, k, n_out, bn, seed, device, *, kind="probe", rstd=False, sumsq=False):
        self.qm, self.m, self.k, self.n_out, self.bn = qm, m, k, n_out, bn
        g = torch.Generator(device=device).manual_seed(seed)
        self.gen, self.device = g, device
        self.sfa_plain = self.sfb_plain = self.sfa = self.sfb = self.sumsq = None
        self.w_scale = None
        self.rstd = None
        ri = lambda lo, hi, *shape: torch.randint(lo, hi, shape, generator=g, device=device)  # noqa: E731
        if kind == "probe":
            x, npk, xmag = probe_x(qm, m, k, g)
            nkb = k // BKE[qm]
            smax = 1.0
            if qm == 2:
                self.sfa_plain = ri(124, 131, n_out, k // 32).to(torch.uint8)
                self.sfb_plain = ri(124, 128, m, k // 32).to(torch.uint8)
                smax = 8.0
            wmax = min(15, int((SUM_LIMIT - 1) // (xmag * smax * nkb * npk)))
            assert wmax >= 1
            # no zero weight: every nonzero x meets a nonzero w in every weight row of the tile
            w = (ri(1, wmax + 1, n_out, k) * (ri(0, 2, n_out, k) * 2 - 1)).float()
            if qm == 1:
                self.w_scale = torch.exp2(ri(-2, 3, n_out).float())
            if qm == 1 or rstd:
                self.rstd = torch.exp2(ri(-2, 2, m).float())
            if sumsq:
                self.sumsq = (ri(1, 5, m) * k).float()              # 1/rms in [0.5, 1]
        else:
            w = torch.randn(n_out, k, generator=g, device=device) * 0.02
            x = torch.randn(m, k, generator=g, device=device)
            if qm == 1:
                from bee2bee_b200 import ops
                wq, self.w_scale = ops.quantize_weight_fp8(w.to(torch.bfloat16))
                xq, self.rstd = ops.quant_fp8_rows(x.to(torch.bfloat16))
                w, x = wq.float(), xq.float()
            elif qm == 2:
                from bee2bee_b200 import ops
                wq, sfa = ops.quantize_weight_mxfp8(w.to(torch.bfloat16))
                xq, sfb = ops.quant_mxfp8_rows(x.to(torch.bfloat16), bn)
                self.sfa_plain = ops.mx_unchunk(sfa, n_out, k, 128)
                self.sfb_plain = ops.mx_unchunk(sfb, m, k, bn)
                w, x = wq.float(), xq.float()
        dt = torch.bfloat16 if qm == 0 else torch.float8_e4m3fn
        poison = POISON if qm == 0 else 448.0
        wbuf = torch.full((n_out + 128, k), poison, device=device)
        wbuf[:n_out] = w
        xbuf = torch.full((m + 8, k), poison, device=device)
        xbuf[:m] = x
        self.wbuf, self.xbuf = wbuf.to(dt), xbuf.to(dt)
        self.w, self.x = self.wbuf[:n_out], self.xbuf[:m]
        self.wd, self.xd = self.w.double(), self.x.double()
        if qm == 2:
            self.wd = self.wd * _bytes_to_scale(self.sfa_plain).repeat_interleave(32, 1)
            self.xd = self.xd * _bytes_to_scale(self.sfb_plain).repeat_interleave(32, 1)
            from bee2bee_b200 import ops
            self.sfa = ops.mx_chunk_layout(self.sfa_plain)
            self.sfb = sf_chunks(self.sfb_plain, bn)
        if kind == "probe":        # the accumulators (rstd / w_scale are powers of two applied after them)
            s = self.xd.abs() @ self.wd.abs().t()
            assert s.max().item() < SUM_LIMIT, s.max().item()

    def rs(self, norm_from_x=False, eps=EPS):
        """per-token scale of the accumulators (fp64)"""
        if norm_from_x:
            return torch.rsqrt(self.xd.pow(2).mean(-1) + eps)
        r = self.rstd.double() if self.rstd is not None else torch.ones(self.m, dtype=torch.float64, device=self.device)
        if self.sumsq is not None:
            r = r * torch.rsqrt(self.sumsq.double() / self.k + eps)
        return r

    def wsc(self):
        if self.w_scale is None:
            return torch.ones(self.n_out, dtype=torch.float64, device=self.device)
        return self.w_scale.double()

    def scale(self, norm_from_x=False):
        return self.rs(norm_from_x)[:, None] * self.wsc()[None, :]


# --------------------------------------------------------------------------- fp64 reference
def gelu64(a):
    return 0.5 * a * (1.0 + torch.tanh(0.7978845608028654 * (a + 0.044715 * a * a * a)))


def silu64(a):
    return a / (1.0 + torch.exp(-a))


def qkv_rows(n_q, n_kv, hd, device="cpu"):
    """per output row: section (0 q, 1 k, 2 v), index within the section, rotary pair index j"""
    q_dim, kv_dim = n_q * hd, n_kv * hd
    f = torch.arange(q_dim + 2 * kv_dim, device=device)
    sect = (f >= q_dim).long() + (f >= q_dim + kv_dim).long()
    start = torch.tensor([0, q_dim, q_dim + kv_dim], device=device)[sect]
    f_in = f - start
    return sect, f_in, (f_in % hd) // 2


def gemm_ref64(op, epi, *, bias=None, residual=None, act_gelu=False, norm_from_x=False, eps=EPS, qkv=None, mut=None):
    """``ops.gemm`` in fp64 (module docstring).  Returns a dict: "out" (PLAIN / GELU / RESIDUAL / GLU) or "q", "k",
    "v" (QKV_ROPE, per token; the cache rows are placed by the caller), "mag" (sum |x w| * scale per output, before
    the epilogue function), "fn" (the magnitude C_FN / C_RS / C_THETA bounds scale with), and "theta" (QKV).
    ``mut`` names a reference-level mutant (the discrimination checks): drop_kb, dup_split, shift_tok, swap_wg,
    swap_gate_up, gate_wscale, mx_neighbour, pos_plus1, sin_flip."""
    mut = mut or {}
    xd, wd = op.xd, op.wd
    if "mx_neighbour" in mut:
        nb = op.sfa_plain.shape[1]
        j = torch.arange(nb, device=op.device) ^ 1
        wd = op.w.double() * _bytes_to_scale(op.sfa_plain[:, j]).repeat_interleave(32, 1)
    K, bke = op.k, BKE[op.qm]
    nkb = K // bke
    kmul = torch.ones(K, dtype=torch.float64, device=op.device)
    if "drop_kb" in mut:
        b = mut["drop_kb"] % nkb
        kmul[b * bke:(b + 1) * bke] = 0.0
    if "dup_split" in mut:
        s = mut["dup_split"]
        for r in range(1, s):
            b = nkb * r // s
            kmul[b * bke:(b + 1) * bke] = 2.0
    acc = (xd * kmul) @ wd.t()
    mag = (xd.abs() * kmul) @ wd.abs().t()
    m, n_out = acc.shape
    if "shift_tok" in mut:
        acc = torch.cat([acc[1:], acc.new_zeros(1, n_out)], 0)
    if "swap_wg" in mut:
        acc = acc.view(m, n_out // 128, 2, 64).flip(2).reshape(m, n_out)
    rs = op.rs(norm_from_x, eps)[:, None]
    wsc = op.wsc()[None, :]
    b = bias.double()[None, :] if bias is not None else torch.zeros(1, n_out, dtype=torch.float64, device=op.device)
    pre = acc * rs * wsc
    a = pre + b
    mag = mag * (rs * wsc).abs()
    res = {"mag": mag, "pre": pre}
    if epi == EPI_PLAIN:
        res["out"], res["fn"] = a, a.abs() * 0
    elif epi == EPI_GELU:
        res["out"], res["fn"] = gelu64(a), a.abs()
    elif epi == EPI_RESIDUAL:
        res["out"], res["fn"] = a + residual.double(), a.abs() * 0
    elif epi == EPI_GLU:
        t = n_out // 128
        rg = (torch.arange(t, device=op.device)[:, None] * 128 + torch.arange(64, device=op.device)[None]).reshape(-1)
        ru = rg + 64
        ag = a[:, rg]
        wsc_u = op.wsc()[rg if "gate_wscale" in mut else ru][None, :]
        u = acc[:, ru] * rs * wsc_u
        act = gelu64 if act_gelu else silu64
        if "swap_gate_up" in mut:
            res["out"] = act(u) * ag
        else:
            res["out"] = act(ag) * u
        res["fn"] = ag.abs() * u.abs()
        res["mag"] = mag[:, rg] * u.abs() + mag[:, ru] * ag.abs()
    elif epi == EPI_QKV_ROPE:
        n_q, n_kv, hd, theta, q_scale, pos = (qkv[k] for k in ("n_q", "n_kv", "hd", "theta", "q_scale", "positions"))
        sect, f_in, j = qkv_rows(n_q, n_kv, hd, op.device)
        o, th = a.clone(), torch.zeros_like(a)
        if theta > 0:
            p = pos.double() + (1.0 if "pos_plus1" in mut else 0.0)
            inv = theta ** (-2.0 * j.double() / hd)
            th = p[:, None] * inv[None, :]
            rot = (sect < 2)[None, :]
            idx = torch.arange(n_out, device=op.device)
            partner = a[:, idx ^ 1]
            odd = (idx % 2 == 1)[None, :]
            sn = torch.sin(th)
            if "sin_flip" in mut:
                sn = torch.where(odd, -sn, sn)
            rot_o = torch.where(odd, a * torch.cos(th) + partner * sn, a * torch.cos(th) - partner * sn)
            o = torch.where(rot, rot_o, a)
            res["fn"] = torch.where(rot, torch.sqrt(a * a + partner * partner), a * 0)
            th = torch.where(rot, th, th * 0)
        else:
            res["fn"] = a.abs() * 0
        q_dim, kv_dim = n_q * hd, n_kv * hd
        qs = torch.ones(n_out, dtype=torch.float64, device=op.device)
        qs[:q_dim] = q_scale
        o = o * qs
        res["fn"] = res["fn"] * qs
        res["theta"] = th
        res["q"], res["k"], res["v"] = o[:, :q_dim], o[:, q_dim:q_dim + kv_dim], o[:, q_dim + kv_dim:]
        res["out"] = o
    return res


def bf16_ulp(ref):
    _, e = torch.frexp(ref)
    return torch.where(ref == 0, torch.zeros_like(ref), torch.ldexp(torch.ones_like(ref), (e - 8).clamp(min=-133)))


def fp32_ulp(ref):
    _, e = torch.frexp(ref)
    return torch.where(ref == 0, torch.zeros_like(ref), torch.ldexp(torch.ones_like(ref), (e - 24).clamp(min=-149)))


def _ratio(err, b):
    """err / b with 0 / 0 = 0 (an exactly zero output where the bound is zero)"""
    return torch.where(b > 0, err / b, torch.where(err > 0, math.inf, 0.0))


def bound(ref, res, epi, qm, *, fp32=False, exact_pre=True, rs_approx=False, theta=0.0):
    """per-element error bound of the module docstring; returns (bound, {constant: its unit})"""
    units = {}
    base = (fp32_ulp(ref) if fp32 else bf16_ulp(ref)) + 2.0 ** -22 * ref.abs()
    if epi in (EPI_GELU, EPI_GLU):
        units["c_fn"] = 2.0 ** -23 * res["fn"]
    if epi == EPI_QKV_ROPE and theta > 0:
        units["c_theta"] = 2.0 ** -22 * (1.0 + res["theta"].abs()) * res["fn"]
    if rs_approx:
        units["c_rs"] = 2.0 ** -23 * res["pre"].abs()
    if not exact_pre:
        units["c_acc%d" % qm] = 2.0 ** -23 * res["mag"]
    consts = {"c_fn": C_FN, "c_theta": C_THETA, "c_rs": C_RS, "c_acc0": C_ACC[0], "c_acc1": C_ACC[1], "c_acc2": C_ACC[2]}
    b = base.clone()
    for k, u in units.items():
        b = b + consts[k] * u
    return base, b, units


# --------------------------------------------------------------------------- CPU: the reference and the probes
def _ops():
    from bee2bee_b200 import ops
    return ops


def test_ref64_matches_torch_oracle_and_helpers():
    """PLAIN / GELU / GLU / QKV semantics against torch_ref and the ops row-interleave helpers; the MX dequantisation
    against ops.mx_dequant / mx_unchunk; the activation chunk layout against mx_chunk_layout at bn 128"""
    from bee2bee_b200.models import torch_ref
    ops = _ops()
    op = Operands(0, 7, 256, 256, 16, 1, "cpu")
    bias = torch.randn(256)
    r = gemm_ref64(op, EPI_PLAIN, bias=bias)
    x, w = op.x.double(), op.w.double()
    torch.testing.assert_close(r["out"], x @ w.t() + bias.double(), rtol=0, atol=0)
    r = gemm_ref64(op, EPI_GELU, bias=bias)
    torch.testing.assert_close(r["out"].float(), torch_ref.gelu_tanh((x @ w.t() + bias.double()).float()), rtol=1e-5,
                               atol=1e-5)
    # norm_from_x: torch_ref.rms_norm with gamma = 1
    ref = torch_ref.rms_norm(op.x.float(), torch.ones(256), EPS, False).double() @ w.t()
    torch.testing.assert_close(gemm_ref64(op, EPI_PLAIN, norm_from_x=True)["out"], ref, rtol=1e-5, atol=1e-5)
    # GLU through glu_interleave_rows
    wg, wu = torch.randn(128, 256).to(torch.bfloat16), torch.randn(128, 256).to(torch.bfloat16)
    op.w = ops.glu_interleave_rows(wg, wu)
    op.wd = op.w.double()
    op.n_out = 256
    for gelu in (False, True):
        g, u = x @ wg.double().t(), x @ wu.double().t()
        act = torch_ref.gelu_tanh(g.float()).double() if gelu else torch.nn.functional.silu(g)
        torch.testing.assert_close(gemm_ref64(op, EPI_GLU, act_gelu=gelu)["out"], act * u, rtol=1e-5, atol=1e-4)
    # QKV: rope_interleave_rows + torch_ref.rope (fp32 angles: small positions)
    hd, nq, nkv = 64, 2, 1
    wq, wk, wv = (torch.randn(n * hd, 256).to(torch.bfloat16) for n in (nq, nkv, nkv))
    op.w = torch.cat([ops.rope_interleave_rows(wq, nq, hd), ops.rope_interleave_rows(wk, nkv, hd), wv], 0)
    op.wd, op.n_out = op.w.double(), op.w.shape[0]
    pos = torch.tensor([0, 1, 2, 5, 17, 40, 99], dtype=torch.int32)
    r = gemm_ref64(op, EPI_QKV_ROPE, qkv=dict(n_q=nq, n_kv=nkv, hd=hd, theta=10000.0, q_scale=0.5, positions=pos))
    perm = torch.arange(hd).view(2, hd // 2).t().reshape(-1)
    q = torch_ref.rope((x @ wq.double().t()).float().view(1, 7, nq, hd), pos.long()[None], 10000.0)[0] * 0.5
    k = torch_ref.rope((x @ wk.double().t()).float().view(1, 7, nkv, hd), pos.long()[None], 10000.0)[0]
    torch.testing.assert_close(r["q"].float(), q[:, :, perm].reshape(7, -1), rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(r["k"].float(), k[:, :, perm].reshape(7, -1), rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(r["v"], x @ wv.double().t(), rtol=0, atol=0)
    # MX dequantisation and chunk layouts
    mx = Operands(2, 40, 512, 256, 32, 2, "cpu")
    wd = ops.mx_dequant(mx.w, ops.mx_unchunk(mx.sfa, 256, 512, 128)).double()
    torch.testing.assert_close(mx.wd, wd, rtol=0, atol=0)
    for bn in (32, 64, 128, 256):
        assert torch.equal(ops.mx_unchunk(sf_chunks(mx.sfb_plain, bn), 40, 512, bn), mx.sfb_plain)
    sf = torch.randint(0, 255, (256, 16), dtype=torch.uint8)
    assert torch.equal(sf_chunks(sf, 128), ops.mx_chunk_layout(sf))


@pytest.mark.parametrize("qm", [0, 1, 2])
@pytest.mark.parametrize("k", [192, 1024, 14336])
def test_probe_sums_are_order_independent(qm, k):
    """fp32 sums of the scaled probe products in three orders (forward, reverse, per k-block then across) equal fp64"""
    k = k if qm == 0 or k % 128 == 0 else k * 2
    op = Operands(qm, 5, k, 128, 32, k + qm, "cpu", rstd=True)
    prod = op.xd[:, None, :] * op.wd[None, :, :]                       # [m, n, K] exact in fp64 and fp32
    ref = prod.sum(-1)
    p32 = prod.float()
    assert torch.equal(p32.double(), prod)
    fwd = p32.cumsum(-1)[..., -1]
    rev = p32.flip(-1).cumsum(-1)[..., -1]
    blk = p32.view(5, 128, -1, BKE[qm]).cumsum(-1)[..., -1].flip(-1).cumsum(-1)[..., -1]
    for s in (fwd, rev, blk):
        assert torch.equal(s.double(), ref)
    assert (op.xd.abs() @ op.wd.abs().t()).max() < SUM_LIMIT


def _mutant_case(name):
    """(operands, epilogue, reference kwargs, mutant, exact?) aimed at one mutant"""
    qkv = dict(n_q=2, n_kv=1, hd=64, theta=10000.0, q_scale=0.5,
               positions=torch.tensor([0, 1, 63, 64, 4095, 8191, 131071], dtype=torch.int32))
    if name == "drop_kb":
        return Operands(0, 5, 5 * 64, 128, 16, 3, "cpu"), EPI_PLAIN, {}, dict(drop_kb=4), True
    if name == "dup_split":
        return Operands(0, 5, 7 * 64, 128, 16, 4, "cpu"), EPI_PLAIN, {}, dict(dup_split=4), True
    if name == "shift_tok":
        return Operands(0, 5, 256, 128, 16, 5, "cpu"), EPI_PLAIN, {}, dict(shift_tok=1), True
    if name == "swap_wg":
        return Operands(1, 5, 256, 256, 16, 6, "cpu"), EPI_RESIDUAL, {}, dict(swap_wg=1), True
    if name == "swap_gate_up":
        return Operands(0, 5, 256, 256, 16, 7, "cpu"), EPI_GLU, {}, dict(swap_gate_up=1), False
    if name == "gate_wscale":
        return Operands(1, 5, 256, 256, 16, 8, "cpu"), EPI_GLU, {}, dict(gate_wscale=1), False
    if name == "mx_neighbour":
        return Operands(2, 5, 512, 128, 32, 9, "cpu"), EPI_PLAIN, {}, dict(mx_neighbour=1), True
    if name in ("pos_plus1", "sin_flip"):
        return Operands(0, 7, 256, 256, 16, 10, "cpu"), EPI_QKV_ROPE, dict(qkv=qkv), {name: 1}, False
    raise ValueError(name)


@pytest.mark.parametrize("name", ["drop_kb", "dup_split", "shift_tok", "swap_wg", "swap_gate_up", "gate_wscale",
                                  "mx_neighbour", "pos_plus1", "sin_flip"])
def test_reference_mutant_is_exposed(name):
    """each mutant changes the exact (bf16-rounded) output of the case aimed at it, or leaves the toleranced case's
    bound by >= 20x"""
    op, epi, kw, mut, exact = _mutant_case(name)
    if epi == EPI_RESIDUAL:
        kw["residual"] = torch.randint(-255, 256, (op.m, op.n_out)).float() / 4
    good = gemm_ref64(op, epi, **kw)
    bad = gemm_ref64(op, epi, mut=mut, **kw)
    if exact:
        assert not torch.equal(good["out"].to(torch.bfloat16), bad["out"].to(torch.bfloat16))
    else:
        theta = kw["qkv"]["theta"] if "qkv" in kw else 0.0
        _, b, _ = bound(good["out"], good, epi, op.qm, theta=theta)
        ratio = _ratio((bad["out"] - good["out"]).abs(), b).max().item()
        assert ratio >= 20.0, ratio


def test_reference_mutant_slot_minus_one_is_exposed():
    """a kernel without the slot >= 0 guard stores the token of slot -1 at cache + (-1) * kv_dim: the guard row in front
    of the cache, which the GPU check requires to keep the sentinel"""
    slots = torch.tensor([3, -1, 0])
    cache = place_cache(torch.ones(3, 4, dtype=torch.float64), slots, 6, write_minus_one=False)
    bad = place_cache(torch.ones(3, 4, dtype=torch.float64), slots, 6, write_minus_one=True)
    assert cache[0].isnan().all() and not bad[0].isnan().any()
    assert torch.equal(cache[1:].isnan(), bad[1:].isnan())


def place_cache(rows, slots, n_slots, write_minus_one=False):
    """expected cache buffer [1 + n_slots, width] (NaN = sentinel): row 0 is the guard row in front of the cache, slot s
    is row s + 1.  ``write_minus_one`` models a kernel that stores slot -1 unguarded (into the guard row)."""
    out = torch.full((n_slots + 1, rows.shape[1]), float("nan"), dtype=torch.float64, device=rows.device)
    for t, s in enumerate(slots.tolist()):
        if s >= 0 or write_minus_one:
            out[s + 1] = rows[t]
    return out


# --------------------------------------------------------------------------- the sweep
def _case_list():
    """(qm, epi, bn, m, k, n_out, stages, splitk, opts): every instantiation once, the options cycled through the
    shapes of the issue's sweep, plus the long-K / Llama-width / narrow-slice cases"""
    cases = []
    per_bn = defaultdict(int)          # shapes cycle per BN ...
    per_kernel = defaultdict(int)      # ... options per (QM, epilogue), so each option meets every QM / epilogue it applies to
    for qm_, epi_, bn_ in [(q, e, b) for b, e, q in INSTANTIATIONS]:
        i = per_bn[bn_]
        per_bn[bn_] += 1
        j = per_kernel[(qm_, epi_)]
        per_kernel[(qm_, epi_)] += 1
        m = (1, bn_ - 1, bn_, bn_ + 1, 2 * bn_ + 3)[i % 5]
        stages = (2, 3, 0)[(i + i // 5) % 3]
        st = stages or DEFAULT_STAGES[bn_]
        splitk = (1, 2, 4, 8)[(i + bn_ // 16) % 4]
        nkb = (st + 1, 2 * st + 1, 2 * st + 3)[(i // 3) % 3]
        nkb = max(nkb, splitk)
        if nkb % splitk == 0 and splitk > 1:
            nkb += 1
        # fp32 output also at j = 3, where it meets norm_from_x / sumsq: a bf16 output would hide the 1/rms error
        opts = dict(bias=j % 2 == 0, out_fp32=epi_ == EPI_PLAIN and j in (0, 2, 3, 4), rstd=j % 3 == 0,
                    act_gelu=j % 2 == 1, theta=0.0 if j % 2 else 10000.0, heads=QKV_HEADS[j % 2],
                    norm_from_x=qm_ == 0 and epi_ in (EPI_PLAIN, EPI_RESIDUAL) and j % 2 == 1,
                    sumsq=qm_ == 2 and epi_ in (EPI_PLAIN, EPI_RESIDUAL) and j % 2 == 1, out2=j % 2 == 1)
        n_out = 128 if epi_ != EPI_GLU else 256
        cases.append((qm_, epi_, bn_, m, nkb * BKE[qm_], n_out, stages, splitk, opts))
    base = dict(bias=True, out_fp32=False, rstd=False, act_gelu=False, theta=0.0, heads=QKV_HEADS[0],
                norm_from_x=False, sumsq=False, out2=True)
    extra = [
        (0, EPI_PLAIN, 16, 15, 4096, 4096, 0, 8, {}),                          # ncol 2, Llama width
        (0, EPI_RESIDUAL, 16, 1, 14336, 4096, 0, 4, {}),                       # ncol 4, down-proj K
        (0, EPI_PLAIN, 32, 33, 14336, 128, 0, 8, dict(rstd=True)),             # ncol 4, rank slices past m_tok
        (0, EPI_GLU, 16, 16, 4096, 1024, 2, 8, dict(act_gelu=False)),
        (1, EPI_PLAIN, 64, 64, 14336, 512, 3, 8, {}),
        (1, EPI_RESIDUAL, 128, 129, 4096, 256, 0, 2, {}),
        (2, EPI_PLAIN, 256, 259, 4096, 256, 2, 2, {}),
        (2, EPI_RESIDUAL, 32, 17, 14336, 4096, 0, 8, {}),
        (2, EPI_PLAIN, 256, 200, 1152, 128, 0, 1, {}),                         # token columns 127 / 128 of a 256 tile
        (0, EPI_QKV_ROPE, 16, 9, 2048, 768, 0, 8, dict(theta=500000.0, heads=QKV_HEADS[1])),
    ]
    for qm_, epi_, bn_, m, k, n_out, stages, splitk, o in extra:
        cases.append((qm_, epi_, bn_, m, k, n_out, stages, splitk, {**base, **o}))
    return cases


CASES = _case_list()


def _case_id(c):
    qm, epi, bn, m, k, n_out, stages, splitk, o = c
    return f"q{qm}-{EPI_NAMES[epi]}-bn{bn}-m{m}-k{k}-n{n_out}-st{stages}-sk{splitk}"


def test_case_list_covers_every_instantiation():
    """all 70 (BN, epilogue, QM) kernels run under exact probes; every epilogue at every BN for bf16; m_tok 1, BN - 1,
    BN, BN + 1 and 2 BN + 3, stages 2 / 3 / default, k-block counts below / at / above 2 stages + 1, 4096 and 14336,
    split-K 1..8 with ncol 2 and 4 for every BN"""
    assert len(INSTANTIATIONS) == 70
    seen = {(c[2], c[1], c[0]) for c in CASES}
    assert seen == set(INSTANTIATIONS)
    for bn in BNS:
        mine = [c for c in CASES if c[2] == bn]
        assert {c[3] for c in mine} >= {1, bn - 1, bn, bn + 1, 2 * bn + 3}
        assert {c[6] for c in mine} == {2, 3, 0}
        assert {c[7] for c in mine} == {1, 2, 4, 8}
        rel = set()
        for c in mine:
            st = c[6] or DEFAULT_STAGES[bn]
            nkb = c[4] // BKE[c[0]]
            rel.add((nkb > 2 * st + 1) - (nkb < 2 * st + 1))
        assert rel == {-1, 0, 1}
    assert {c[4] for c in CASES} >= {4096, 14336}
    assert {c[2] // c[7] for c in CASES} >= {2, 4}
    assert any(c[5] >= 4096 for c in CASES)
    # every option fires, on every QM / epilogue it applies to
    has = lambda qm, epi, **want: any(c[0] == qm and c[1] == epi and all(c[8][k] == v for k, v in want.items())  # noqa: E731
                                      for c in CASES)
    for qm in (0, 1, 2):
        assert has(qm, EPI_PLAIN, out_fp32=True) and has(qm, EPI_PLAIN, out_fp32=False)
        assert has(qm, EPI_GLU, act_gelu=False) and has(qm, EPI_GLU, act_gelu=True)
        assert has(qm, EPI_QKV_ROPE, theta=0.0) and has(qm, EPI_QKV_ROPE, theta=10000.0)
        assert has(qm, EPI_RESIDUAL, out2=True) and has(qm, EPI_RESIDUAL, out2=False)
        for epi in EPI_NAMES:
            assert has(qm, epi, bias=True) and has(qm, epi, bias=False)
    for epi in (EPI_PLAIN, EPI_RESIDUAL):
        assert has(0, epi, norm_from_x=True) and has(2, epi, sumsq=True)
        assert has(2, epi, rstd=True) and has(0, epi, rstd=True)
    assert has(2, EPI_PLAIN, sumsq=True, rstd=True) or has(2, EPI_RESIDUAL, sumsq=True, rstd=True)
    assert has(0, EPI_PLAIN, norm_from_x=True, out_fp32=True) and has(2, EPI_PLAIN, sumsq=True, out_fp32=True)


def test_probe_positions_cover_every_target():
    """for every case of the sweep: every (token, k-block) holds a nonzero x -- so the first and last k-block of every
    split-K rank's share are hit for every token column --, every token hits all 8 swizzle chunks (all 4 MMA k-steps,
    all 4 MX scale blocks), tiles of >= 8 tokens hit every (token row % 8, chunk) pair, and the probe weights have no
    zero, so every weight row (63 / 64, 127 / 128 included) meets every nonzero x"""
    for qm, epi, bn, m, k, n_out, stages, splitk, o in CASES:
        g = torch.Generator().manual_seed(m + k)
        x, _, _ = probe_x(qm, m, k, g)
        bke = BKE[qm]
        nkb = k // bke
        nz = (x != 0).view(m, nkb, bke)
        assert nz.any(-1).all(), (qm, m, k)
        for r in range(splitk):
            lo, hi = nkb * r // splitk, nkb * (r + 1) // splitk
            assert nz[:, lo].any(-1).all() and nz[:, hi - 1].any(-1).all()
        chunk = nz.view(m, nkb, 8, bke // 8).any(-1).any(1)                     # [m, 8]: token hits chunk
        assert chunk.all(), (qm, m, k)
        for t0 in range(0, m, bn):
            rows = torch.arange(t0, min(m, t0 + bn))
            if rows.numel() >= 8:
                pairs = torch.zeros(8, 8, dtype=torch.bool)
                for t in rows.tolist():
                    pairs[t % 8] |= chunk[t]
                assert pairs.all()
    for qm in (0, 1, 2):
        op = Operands(qm, 3, 1024, 256, 32, qm, "cpu")
        assert (op.w.float() != 0).all()


# --------------------------------------------------------------------------- GPU: running a case
def _sentinel(shape, fp32=False, device="cuda"):
    if fp32:
        return torch.full(shape, SENT32, dtype=torch.int32, device=device).view(torch.float32)
    return torch.full(shape, SENT16, dtype=torch.int16, device=device).view(torch.bfloat16)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


class Run:
    """the buffers of one GEMM call: outputs behind ``ld_out`` > width, residual behind ``ld_res`` > n_out, q / KV
    buffers with sentinel rows, all prefilled"""

    def __init__(self, op, epi, bn, stages, splitk, opts, seed):
        dev = op.device
        self.op, self.epi, self.bn, self.stages, self.splitk, self.o = op, epi, bn, stages, splitk, opts
        g = torch.Generator(device=dev).manual_seed(seed)
        m, n = op.m, op.n_out
        self.width = n // 2 if epi == EPI_GLU else n
        self.ld = self.width + 40
        self.bias = (torch.randint(-128, 129, (n,), generator=g, device=dev).float() / 4) if opts.get("bias") else None
        self.residual = None
        if epi == EPI_RESIDUAL:
            rbuf = torch.randint(-255, 256, (m, n + 72), generator=g, device=dev).float() / 4
            self.rbuf = rbuf.to(torch.bfloat16)
            self.residual = self.rbuf[:, :n]
        if epi == EPI_QKV_ROPE:
            hd, nq, nkv = opts["heads"]
            self.qkv = dict(n_q=nq, n_kv=nkv, hd=hd, theta=opts["theta"], q_scale=0.5,
                            positions=torch.tensor([POSITIONS[(t * 3 + seed) % len(POSITIONS)] for t in range(m)],
                                                   dtype=torch.int32, device=dev))
            self.n_slots = m + 9
            perm = torch.randperm(self.n_slots, generator=g, device=dev)[:m].int()
            perm[torch.arange(m, device=dev) % 5 == 2] = -1
            self.slots = perm
        self.fp32 = bool(opts.get("out_fp32"))

    def fresh(self):
        op, m = self.op, self.op.m
        if self.epi == EPI_QKV_ROPE:
            # each buffer starts with a guard row: the kernel gets the view from row 1, so a store to token / slot -1
            # lands in the guard row instead of unrelated memory
            hd, nq, nkv = self.o["heads"]
            return dict(q=_sentinel((1 + m + 2, nq * hd)), k=_sentinel((1 + self.n_slots, nkv * hd)),
                        v=_sentinel((1 + self.n_slots, nkv * hd)))
        bufs = dict(out=_sentinel((m + 2, self.ld), self.fp32))
        if self.epi == EPI_RESIDUAL and self.o.get("out2"):
            bufs["out2"] = _sentinel((m + 2, self.ld))
        return bufs

    def launch(self, bufs, **extra):
        ops = _ops()
        op = self.op
        kw = dict(epi=self.epi, bn=self.bn, splitk=self.splitk, stages=self.stages, bias=self.bias, eps=EPS,
                  rstd=op.rstd, w_scale=op.w_scale, sfa=op.sfa, sfb=op.sfb, sumsq=op.sumsq,
                  norm_from_x=bool(self.o.get("norm_from_x")), act_gelu=bool(self.o.get("act_gelu")))
        if self.epi == EPI_QKV_ROPE:
            q = self.qkv
            kw.update(q_out=bufs["q"][1:], k_cache=bufs["k"][1:], v_cache=bufs["v"][1:], positions=q["positions"],
                      slots=self.slots,
                      n_q_heads=q["n_q"], n_kv_heads=q["n_kv"], head_dim=q["hd"], rope_theta=q["theta"],
                      q_scale=q["q_scale"])
        else:
            kw.update(out_ptr=bufs["out"].data_ptr(), ld_out=self.ld, out_fp32=self.fp32)
        if self.epi == EPI_RESIDUAL:
            kw["residual"] = self.residual
            if "out2" in bufs:
                kw["out2_ptr"] = bufs["out2"].data_ptr()
        kw.update(extra)
        ops.gemm(op.w, op.x, **kw)
        torch.cuda.synchronize()
        return bufs

    def ref(self, **mut):
        kw = dict(bias=self.bias, residual=self.residual, act_gelu=bool(self.o.get("act_gelu")),
                  norm_from_x=bool(self.o.get("norm_from_x")))
        if self.epi == EPI_QKV_ROPE:
            kw["qkv"] = self.qkv
        return gemm_ref64(self.op, self.epi, mut=mut, **kw)


def _check(tag, key, got, ref, res, epi, qm, *, exact, fp32=False, rs_approx=False, theta=0.0, part=None):
    """exact: bytes equal ref rounded to the output dtype; otherwise within the error model"""
    dt = torch.float32 if fp32 else torch.bfloat16
    if exact:
        want = ref.to(dt)
        bad = _bits(got) != _bits(want)
        if bad.any():
            t, n = bad.nonzero()[0].tolist()
            raise AssertionError(f"{tag}: {bad.sum().item()} outputs differ from the exact reference, first at token {t}, "
                                 f"column {n}: got {got[t, n].item()} want {want[t, n].item()}")
        MEASURED[key] = max(MEASURED[key], 0.0)
        return
    if part is not None:
        res = {k: (v[:, part] if torch.is_tensor(v) and v.dim() == 2 else v) for k, v in res.items()}
    base, b, units = bound(ref, res, epi, qm, fp32=fp32, exact_pre=not key[1].startswith("random"),
                           rs_approx=rs_approx, theta=theta)
    err = (got.double() - ref).abs()
    assert torch.isfinite(got.double()).all(), f"{tag}: non-finite output"
    ratio = _ratio(err, b)
    worst = ratio.max().item()
    MEASURED[key] = max(MEASURED[key], worst)
    excess = (err - base).clamp(min=0)
    for name, u in units.items():
        # the constant this output needs if the whole excess were charged to it
        c = torch.where(u > 0, excess / u, torch.where(excess > 0, torch.full_like(u, math.inf), torch.zeros_like(u)))
        C_MEASURED[name] = max(C_MEASURED[name], c.max().item())
    if worst > 1.0:
        idx = (ratio == ratio.max()).nonzero()[0].tolist()
        raise AssertionError(f"{tag}: |out - ref| / bound = {worst:.3f} at {idx}: out {got[idx[0], idx[1]].item()} "
                             f"ref {ref[idx[0], idx[1]].item()} bound {b[idx[0], idx[1]].item():.3g}")


def check_run(run, bufs, tag):
    """every output against the reference, every byte outside the outputs still the sentinel"""
    op, epi, o = run.op, run.epi, run.o
    m = op.m
    rs_approx = bool(o.get("norm_from_x")) or op.sumsq is not None
    key = (op.qm, EPI_NAMES[epi])
    res = run.ref()
    if epi == EPI_QKV_ROPE:
        theta = run.qkv["theta"]
        exact = theta == 0 and not rs_approx
        q = bufs["q"]                                           # guard row, m token rows, 2 rows past m_tok
        assert (_bits(q[0]) == SENT16).all(), f"{tag}: q guard row in front of the buffer written"
        assert (_bits(q[1 + m:]) == SENT16).all(), f"{tag}: q rows past m_tok written"
        q_dim = q.shape[1]
        kv_dim = bufs["k"].shape[1]
        _check(tag + " q", key, q[1:1 + m], res["q"], res, epi, op.qm, exact=exact, rs_approx=rs_approx, theta=theta,
               part=slice(0, q_dim))
        for name, lo in (("k", q_dim), ("v", q_dim + kv_dim)):
            cache = bufs[name]                                  # guard row, then slot s at row s + 1
            want = place_cache(res[name], run.slots, run.n_slots)
            keep = want.isnan().all(-1)
            assert keep[0]
            assert (_bits(cache[keep]) == SENT16).all(), \
                f"{tag}: {name} cache guard row (slot -1) or a slot no token names was written"
            live = run.slots >= 0
            _check(f"{tag} {name}", key, cache[run.slots[live].long() + 1], res[name][live],
                   {k: (v[live] if torch.is_tensor(v) and v.dim() == 2 else v) for k, v in res.items()}, epi, op.qm,
                   exact=exact, rs_approx=rs_approx, theta=theta if name == "k" else 0.0,
                   part=slice(lo, lo + kv_dim))
        return
    for name in ("out", "out2"):
        if name not in bufs:
            continue
        buf = bufs[name]
        bits = _bits(buf)
        sent = SENT32 if run.fp32 and name == "out" else SENT16
        assert (bits[m:] == sent).all(), f"{tag}: {name} rows past m_tok written"
        assert (bits[:, run.width:] == sent).all(), f"{tag}: {name} columns past the width written"
        exact = epi in (EPI_PLAIN, EPI_RESIDUAL) and not rs_approx
        _check(f"{tag} {name}", key, buf[:m, :run.width], res["out"], res, epi, op.qm, exact=exact,
               fp32=run.fp32 and name == "out", rs_approx=rs_approx)


def _report():
    print("\nMEASURED " + "  ".join(f"q{k[0]}/{k[1]}={v:.3f}" for k, v in sorted(MEASURED.items())))
    print("MEASURED constants " + "  ".join(f"{k}={v:.3g}" for k, v in sorted(C_MEASURED.items())))


def _resolve(bn, epi, k, qm, stages, splitk):
    return tuple(_ops().native().gemm_resolve(bn, epi, k, qm, stages, splitk))


def run_twice(run, tag, **extra):
    a = run.launch(run.fresh(), **extra)
    b = run.launch(run.fresh(), **extra)
    for name in a:
        assert torch.equal(_bits(a[name]), _bits(b[name])), f"{tag}: two identical calls differ in {name}"
    return a


@gpu
@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_exact_probes_match_ref64(case):
    """one instantiation under exact probes: the (stages, split-K) the case names is what runs, outputs equal the fp64
    reference (bit for bit where the epilogue is exact), poison and sentinels untouched, identical bytes twice"""
    qm, epi, bn, m, k, n_out, stages, splitk, o = case
    if epi == EPI_QKV_ROPE:
        hd, nq, nkv = o["heads"]
        n_out = (nq + 2 * nkv) * hd
    st = stages or DEFAULT_STAGES[bn]
    assert _resolve(bn, epi, k, qm, stages, splitk) == (st, splitk)
    seed = zlib.crc32(_case_id(case).encode()) % 100003
    op = Operands(qm, m, k, n_out, bn, seed, "cuda", rstd=o["rstd"] or qm == 1, sumsq=o["sumsq"])
    run = Run(op, epi, bn, stages, splitk, o, seed + 1)
    tag = _case_id(case)
    check_run(run, run_twice(run, tag), tag)
    _report()


@gpu
def test_sweep_covers_every_allowed_splitk():
    """for every BN, ring depth and epilogue the split-K values the resolver keeps are exactly {1, 2, 4, 8}, all of which
    the sweep runs; 3 and 7 round down, > 8 clamps to 8, fewer k-blocks clamp; stages outside 2..default clamp"""
    for bn in BNS:
        for stages in (2, 3, 0):
            for epi in EPI_NAMES:
                keep = {s for s in range(1, 9) if _resolve(bn, epi, 14336, 0, stages, s)[1] == s}
                assert keep == {1, 2, 4, 8}, (bn, stages, epi, keep)
                assert {c[7] for c in CASES if c[2] == bn} >= keep
        assert _resolve(bn, 0, 14336, 0, 0, 3) == (DEFAULT_STAGES[bn], 2)
        assert _resolve(bn, 0, 14336, 0, 0, 7) == (DEFAULT_STAGES[bn], 4)
        assert _resolve(bn, 0, 14336, 0, 0, 99) == (DEFAULT_STAGES[bn], 8)
        assert _resolve(bn, 0, 14336, 0, 0, -1) == (DEFAULT_STAGES[bn], 1)
        assert _resolve(bn, 0, 3 * 64, 0, 0, 8) == (DEFAULT_STAGES[bn], 2)        # 3 k-blocks -> 3 -> 2
        assert _resolve(bn, 0, 3 * 128, 1, 0, 8) == (DEFAULT_STAGES[bn], 2)
        assert _resolve(bn, 0, 4096, 0, 1, 1) == (2, 1)
        assert _resolve(bn, 0, 4096, 0, 99, 1) == (DEFAULT_STAGES[bn], 1)
        assert _resolve(bn, 0, 4096, 0, -5, 1) == (DEFAULT_STAGES[bn], 1)
    with pytest.raises(RuntimeError):
        _resolve(48, 0, 4096, 0, 0, 1)
    with pytest.raises(RuntimeError):
        _resolve(16, 0, 4096, 2, 0, 1)


@gpu
@pytest.mark.parametrize("theta", [10000.0, 500000.0])
def test_rope_positions_match_ref64(theta):
    """QKV + RoPE at positions up to 131071 (Llama-3.1 context) on exact pre-activations: the error is the angle
    error of the fast-math inv_freq / __sincosf only"""
    o = dict(bias=True, theta=theta, heads=(128, 4, 2), rstd=False, out2=False)
    for qm, bn, splitk in ((0, 16, 4), (1, 32, 2), (2, 64, 1)):
        op = Operands(qm, 24, 1024, 1024, bn, int(theta) + qm, "cuda", rstd=qm == 1)
        run = Run(op, EPI_QKV_ROPE, bn, 0, splitk, o, qm)
        run.qkv["positions"] = torch.tensor([POSITIONS[t % 8] for t in range(24)], dtype=torch.int32, device="cuda")
        check_run(run, run_twice(run, f"rope q{qm}"), f"rope theta={theta} q{qm}")
    _report()


@gpu
@pytest.mark.parametrize("qm", [0, 1, 2])
@pytest.mark.parametrize("m,k,n_out,bn,splitk", [(16, 4096, 1024, 16, 4), (33, 14336, 512, 64, 2),
                                                 (300, 4096, 256, 128, 1)])
def test_random_llama_inputs_within_acc_bound(qm, m, k, n_out, bn, splitk):
    """Llama-magnitude random operands (quantised by the project's own quantisers for fp8 / MX, the reference reads the
    same quantised values), fp32 output: the error is the accumulation error C_ACC[QM] 2^-23 sum |x w| * scale"""
    if qm == 2 and bn == 16:
        bn = 32
    op = Operands(qm, m, k, n_out, bn, m + k + qm, "cuda", kind="random")
    o = dict(out_fp32=True)
    run = Run(op, EPI_PLAIN, bn, 0, splitk, o, 1)
    assert _resolve(bn, EPI_PLAIN, k, qm, 0, splitk)[1] == splitk
    bufs = run_twice(run, "random")
    res = run.ref()
    out = bufs["out"][:m, :n_out]
    assert (_bits(bufs["out"][:, n_out:]) == SENT32).all()
    _check(f"random q{qm} m{m} k{k}", (qm, "random"), out, res["out"], res, EPI_PLAIN, qm, exact=False, fp32=True)
    _report()


@gpu
def test_norm_from_x_wins_over_rstd():
    """with both ``norm_from_x`` and ``rstd`` the kernel scales by the 1/rms of the raw rows and ignores ``rstd``"""
    op = Operands(0, 20, 2048, 256, 32, 77, "cuda")
    o = dict(norm_from_x=True, bias=True)
    run = Run(op, EPI_PLAIN, 32, 0, 2, o, 5)
    both = run.launch(run.fresh(), rstd=torch.full((20,), 4.0, device="cuda"))
    alone = run.launch(run.fresh())
    assert torch.equal(_bits(both["out"]), _bits(alone["out"]))
    check_run(run, both, "norm_from_x + rstd")
    _report()


@gpu
def test_handoff_release_counters():
    """several token tiles x split-K: after each call signal_epoch and bump_epoch advance by one, signal_flag and
    ack_flag carry the new epochs, done_counter is back to 0, and the bytes match a call without the handoff"""
    op = Operands(0, 40, 1024, 384, 16, 91, "cuda")
    run = Run(op, EPI_RESIDUAL, 16, 0, 4, dict(bias=True, out2=True), 3)
    plain = run.launch(run.fresh())
    fl = torch.zeros(8, dtype=torch.int32, device="cuda")
    a = lambda i: fl.data_ptr() + 4 * i  # noqa: E731
    for call in (1, 2):
        got = run.launch(run.fresh(), signal_flag=a(0), signal_epoch=a(1), done_counter=a(2), bump_epoch=a(3),
                         ack_flag=a(4))
        assert fl[:5].tolist() == [call, call, 0, call, call], fl.tolist()
        for name in got:
            assert torch.equal(_bits(got[name]), _bits(plain[name]))
    check_run(run, plain, "handoff")


@gpu
@pytest.mark.parametrize("lag", [0, 1])
def test_satisfied_waits_match_no_flags(lag):
    """a head GEMM whose wait_flag is already published and a tail GEMM whose free_flag already acknowledges the
    payload (free_lag 0 and 1) give the bytes of a call without flags; norm_from_x makes the consumer warps wait too"""
    op = Operands(0, 20, 1024, 256, 32, 93, "cuda")
    run = Run(op, EPI_PLAIN, 32, 0, 2, dict(norm_from_x=True), 4)
    plain = run.launch(run.fresh())
    fl = torch.tensor([6, 5, 3, 3 - lag], dtype=torch.int32, device="cuda")   # wait_flag, wait_epoch, epoch, free_flag
    a = lambda i: fl.data_ptr() + 4 * i  # noqa: E731
    got = run.launch(run.fresh(), wait_flag=a(0), wait_epoch=a(1), signal_epoch=a(2), free_flag=a(3), free_lag=lag)
    assert torch.equal(_bits(got["out"]), _bits(plain["out"]))
    assert fl.tolist() == [6, 5, 3, 3 - lag]
    check_run(run, got, f"waits lag {lag}")


@gpu
@pytest.mark.parametrize("what", ["n_out", "k_bf16", "k_fp8", "mx_bn16", "mx_no_sfb", "qkv_width", "fp8_norm_from_x",
                                  "bn48"])
def test_refused_launches(what):
    """unsupported shapes and options raise before any launch and leave the output untouched"""
    ops = _ops()
    dev = "cuda"
    qm, n_out, k, bn = 0, 256, 512, 32
    if what == "n_out":
        n_out = 200
    elif what == "k_bf16":
        k = 96
    elif what == "k_fp8":
        qm, k = 1, 192
    elif what in ("mx_bn16", "mx_no_sfb"):
        qm, bn = 2, (16 if what == "mx_bn16" else 32)
    elif what == "fp8_norm_from_x":
        qm = 1
    elif what == "bn48":
        bn = 48
    dt = torch.bfloat16 if qm == 0 else torch.float8_e4m3fn
    w = torch.ones(n_out, k, device=dev).to(dt)
    x = torch.ones(4, k, device=dev).to(dt)
    out = _sentinel((4, n_out))
    kw = dict(bn=bn, splitk=1, out_ptr=out.data_ptr(), ld_out=n_out)
    if qm == 1:
        kw.update(w_scale=torch.ones(n_out, device=dev), rstd=torch.ones(4, device=dev))
    if qm == 2:
        kw["sfa"] = torch.full(((n_out // 128) * (k // 128) * 512,), 127, dtype=torch.uint8, device=dev)
        if what != "mx_no_sfb":
            kw["sfb"] = torch.full((k // 128 * 512,), 127, dtype=torch.uint8, device=dev)
    if what == "fp8_norm_from_x":
        kw["norm_from_x"] = True
    if what == "qkv_width":
        w = torch.ones(4 * 64, k, device=dev).to(dt)       # two q heads and one kv head of 64: kv width 64
        q = _sentinel((4, 128))
        kc = _sentinel((8, 64))
        kw = dict(bn=bn, splitk=1, epi=EPI_QKV_ROPE, q_out=q, k_cache=kc, v_cache=kc,
                  slots=torch.zeros(4, dtype=torch.int32, device=dev), n_q_heads=2, n_kv_heads=1, head_dim=64)
    with pytest.raises(RuntimeError):
        ops.gemm(w, x, **kw)
    torch.cuda.synchronize()
    assert (_bits(out) == SENT16).all()
