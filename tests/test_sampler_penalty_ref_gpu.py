"""Presence and frequency penalties in the fused sampler (``sample_kernel``) against a plain reference, at every cluster
size the launcher picks, with draws aimed at chosen tokens; the per-row count table the sampler keeps; and the engine
that carries both.

Semantics (vLLM / OpenAI): c[v] is how often id v has been generated for the row (an int16 table, saturating at 32767).
After soft-cap and the repetition penalty, and before temperature, every logit with c > 0 becomes
(l - f c) - p in fp32, round-to-nearest at each step (the kernel writes it with ``_rn`` intrinsics, so no FMA).  A row
reads its counts only when p or f is non-zero; greedy rows are penalised too.  The thread that publishes a token adds
one to its count.

Reference (``PenRef``, a ``RowRef`` with the penalty step inserted):
  * without soft-cap every step before temperature is IEEE-exact but the repetition penalty's division, which the
    kernel computes approximately (--use_fast_math).  The row is transformed in numpy float32 in the kernel's order, and
    the allowed set is RowRef's on that row (pen = 1, cap = 0); a seen token with l > 0 widens its error by the
    division's relative 2^-21 of |l / pen| (the subtraction can cancel, so RowRef's |l| 2^-21 does not cover it);
  * with soft-cap, tanh is approximate: the penalty step follows RowRef's fp64 soft-cap and penalty, and each token's
    error grows by the fp32 rounding of the product and the two subtractions (2^-24 of each operand and result);
  * rows with top-k or min-p use ``FiltRef`` of ``test_sampler_topk_ref_gpu`` on the float32-transformed row.

Probes put penalised tokens on the ids where the kernel hands over (CTA slices, warp chunks, the scalar tail): c = 0
beside c = 1 at equal logits, large and saturated counts, negative penalties, p only / f only / both, a repetition
penalty in the same row, greedy rows whose argmax the penalty moves, top-k / top-p / min-p on penalised rows, and a
soft-capped launch.  Every row also carries a few hundred counted ids in the bulk of the vocabulary."""
from __future__ import annotations

from collections import defaultdict

import numpy as np
import pytest
import torch

from test_sampler_ref_gpu import (AIM_AT, STEPS, VARIANTS, Launch, RowRef, aim_seed, cluster_cases, cta_edges,
                                  handover_ids, pack_bits, u01)
from test_sampler_topk_ref_gpu import FiltRef

gpu = pytest.mark.gpu

VOCABS = (32000, 128256, 151936)
REST, BAND = -10.0, 10.0
COUNT_MAX = 32767
SOFTCAP = 30.0
PVARIANTS = ("pf_spread", "pf_switch", "pf_large", "pf_neg", "pf_greedy", "pf_repen", "pf_repen_greedy", "pf_off",
             "pk_topk", "pk_minp", "pk_all")
CAP_VARIANTS = ("pc_sampled", "pc_greedy", "pc_topp")
PF_SETS = ((0.5, 0.0), (0.0, 0.5), (0.5, 0.5), (-0.5, -0.25))     # p only, f only, both, negative
MEASURED: dict = defaultdict(float)


# --------------------------------------------------------------------------- reference
def penalise32(raw, seen, counts, pen, pres, freq):
    """the kernel's logits before temperature without soft-cap, in numpy float32"""
    l = np.asarray(raw, np.float32).copy()
    if seen is not None and np.float32(pen) != 1.0:
        with np.errstate(invalid="ignore"):
            pl = np.where(l > 0, l / np.float32(pen), l * np.float32(pen)).astype(np.float32)
        l = np.where(seen, pl, l)
    if counts is not None and (pres != 0.0 or freq != 0.0):
        c = np.asarray(counts).astype(np.float32)
        with np.errstate(invalid="ignore"):
            pf = ((l - np.float32(freq) * c).astype(np.float32) - np.float32(pres)).astype(np.float32)
        l = np.where(np.asarray(counts) > 0, pf, l)
    return l.astype(np.float32)


class PenRef(RowRef):
    """Allowed tokens of one row with presence / frequency penalties (see the module docstring).  ``mutant``:
    "every_id" penalises c = 0 too; "after_temp" subtracts the penalties after temperature."""

    def __init__(self, raw, seen=None, counts=None, pres=0.0, freq=0.0, temp=0.0, top_p=1.0, pen=1.0, cap=0.0,
                 mutant=None):
        raw = np.asarray(raw, dtype=np.float32)
        V = raw.size
        temp, pen = float(np.float32(temp)), float(np.float32(pen))
        pres, freq = float(np.float32(pres)), float(np.float32(freq))
        self.raw = raw
        self.top_p = min(float(np.float32(top_p)), 1.0)
        s = np.zeros(V, bool) if seen is None or pen == 1.0 else np.asarray(seen, bool)
        on = counts is not None and (pres != 0.0 or freq != 0.0)
        c = np.asarray(counts, np.int64) if on else np.zeros(V, np.int64)
        hit = np.ones(V, bool) if mutant == "every_id" else c > 0
        self.seen_eff, self.counts = s, c
        self.greedy = not temp > 0
        scale = 1.0 if self.greedy else 1.0 / temp
        if cap > 0:
            l = cap * np.tanh(raw.astype(np.float64) / cap)
            with np.errstate(invalid="ignore"):
                l = np.where(s, np.where(l > 0, l / pen, l * pen), l)
            fc = freq * c
            l1 = l - fc
            l2 = l1 - pres
            pre_dl = np.where(hit, (np.abs(l) + np.abs(fc) + np.abs(l1) + np.abs(l2)) * 2.0 ** -24, 0.0)
            pre_dl = pre_dl + cap * 2.0 ** -10.5 * max(pen, 1.0)
            if mutant != "after_temp":
                l = np.where(hit, l2, l)
        else:
            cnt = np.where(hit, np.maximum(c, 1), 0) if mutant == "every_id" else c
            l32 = penalise32(raw, s, cnt if mutant != "after_temp" else None, pen, pres, freq)
            l = l32.astype(np.float64)
            with np.errstate(invalid="ignore"):
                pre_dl = np.where(s & (raw > 0) & np.isfinite(l), (np.abs(raw / pen) + np.abs(l)) * 2.0 ** -21, 0.0)
        l = l * scale
        if mutant == "after_temp":
            l = np.where(hit, l - freq * c - pres, l)
        fin = np.isfinite(l)
        dl = np.where(fin, np.abs(np.where(fin, l, 0.0)) * 2.0 ** -21 + pre_dl * scale, 0.0)
        self.l, self.dl = l, dl
        self.jmax = int(np.argmax(l))
        mx = l[self.jmax]
        if self.greedy:
            cand = np.nonzero(l + dl >= mx - dl[self.jmax])[0]
            # tokens with the same input, seen bit and count are computed bit for bit alike: only the lowest id
            key = ((raw.view(np.uint32).astype(np.uint64) << np.uint64(17)) | (np.minimum(c, COUNT_MAX).astype(np.uint64)
                                                                               << np.uint64(1)) | s.astype(np.uint64))
            _, first = np.unique(key[cand], return_index=True)
            self.g_allowed = np.sort(cand[first])
            return
        # from here on as RowRef
        x = np.where(fin, l - mx, -np.inf)
        e = np.exp(x)
        pos = e > 0
        eps = np.where(pos, dl + dl[self.jmax] + np.abs(np.where(pos, x, 0.0)) * 2.0 ** -22 + 2.0 ** -21, 0.0)
        Z = e.sum()
        need = self.top_p * Z
        eps_m = 2.0 * (eps * e).sum() + 2.0 * V * 2.0 ** -32
        ea = np.sort(e)
        suf = np.append(np.cumsum(ea[::-1])[::-1], 0.0)

        def gt(t):
            return suf[np.searchsorted(ea, t, side="right")]

        A = gt(e)
        tie = suf[np.searchsorted(ea, e, side="left")] - A
        a_plus = np.maximum(gt(e * (1.0 - 4.0 * eps)) - tie, 0.0)
        tiny = Z * 1e-12
        must = pos & ((a_plus < need - eps_m) | (a_plus <= tiny))
        cand = pos & (A <= need + eps_m)
        b = np.nonzero(cand)[0][np.argmin(e[cand])]
        may = (pos & (e >= e[b] * (1.0 - 2.0 ** -16 - 4.0 * eps[b]))) | must
        self.e, self.eps, self.must, self.may, self.pos = e, eps, must, may, pos
        self.kept = pos & ((A < need) | (A <= tiny))
        em, eM = e * must, e * may
        self.C_must, self.C_may = np.cumsum(em) - em, np.cumsum(eM) - eM
        self.T_must, self.T_may = em.sum(), eM.sum()
        self.eps_c = 2.0 ** -17 * self.T_may + 2.0 * (eps * eM).sum()


# --------------------------------------------------------------------------- probes
class PProbe:
    def __init__(self, name, raw, counts, *, pres, freq, temp=0.0, top_p=1.0, pen=1.0, seen=None, top_k=0,
                 min_p=0.0, aims=None, expect=None):
        self.name, self.raw, self.counts, self.pres, self.freq = name, raw, counts, pres, freq
        self.temp, self.top_p, self.pen, self.seen, self.top_k, self.min_p = temp, top_p, pen, seen, top_k, min_p
        self.aims, self.expect = aims, expect

    def ref(self, cap=0.0, mutant=None):
        if self.top_k or self.min_p:
            l = penalise32(self.raw, self.seen, self.counts, self.pen, self.pres, self.freq)
            return FiltRef(l, self.temp, self.top_p, self.top_k, self.min_p)
        return PenRef(self.raw, self.seen, self.counts, self.pres, self.freq, self.temp, self.top_p, self.pen, cap,
                      mutant=mutant)


def make_pprobe(name, V, cs, i, rng):
    H = handover_ids(V, cs)
    temp3 = (0.7, 1.0, 1.3)[i % 3]
    pres, freq = PF_SETS[i % len(PF_SETS)]

    def pick(k, pool=H):
        pool = np.asarray(pool)
        if k > len(pool):
            other = np.setdiff1d(np.arange(V), pool)
            return rng.permutation(np.concatenate([pool, rng.choice(other, k - len(pool), replace=False)]))
        return rng.choice(pool, k, replace=False)

    raw = (REST + 0.5 * rng.standard_normal(V)).astype(np.float32)
    counts = np.zeros(V, np.int32)
    bulk = rng.choice(V, 300, replace=False)               # a realistic history: a few hundred ids, mostly once
    counts[bulk] = rng.choice([1, 1, 1, 2, 3, 7], 300)
    tail = V % 4
    if tail:
        counts[V - tail:] = 2                              # the scalar tail of the last slice
    if name == "pf_spread":                                # penalised band tokens on hand-over ids
        band = pick(8)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, 8)
        counts[band] = rng.permutation([0, 1, 2, 3, 0, 5, 1, 0])
        return PProbe(name, raw, counts, pres=pres, freq=freq, temp=temp3, top_p=(1.0, 0.9)[(i // 4) % 2], aims=band)
    if name == "pf_switch":                                # equal logits, c = 0 against c = 1
        ab = pick(2, cta_edges(V, cs) if cs >= 2 else H)
        rest = pick(3, np.setdiff1d(H, ab))
        raw[ab] = BAND
        raw[rest] = BAND - np.array([0.2, 0.45, 0.7], np.float32)
        counts[ab] = (0, 1)
        counts[rest] = 0
        pres, freq = ((0.7, 0.0), (0.0, 0.7), (0.35, 0.35))[i % 3]
        return PProbe(name, raw, counts, pres=pres, freq=freq, temp=1.0, aims=np.concatenate([ab, rest]))
    if name == "pf_large":                                 # large and saturated counts
        band = pick(5)
        c = np.array([1000, 20000, COUNT_MAX, COUNT_MAX, 0])
        freq, pres = (1e-3, 2.5e-4)[i % 2], (0.0, 0.25)[(i // 2) % 2]
        raw[band] = (BAND + freq * c + (pres if i % 4 >= 2 else 0.0) * (c > 0)
                     - np.array([0.0, 0.3, 0.6, 0.9, 0.45])).astype(np.float32)
        counts[band] = c
        return PProbe(name, raw, counts, pres=pres, freq=freq, temp=temp3, aims=band)
    if name == "pf_neg":                                   # negative penalties favour the counted tokens
        band = pick(6)
        raw[band] = BAND - np.array([1.0, 1.0, 0.5, 0.6, 0.8, 1.6], np.float32)
        counts[band] = (2, 1, 0, 0, 0, 4)
        return PProbe(name, raw, counts, pres=-0.5, freq=-0.25, temp=temp3, top_p=(1.0, 0.95)[i % 2], aims=band)
    if name == "pf_greedy":                                # the penalty moves the argmax (or, negative, onto a token)
        a, b, c3 = pick(3, cta_edges(V, cs) if cs >= 2 else H)
        counts[[a, b, c3]] = 0
        if i % 3 < 2:
            raw[a], raw[b], raw[c3] = BAND, BAND - 1.0, BAND - 1.25
            counts[a] = 3
            pres, freq = ((0.0, 0.5), (1.1, 0.0))[i % 3]
            expect = b
        else:
            raw[a], raw[b], raw[c3] = BAND - 1.0, BAND, BAND - 0.1
            counts[a] = 2
            pres, freq = -0.6, -0.3
            expect = a
        return PProbe(name, raw, counts, pres=pres, freq=freq, expect=int(expect))
    if name in ("pf_repen", "pf_repen_greedy"):            # repetition penalty and counts on the same tokens
        band = pick(8)
        seen = rng.random(V) < 0.01
        seen[band] = np.arange(8) % 2 == 0
        counts[band] = (1, 0, 2, 1, 0, 3, 0, 1)
        pen = (1.15, 2.0)[i % 2]
        if name == "pf_repen":
            raw[band] = np.array([2.0, 1.2, 0.6, 0.2, -0.3, -0.8, -1.3, -2.0], np.float32)
            return PProbe(name, raw, counts, pres=0.3, freq=0.2, temp=1.0, top_p=(1.0, 0.9)[(i // 2) % 2], pen=pen,
                          seen=seen, aims=band)
        raw = (2.0 + 0.5 * rng.standard_normal(V)).astype(np.float32)
        raw[band] = np.array([10.0, 9.0, 9.5, 8.0, 7.0, 6.0, 5.0, 4.0], np.float32)
        return PProbe(name, raw, counts, pres=0.3, freq=0.2, pen=pen, seen=seen)
    if name == "pf_off":                                   # counts present, both penalties off
        band = pick(7)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, 7)
        counts[band] = 4
        return PProbe(name, raw, counts, pres=0.0, freq=0.0, temp=temp3, top_p=0.9, aims=band)
    if name in ("pk_topk", "pk_minp", "pk_all"):           # top-k / top-p / min-p on the penalised row
        band = pick(10)
        eb = np.exp(-0.25 * np.arange(10))
        raw[band] = (temp3 * np.log(eb) + BAND).astype(np.float32)
        counts[band] = 0
        counts[band[[0, 3]]] = (2, 1)                      # the penalty reorders the top of the band
        kw = {"pk_topk": dict(top_k=3), "pk_minp": dict(min_p=0.3),
              "pk_all": dict(top_k=6, top_p=0.8, min_p=0.1)}[name]
        return PProbe(name, raw, counts, pres=0.1, freq=0.2, temp=temp3, aims=band[:6], **kw)
    if name.startswith("pc_"):                             # soft-capped launch
        raw = rng.uniform(-60.0, 0.0, V).astype(np.float32)
        band = pick(5)
        raw[band] = np.array([60.0, 45.0, 38.0, 34.0, 31.0]) + rng.uniform(-0.5, 0.5, 5)
        counts[band] = (2, 0, 1, 0, 3)
        if name == "pc_greedy":
            return PProbe(name, raw, counts, pres=1.0, freq=0.5)
        return PProbe(name, raw, counts, pres=0.5, freq=0.5, temp=1.0, top_p=0.95 if name == "pc_topp" else 1.0,
                      aims=band)
    raise ValueError(name)


class PLaunch:
    """B probe rows for one ``sample`` call; per-sequence state (and the count table) at row_map[b] of n_state rows,
    junk in the state rows no logits row maps to.  ``off_rows``: rows whose penalties are zeroed."""

    def __init__(self, V, cs, B, variants, *, cap=0.0, rounds=len(STEPS), seed=0, offset=0, row_map=None,
                 n_state=None, off_rows=()):
        rng = np.random.default_rng(seed)
        self.V, self.cs, self.B, self.cap = V, cs, B, cap
        self.row_map = np.arange(B) if row_map is None else np.asarray(row_map)
        S = self.n_state = B if n_state is None else n_state
        self.probes = [make_pprobe(variants[(i + offset) % len(variants)], V, cs, i, rng) for i in range(B)]
        for b in off_rows:
            self.probes[b].pres, self.probes[b].freq = 0.0, 0.0
        self.refs = [p.ref(cap) if bb >= 0 else None for p, bb in zip(self.probes, self.row_map)]
        self.logits = np.stack([p.raw for p in self.probes])
        self.temp = rng.uniform(0.5, 2.0, S).astype(np.float32)
        self.top_p = rng.uniform(0.1, 1.0, S).astype(np.float32)
        self.pen = rng.uniform(1.0, 3.0, S).astype(np.float32)
        self.top_k = rng.integers(1, 100, S).astype(np.int32)
        self.min_p = rng.uniform(0.0, 1.0, S).astype(np.float32)
        self.pres = rng.uniform(-2.0, 2.0, S).astype(np.float32)
        self.freq = rng.uniform(-2.0, 2.0, S).astype(np.float32)
        self.cstride = (V + 7) // 8 * 8
        self.counts = rng.integers(0, 50, (S, self.cstride)).astype(np.int16)
        seen = rng.random((S, V)) < 0.3
        for p, bb in zip(self.probes, self.row_map):
            if bb >= 0:
                self.temp[bb], self.top_p[bb], self.pen[bb] = p.temp, p.top_p, p.pen
                self.top_k[bb], self.min_p[bb], self.pres[bb], self.freq[bb] = p.top_k, p.min_p, p.pres, p.freq
                self.counts[bb] = 0
                self.counts[bb, :V] = p.counts
                seen[bb] = False if p.seen is None else p.seen
        self.seen = pack_bits(seen)
        self.steps = STEPS[:rounds]
        self.seeds = rng.integers(0, 1 << 32, (rounds, S), dtype=np.uint64).astype(np.uint32)
        self.draws = []
        for t, step in enumerate(self.steps):
            row = []
            for b, (p, ref, bb) in enumerate(zip(self.probes, self.refs, self.row_map)):
                if bb < 0:
                    row.append(None)
                    continue
                aim = None
                if not ref.greedy and p.aims is not None:
                    aims = [int(k) for k in p.aims if ref.must[k] and np.subtract(*ref.window(k)) < 0]
                    if aims:
                        aim = aims[(t + b) % len(aims)]
                        s = aim_seed(*ref.window(aim), step, b, AIM_AT[(t + b) % len(AIM_AT)])
                        if s is None:
                            aim = None
                        else:
                            self.seeds[t, bb] = s
                u = u01(self.seeds[t, bb], step, b)
                row.append((u, ref.allowed(u), aim))
            self.draws.append(row)

    def check(self, t, out_state, tag):
        bad = []
        for b, (p, ref, d) in enumerate(zip(self.probes, self.refs, self.draws[t])):
            if d is None:
                continue
            u, allowed, aim = d
            tok = int(out_state[self.row_map[b]])
            if not 0 <= tok < self.V:
                bad.append(f"{tag} row {b} {p.name}: token {tok} out of range")
                continue
            r = ref.ratio(tok, u)
            MEASURED[p.name] = max(MEASURED[p.name], r)
            if p.expect is not None and tok != p.expect:
                bad.append(f"{tag} row {b} {p.name}: greedy expected {p.expect}, got {tok}")
            elif aim is not None and tok != aim:
                bad.append(f"{tag} row {b} {p.name}: aimed at {aim}, got {tok} (u={u:.7f}, err/bound {r:.3g})")
            elif tok not in allowed:
                bad.append(f"{tag} row {b} {p.name}: token {tok} not in {allowed[:8].tolist()} (err/bound {r:.3g})")
        return bad

    def counts_after(self, out_state):
        """the count table after one launch from ``self.counts``: +1 (saturating) at each mapped row's token"""
        exp = self.counts.astype(np.int32)
        for bb in self.row_map:
            if bb >= 0:
                tok = int(out_state[bb])
                exp[bb, tok] = min(exp[bb, tok] + 1, COUNT_MAX)
        return exp.astype(np.int16)


# --------------------------------------------------------------------------- CPU: the reference and the probes
def test_penref_without_penalties_is_rowref():
    """p = f = 0 (or no counts): PenRef's sets are RowRef's, with and without soft-cap and repetition penalty"""
    rng = np.random.default_rng(3)
    for i in range(12):
        V = (1000, 3001)[i % 2]
        raw = (rng.standard_normal(V) * (1.0, 3.0)[i % 2]).astype(np.float32)
        temp, top_p, cap = (0.7, 1.0, 1.5)[i % 3], (0.5, 0.9, 0.95)[i % 3], (0.0, 30.0)[(i // 2) % 2]
        seen = rng.random(V) < 0.1
        counts = rng.integers(0, 3, V)
        for kw in (dict(counts=counts), dict(counts=None, pres=0.5, freq=0.5)):
            a = PenRef(raw, seen, temp=temp, top_p=top_p, pen=1.3, cap=cap, **kw)
            b = RowRef(raw, seen, temp=temp, top_p=top_p, pen=1.3, cap=cap)
            assert np.array_equal(a.must, b.must) and np.array_equal(a.may, b.may), i
            if cap == 0.0:
                g = PenRef(raw, seen, temp=0.0, pen=1.3, **kw)
                assert g.g_allowed.tolist() == RowRef(raw, seen, temp=0.0, pen=1.3).g_allowed.tolist(), i


def test_penref_matches_sample_reference_where_unambiguous():
    """greedy PenRef picks torch_ref's token; where must == may every kept token of the penalised row is drawn by
    torch_ref.sample_reference and nothing else is"""
    from bee2bee_b200.models import torch_ref
    rng = np.random.default_rng(4)
    checked = 0
    for i in range(24):
        V = 400
        raw = (rng.standard_normal(V) * 2.0).astype(np.float32)
        counts = np.where(rng.random(V) < 0.3, rng.integers(1, 6, V), 0).astype(np.int32)
        pres, freq = PF_SETS[i % 4]
        temp, top_p = (0.7, 1.0, 1.3)[i % 3], (1.0, 0.9, 0.6)[i % 3]
        ct = torch.from_numpy(counts)[None]
        g = PenRef(raw, counts=counts, pres=pres, freq=freq)
        exp = torch_ref.sample_reference(torch.from_numpy(raw)[None], None, 0.0, 1.0, 1.0, counts=ct, presence=pres,
                                         frequency=freq)
        assert g.g_allowed.tolist() == [int(exp[0])], i
        ref = PenRef(raw, counts=counts, pres=pres, freq=freq, temp=temp, top_p=top_p)
        if (ref.must != ref.may).any():
            continue
        checked += 1
        drawn = set(torch_ref.sample_reference(torch.from_numpy(raw)[None].repeat(4000, 1), None, temp, top_p, 1.0,
                                               torch.Generator().manual_seed(i), counts=ct.repeat(4000, 1),
                                               presence=pres, frequency=freq).tolist())
        assert drawn <= set(np.nonzero(ref.must)[0].tolist()), i
        likely = ref.must & (ref.e > 0.01 * ref.T_must)
        assert set(np.nonzero(likely)[0].tolist()) <= drawn, i
    assert checked >= 12


def test_penalty_step_is_exact_in_float32():
    """(l - f c) - p in float32 differs from the fused form on some inputs: the reference pins the unfused one"""
    rng = np.random.default_rng(6)
    l = rng.uniform(-20, 20, 20000).astype(np.float32)
    f = np.float32(0.7)
    c = rng.integers(1, 1000, 20000)
    a = penalise32(l, None, c, 1.0, 0.3, 0.7)
    fused = (l.astype(np.float64) - np.float64(f) * c).astype(np.float32) - np.float32(0.3)
    assert (a != fused).any()
    assert np.array_equal(a, ((l - f * c.astype(np.float32)).astype(np.float32) - np.float32(0.3)).astype(np.float32))


@pytest.mark.parametrize("V,cs", [(32000, 1), (32000, 8), (128256, 4), (151936, 8)])
def test_aimed_draws_allow_exactly_one_token(V, cs):
    """every aimed draw allows exactly its token, every sampled probe kind gets aims, and every greedy row whose
    argmax the penalty moves allows exactly the expected token"""
    aimed = defaultdict(int)
    for variants, cap in ((PVARIANTS, 0.0), (CAP_VARIANTS, SOFTCAP)):
        L = PLaunch(V, cs, 2 * len(variants), variants, cap=cap, rounds=3, seed=V + cs)
        for t in range(3):
            for p, ref, d in zip(L.probes, L.refs, L.draws[t]):
                u, allowed, aim = d
                if aim is not None:
                    assert allowed.tolist() == [aim], (p.name, t, aim, allowed[:8])
                    aimed[p.name] += 1
                if p.expect is not None:
                    assert allowed.tolist() == [p.expect], (p.name, allowed[:8])
                    assert int(np.argmax(ref.l)) == p.expect
                    assert int(np.argmax(p.raw)) != p.expect or p.pres < 0
                assert ref.point(u) in allowed, (p.name, t)
    for name in PVARIANTS + CAP_VARIANTS:
        if "greedy" not in name:
            assert aimed[name] > 0, name


@pytest.mark.parametrize("mutant,names", [("every_id", ("pf_switch",)), ("after_temp", ("pf_spread", "pf_neg"))])
def test_probe_catches_reference_mutant(mutant, names):
    """penalising c = 0 as well, or subtracting the penalties after temperature, leaves the allowed set on a probe"""
    V, cs, B = 32000, 4, 9
    L = PLaunch(V, cs, B, names, rounds=len(STEPS), seed=11)
    hits = 0
    for t in range(len(L.steps)):
        for p, ref, d in zip(L.probes, L.refs, L.draws[t]):
            if ref.greedy:
                continue
            hits += p.ref(mutant=mutant).point(d[0]) not in d[1]
            assert ref.point(d[0]) in d[1], (p.name, t)
    assert hits > 0


# --------------------------------------------------------------------------- GPU
def _ops():
    from bee2bee_b200 import ops
    return ops


def _i32(a, dev="cuda"):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).astype(np.uint32).view(np.int32))).to(dev)


def _step(step):
    return _i32(np.array([step], np.uint64).astype(np.uint32))


def _state(L, dev="cuda"):
    f = {k: torch.from_numpy(getattr(L, k)).to(dev) for k in ("temp", "top_p", "pen", "top_k", "min_p", "pres", "freq")}
    return f


def _run(L, tag, row_map=False):
    """every round of L through ``sample`` from the launch's count table; checks tokens, the count table after each
    launch and identical bytes on a repeat of the first round"""
    ops, dev = _ops(), "cuda"
    logits = torch.from_numpy(L.logits).to(dev)
    st = _state(L)
    rm = torch.from_numpy(L.row_map.astype(np.int32)).to(dev)
    out = torch.empty(L.n_state, dtype=torch.int32, device=dev)
    bad, outs = [], []
    for t, step in enumerate(L.steps):
        reps = []
        for _ in range(2 if t == 0 else 1):
            counts = torch.from_numpy(L.counts).to(dev)
            out.fill_(-1)
            ops.sample(logits, out, seen=torch.from_numpy(L.seen).to(dev), temperature=st["temp"], top_p=st["top_p"],
                       rep_penalty=st["pen"], top_k=st["top_k"], min_p=st["min_p"], seeds=_i32(L.seeds[t]),
                       step=_step(step), softcap=L.cap, counts=counts, presence=st["pres"], frequency=st["freq"],
                       row_map=rm.data_ptr() if row_map else 0)
            reps.append((out.cpu().numpy().copy(), counts.cpu().numpy()))
        if len(reps) == 2:
            assert all(np.array_equal(a, b) for a, b in zip(reps[0], reps[1])), f"{tag}: two identical launches differ"
        got, counts_after = reps[0]
        bad += L.check(t, got, f"{tag} step {step:#x}")
        if not np.array_equal(counts_after, L.counts_after(got)):
            bad.append(f"{tag} step {step:#x}: the count table is not the old counts plus the drawn tokens")
        outs.append(got)
    return outs, bad


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_penalties_match_ref64_at_every_cluster_size(V):
    """every penalty probe at every cluster size V reaches, and a soft-capped launch at the largest"""
    bad = []
    cases = cluster_cases(V)
    for cs, B in sorted(cases.items()):
        L = PLaunch(V, cs, B, PVARIANTS, seed=V + cs, offset=(V // 13 + 3 * cs) % len(PVARIANTS))
        bad += _run(L, f"V={V} cs={cs} B={B}")[1]
    cs = max(cases)
    L = PLaunch(V, cs, cases[cs], CAP_VARIANTS, cap=SOFTCAP, rounds=4, seed=V + 100 + cs)
    bad += _run(L, f"V={V} cs={cs} softcap")[1]
    print("\nerr/bound per probe: " + "  ".join(f"{k}={v:.3f}" for k, v in sorted(MEASURED.items())))
    assert not bad, f"{len(bad)} failures:\n" + "\n".join(bad[:12])


@gpu
def test_row_map_mixes_penalised_and_plain_rows():
    """one launch through row_map with skipped rows, some rows with both penalties off and junk penalties and counts
    in the state rows no logits row maps to: those rows' counts are not touched"""
    V, B, S = 128256, 12, 17
    row_map = np.array([5, 0, 16, 2, -1, 7, 1, 12, 3, -1, 9, 14])
    cs = int(_ops().native().sample_cluster_size(B, V))
    L = PLaunch(V, cs, B, PVARIANTS, rounds=4, seed=21, row_map=row_map, n_state=S, off_rows=(1, 5, 8, 11))
    outs, bad = _run(L, "row_map", row_map=True)
    free = [r for r in range(S) if r not in set(int(x) for x in row_map if x >= 0)]
    assert all((o[free] == -1).all() for o in outs)
    assert not bad, "\n".join(bad[:12])


@gpu
def test_counts_track_emitted_tokens_over_launches():
    """repeated launches on one table: each row's counts are the histogram of the tokens it emitted (on top of its
    starting counts), increments saturate at 32767, and rows that row_map skips are not touched"""
    ops, dev = _ops(), "cuda"
    V, B, S = 32000, 6, 8
    rng = np.random.default_rng(9)
    row_map = np.array([3, -1, 0, 6, 1, 4], np.int32)
    counts0 = np.zeros((S, V), np.int16)
    counts0[7] = rng.integers(0, 9, V)                      # state rows nothing maps to keep their bytes
    counts0[2] = 5
    logits = (rng.standard_normal((B, V)) * 2).astype(np.float32)
    logits[2, 77] = 40.0                                    # row 2 -> state 0: greedy on id 77 whose count saturates
    counts0[0, 77] = COUNT_MAX - 3
    temp = np.full(S, 0.9, np.float32)
    temp[0] = 0.0
    pres = np.full(S, 0.4, np.float32)
    freq = np.full(S, 0.3, np.float32)
    pres[[0, 1]] = freq[[0, 1]] = 0.0                       # states 0 and 1 count without being penalised
    counts = torch.from_numpy(counts0).to(dev)
    out = torch.empty(S, dtype=torch.int32, device=dev)
    rm = _i32(row_map)
    args = dict(temperature=torch.from_numpy(temp).to(dev), top_p=torch.ones(S, device=dev),
                presence=torch.from_numpy(pres).to(dev), frequency=torch.from_numpy(freq).to(dev),
                row_map=rm.data_ptr())
    hist = np.zeros((S, V), np.int64)
    for step in range(40):
        out.fill_(-1)
        ops.sample(torch.from_numpy(logits).to(dev), out, counts=counts, seeds=_i32(np.arange(S) + 11),
                   step=_step(step), **args)
        got = out.cpu().numpy()
        for bb in row_map[row_map >= 0]:
            hist[bb, got[bb]] += 1
    exp = np.minimum(counts0.astype(np.int64) + hist, COUNT_MAX)
    assert np.array_equal(counts.cpu().numpy().astype(np.int64), exp)
    assert counts[0, 77].item() == COUNT_MAX and hist[0, 77] == 40
    assert all(hist[bb].sum() == 40 for bb in row_map[row_map >= 0])
    assert np.array_equal(counts.cpu().numpy()[[2, 5, 7]], counts0[[2, 5, 7]])


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_zero_penalties_change_nothing(V):
    """presence / frequency passed as zeros, with or without a count table, and a count table alone give the tokens
    of the launch without them, on the plain sampler probes, at every cluster size"""
    ops, dev = _ops(), "cuda"
    for cs, B in sorted(cluster_cases(V).items()):
        L = Launch(V, cs, B, VARIANTS, rounds=3, seed=V + 7 * cs)
        logits = torch.from_numpy(L.logits).to(dev)
        temp, top_p, pen = (torch.from_numpy(a).to(dev) for a in (L.temp, L.top_p, L.pen))
        z = torch.zeros(L.n_state, device=dev)
        c0 = torch.from_numpy(np.random.default_rng(V).integers(0, 9, (L.n_state, (V + 7) // 8 * 8))
                              .astype(np.int16)).to(dev)
        bad = []
        for t, step in enumerate(L.steps):
            res = []
            for kw in ({}, dict(counts=c0.clone(), presence=z, frequency=z), dict(presence=z, frequency=z),
                       dict(counts=c0.clone()), dict(presence=z + 1.5, frequency=z - 0.5)):
                out = torch.full((L.n_state,), -1, dtype=torch.int32, device=dev)
                ops.sample(logits, out, seen=torch.from_numpy(L.seen).to(dev), temperature=temp, top_p=top_p,
                           rep_penalty=pen, seeds=_i32(L.seeds[t]), step=_step(step), **kw)
                res.append(out.cpu().numpy())
            assert all(np.array_equal(res[0], r) for r in res[1:]), f"V={V} cs={cs} step {step:#x}"
            bad += L.check(t, res[0], f"V={V} cs={cs} step {step:#x}")
        assert not bad, "\n".join(bad[:12])


@gpu
def test_refused_penalty_tensors():
    """wrong dtype, device, length, width, stride or alignment is refused before any launch"""
    ops, dev = _ops(), "cuda"
    V, B = 1000, 4
    logits = torch.randn(B, V, device=dev)
    temp = torch.ones(B, device=dev)
    out = torch.full((B,), -5, dtype=torch.int32, device=dev)
    table = torch.zeros(B, 1008, dtype=torch.int16, device=dev)
    bad_calls = [dict(presence=torch.zeros(B, dtype=torch.int32, device=dev)), dict(presence=torch.zeros(B)),
                 dict(presence=torch.zeros(B + 1, device=dev)), dict(frequency=torch.zeros(B, dtype=torch.float64,
                                                                                           device=dev)),
                 dict(frequency=torch.zeros(B - 1, device=dev)), dict(frequency=torch.zeros(B, 1, device=dev)),
                 dict(counts=torch.zeros(B, 1008, dtype=torch.int32, device=dev)),
                 dict(counts=torch.zeros(B, 1008, dtype=torch.int16)),
                 dict(counts=torch.zeros(B + 1, 1008, dtype=torch.int16, device=dev)),
                 dict(counts=torch.zeros(B, 992, dtype=torch.int16, device=dev)),             # narrower than V
                 dict(counts=torch.zeros(B, 1004, dtype=torch.int16, device=dev)),            # stride % 8 != 0
                 dict(counts=table[:, 2:]),                                                   # 4-byte aligned rows
                 dict(counts=torch.zeros(1008, B, dtype=torch.int16, device=dev).t()),        # column-major
                 dict(counts=torch.zeros(B * 1008, dtype=torch.int16, device=dev))]
    for kw in bad_calls:
        with pytest.raises(RuntimeError):
            ops.sample(logits, out, temperature=temp, **kw)
    torch.cuda.synchronize()
    assert (out == -5).all()
    ops.sample(logits, out, temperature=temp, counts=table[:, 8:], presence=temp)      # 16-byte offset: accepted
    torch.cuda.synchronize()
    assert (out >= 0).all()


# --------------------------------------------------------------------------- GPU: the engine
def _runner(max_batch=4):
    from bee2bee_b200.engine.runner import GpuRunner
    from bee2bee_b200.models.config import resolve_config
    cfg = resolve_config("tiny-llama")
    torch.manual_seed(0)
    return cfg, GpuRunner(cfg, "", 0, 1, torch.device("cuda:0"), max_batch=max_batch, groups=1, max_seq_len=512,
                          max_prefill_tokens=128, seed=0, use_graphs=True)


def _seq(slot, prompt, **kw):
    from bee2bee_b200.engine.runner import SeqInit
    return SeqInit(slot=slot, prompt=prompt, pages=list(range(1 + 8 * slot, 9 + 8 * slot)), **kw)


@gpu
def test_runner_counts_are_histogram_of_generated_tokens():
    """after prefill and decode bursts, every slot's count row is the histogram of the tokens it generated (the prompt
    not included); re-admitting a slot zeroes its row"""
    cfg, runner = _runner()
    V = cfg.vocab_size
    try:
        assert runner.counts.shape == (4, (V + 7) // 8 * 8) and not runner.counts.any()     # zeroed after warm-up
        prompts = [[7, 7, 7, 3, 3, 9] * 4, [11, 12, 13], list(range(40, 100)), [5] * 9]
        seqs = [_seq(i, p, temperature=(0.9, 0.0, 0.8, 0.0)[i], presence_penalty=(0.5, 1.0, 0.0, -0.5)[i],
                     frequency_penalty=(0.5, 0.0, 0.0, 0.25)[i], seed=i) for i, p in enumerate(prompts)]
        runner.prefill(seqs)
        runner.decode(7)
        runner.decode(5)
        runner.sync()
        hist, hpos = runner.read_history()
        counts = runner.counts.cpu().numpy()
        for s in range(4):
            toks = hist[s, :int(hpos[s])].numpy()
            assert len(toks) == 13
            assert np.array_equal(counts[s, :V], np.bincount(toks, minlength=V)), s
            assert not counts[s, V:].any()
        runner.prefill([_seq(1, [21, 22, 23], temperature=0.0, presence_penalty=1.0)])
        runner.sync()
        first = int(runner.tokens[1])
        row = runner.counts[1].cpu().numpy()
        assert row[first] == 1 and row.sum() == 1
        assert np.array_equal(runner.counts.cpu().numpy()[[0, 2, 3]], counts[[0, 2, 3]])
    finally:
        runner.close()


@gpu
def test_engine_neighbour_penalty_leaves_request_unchanged():
    """two requests submitted together in two runs: A has penalties off in both, B has them on in one run only; A's
    tokens are the same in both runs"""
    from bee2bee_b200.engine.core import Engine, SamplingParams
    outs = []
    for b_pen in (dict(presence_penalty=1.5, frequency_penalty=1.0), {}):
        eng = Engine("tiny-llama", device="cuda:0", max_batch=4, max_seq_len=256, decode_burst=4)
        try:
            ra = eng.submit([1, 5, 9, 33, 2, 7], SamplingParams(max_new_tokens=16, temperature=0.8, ignore_eos=True,
                                                                seed=1))
            rb = eng.submit([4, 4, 19, 4, 4], SamplingParams(max_new_tokens=16, temperature=0.0, ignore_eos=True,
                                                             seed=2, **b_pen))
            while not (ra.done.is_set() and rb.done.is_set()):
                eng.step()
        finally:
            eng.close()
        assert ra.error is None and rb.error is None
        outs.append((list(ra.out_ids), list(rb.out_ids)))
    assert outs[0][0] == outs[1][0]
    assert outs[0][1] != outs[1][1]          # B's penalty acts (greedy, strong penalties on a repeating model)


def _unpack(bits, V):
    return np.unpackbits(bits.view(np.uint8), axis=-1, bitorder="little")[..., :V].astype(bool)


@gpu
def test_greedy_penalties_match_gpu_logits():
    """greedy decoding with penalties, one step at a time, against the GPU's own logits: each step's token is the
    argmax of that row's logits after the repetition penalty and the penalty step in float32 (ties and the division's
    rounding as PenRef allows); rows with penalties on and off"""
    cfg, runner = _runner()
    V = cfg.vocab_size
    assert cfg.final_softcap == 0
    moved = 0
    try:
        prompts = [list(range(5, 45)), [7, 3, 9], list(range(200, 264)), [9, 9, 9, 9]]
        pf = [(0.0, 0.0), (1.0, 0.6), (0.4, 1.2), (0.0, 0.0)]
        reps = [1.0, 1.0, 1.3, 1.3]
        runner.prefill([_seq(i, p, temperature=0.0, top_p=1.0, repetition_penalty=reps[i], presence_penalty=pf[i][0],
                             frequency_penalty=pf[i][1], seed=i) for i, p in enumerate(prompts)])
        runner.sync()
        bad = []
        for step in range(24):
            counts = runner.counts[:4, :V].cpu().numpy()
            seen = _unpack(runner.seen[:4].cpu().numpy(), V)
            runner.decode(1)
            runner.sync()
            logits = runner.piece.logits[:4, :V].float().cpu().numpy()
            toks = runner.tokens[:4].cpu().numpy()
            for b in range(4):
                ref = PenRef(logits[b], seen[b], counts[b], pf[b][0], pf[b][1], pen=reps[b])
                if reps[b] == 1.0:             # every step is exact in fp32: the argmax, ties to the lowest id
                    exact = int(np.argmax(penalise32(logits[b], None, counts[b], 1.0, *pf[b])))
                    if int(toks[b]) != exact:
                        bad.append(f"step {step} row {b}: token {int(toks[b])}, argmax {exact}")
                elif int(toks[b]) not in ref.g_allowed:
                    bad.append(f"step {step} row {b}: token {int(toks[b])} not in {ref.g_allowed[:4].tolist()}")
                if pf[b] != (0.0, 0.0):
                    plain = RowRef(logits[b], seen[b], pen=reps[b])
                    moved += int(toks[b]) not in plain.g_allowed
    finally:
        runner.close()
    assert not bad, "\n".join(bad[:12])
    assert moved > 0, "no step had a penalised argmax different from the unpenalised one"
