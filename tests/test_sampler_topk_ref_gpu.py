"""Top-k and min-p in the fused sampler (``sample_kernel``) against a plain fp64 reference, at every cluster size the
launcher picks, with draws aimed at chosen tokens.

Semantics (transformers' processor order after temperature), with e = exp(l - max):
  * top-k (k <= 0 or k >= V = off): K = the tokens whose e is at least the k-th largest e; ties at the k-th are kept;
  * top-p over K: need = min(top_p, 1) Z_K, Z_K the mass of K; the nucleus is the smallest highest-e prefix of K whose
    mass reaches need, whole tie groups (as in ``test_sampler_ref_gpu``);
  * min-p (<= 0 = off): keep e >= min(min_p, 1), i.e. p >= min_p p_max;
  * greedy rows (temperature <= 0) ignore both; the draw is the id-order inverse CDF of the kept set.

Reference (``FiltRef``): the allowed tokens of one row, under the error model of ``test_sampler_ref_gpu.RowRef`` (eps_e
per token, eps_m for histogram mass, eps_c for the draw's prefix sums) plus:
  * top-k is decided on the 22-bit key prefix of the k-th largest kernel e, so must_K = tokens that fewer than k others
    (their own tie group excepted) can exceed after an error of 4 eps_e, and may_K = tokens with
    e >= e_k (1 - 2^-16 - 4 eps_k); when e_k (1 - 2^-16) is below 2^-32 every token may be kept (all e < 2^-32 share
    key 0);
  * Z_K lies between the mass of must_K and of may_K (each +- eps_m), so top-p's need does too; top_p >= 1 with top-k
    keeps exactly K (need equals the kernel's Z_K);
  * min-p is decided on the full 28-bit key: must_M = e (1 - 4 eps_e) >= min_p (1 + 2^-22) or e = 1, may_M =
    e (1 + 4 eps_e) >= min(min_p, 1 - 2^-22) (1 - 2^-22) (e within 2^-24 of 1 shares the key of 1).
  must = must_K & must_P & must_M and may = may_K & may_P & may_M; the draw windows are RowRef's.

Probes put the k-th token, tie groups and min-p boundaries on the ids where the kernel hands over (CTA slices, warp
chunks), at V in {32000, 128256, 151936} and every cluster size those reach.  The CPU tests check the reference against
``torch_ref.sample_reference`` and transformers' warpers, that every aimed draw allows exactly one token, and that each
reference-level mutant (need from Z instead of Z_K, the tie group at the k-th cut to k tokens, k - 1 kept, min-p
relative to the sum instead of the max) leaves the allowed set on some probe."""
from __future__ import annotations

from collections import defaultdict

import numpy as np
import pytest
import torch

from test_sampler_ref_gpu import (AIM_AT, STEPS, VARIANTS, Launch, RowRef, aim_seed, cluster_cases, cta_edges,
                                  cta_slices, handover_ids, u01)

gpu = pytest.mark.gpu

VOCABS = (32000, 128256, 151936)
REST, BAND = -10.0, 10.0
KVARIANTS = ("k_edge", "k_ties", "k_one", "k_one_tie", "k_vm1", "k_v", "k_gtv", "k_many", "kp_inside", "kp_zk",
             "kp_all", "minp_edge", "minp_one", "mix_k", "mix_p", "mix_m", "greedy_kpm")
MEASURED: dict = defaultdict(float)


# --------------------------------------------------------------------------- fp64 reference
class FiltRef(RowRef):
    """Allowed tokens of one row with top-k, top-p and min-p (see the module docstring).  No penalty or soft-cap:
    those steps come before the filters and are covered by ``test_sampler_ref_gpu``."""

    def __init__(self, raw, temp=0.0, top_p=1.0, top_k=0, min_p=0.0):
        raw = np.asarray(raw, dtype=np.float32)
        V = raw.size
        self.raw = raw
        self.top_p = min(float(np.float32(top_p)), 1.0)
        self.top_k, self.min_p = int(top_k), float(np.float32(min_p))
        self.k_on = 0 < self.top_k < V
        temp = float(np.float32(temp))
        self.greedy = not temp > 0
        if self.greedy:
            g = RowRef(raw, temp=0.0)
            self.g_allowed, self.l, self.dl, self.jmax = g.g_allowed, g.l, g.dl, g.jmax
            return
        l = raw.astype(np.float64) / temp
        fin = np.isfinite(l)
        dl = np.where(fin, np.abs(np.where(fin, l, 0.0)), 0.0) * 2.0 ** -21
        self.l, self.dl = l, dl
        self.jmax = int(np.argmax(l))
        x = np.where(fin, l - l[self.jmax], -np.inf)
        e = np.exp(x)
        pos = e > 0
        eps = np.where(pos, dl + dl[self.jmax] + np.abs(np.where(pos, x, 0.0)) * 2.0 ** -22 + 2.0 ** -21, 0.0)
        Z = e.sum()
        eps_m = 2.0 * (eps * e).sum() + 2.0 * V * 2.0 ** -32
        tiny = Z * 1e-12
        ea = np.sort(e)
        suf = np.append(np.cumsum(ea[::-1])[::-1], 0.0)

        def gt(t):
            return suf[np.searchsorted(ea, t, side="right")]

        A = gt(e)
        tie = suf[np.searchsorted(ea, e, side="left")] - A
        n_tie = np.searchsorted(ea, e, side="right") - np.searchsorted(ea, e, side="left")
        self.e, self.eps, self.pos, self.A, self.Z, self.tiny = e, eps, pos, A, Z, tiny
        # ---- top-k
        if self.k_on:
            self.ek = ea[::-1][self.top_k - 1]
            n_over = V - np.searchsorted(ea, e * (1.0 - 4.0 * eps), side="right")
            must_k = pos & (n_over - n_tie < self.top_k)
            eps_k = eps[pos & (e >= self.ek * (1.0 - 2.0 ** -10))].max()
            low = self.ek * (1.0 - 2.0 ** -16 - 4.0 * eps_k)
            if low <= 2.0 ** -32 * (1.0 + 2.0 ** -10):
                low = 0.0
            may_k = (pos & (e >= low)) | must_k
        else:
            must_k = may_k = pos
        # ---- top-p over K
        if self.k_on and self.top_p >= 1.0:
            must_p = pos & ((e >= 2.0 ** -32 * (1.0 + 2.0 ** -10)) | (A <= tiny))
            may_p = pos
        else:
            zk_lo, zk_hi = ((e * must_k).sum() - eps_m, (e * may_k).sum() + eps_m) if self.k_on else (Z, Z)
            need_lo, need_hi = self.top_p * zk_lo, self.top_p * zk_hi
            a_plus = np.maximum(gt(e * (1.0 - 4.0 * eps)) - tie, 0.0)
            must_p = pos & ((a_plus < need_lo - eps_m) | (a_plus <= tiny))
            cand = pos & may_k & (A <= need_hi + eps_m)
            b = np.nonzero(cand)[0][np.argmin(e[cand])]
            may_p = (pos & (e >= e[b] * (1.0 - 2.0 ** -16 - 4.0 * eps[b]))) | must_p
        # ---- min-p
        if self.min_p > 0.0:
            mp = min(self.min_p, 1.0)
            must_m = pos & ((e * (1.0 - 4.0 * eps) >= mp * (1.0 + 2.0 ** -22)) | (e == 1.0))
            may_m = (pos & (e * (1.0 + 4.0 * eps) >= min(mp, 1.0 - 2.0 ** -22) * (1.0 - 2.0 ** -22))) | must_m
        else:
            must_m = may_m = pos
        must, may = must_k & must_p & must_m, may_k & may_p & may_m
        assert not (must & ~may).any()
        self.must, self.may = must, may
        self.kept = self.exact_kept()
        em, eM = e * must, e * may
        self.C_must, self.C_may = np.cumsum(em) - em, np.cumsum(eM) - eM
        self.T_must, self.T_may = em.sum(), eM.sum()
        self.eps_c = 2.0 ** -17 * self.T_may + 2.0 * (eps * eM).sum()

    def exact_kept(self, mutant=None):
        """the kept set of the exact rule, optionally under a reference-level mutant"""
        e, pos, A = self.e, self.pos, self.A
        K = pos.copy()
        if self.k_on:
            k = self.top_k
            if mutant == "ties_cut":                          # exactly k tokens: the k-th tie group cut by id
                order = np.lexsort((np.arange(e.size), -e))
                K = np.zeros_like(pos)
                K[order[:k]] = True
            elif mutant == "k_minus_1":
                K = pos & (e >= np.sort(e)[::-1][max(k - 1, 1) - 1])
            else:
                K = pos & (e >= self.ek)
        Zsel = self.Z if mutant == "need_from_Z" else (e * K).sum()
        P = K & ((A < self.top_p * Zsel) | (A <= self.tiny)) if self.top_p < 1.0 else K
        if self.min_p > 0.0:
            thr = min(self.min_p, 1.0) * ((e * P).sum() if mutant == "minp_sum" else 1.0)
            P = P & ((e >= thr) | (A <= self.tiny))
        return P

    def point(self, u, mutant=None):
        if self.greedy:
            return super().point(u, mutant)
        c = np.cumsum(self.e * self.exact_kept(mutant))
        return int(np.argmax(c > u * c[-1]))


# --------------------------------------------------------------------------- probes
class KProbe:
    def __init__(self, name, raw, *, temp, top_p=1.0, top_k=0, min_p=0.0, aims=None):
        self.name, self.raw, self.temp, self.top_p, self.top_k, self.min_p = name, raw, temp, top_p, top_k, min_p
        self.aims = aims


def _raw_of(e, temp):
    return (temp * np.log(np.asarray(e, np.float64)) + BAND).astype(np.float32)


def _e64(raw, temp):
    l = raw.astype(np.float64) / temp
    return np.exp(l - l.max())


def make_kprobe(name, V, cs, i, rng):
    H = handover_ids(V, cs)
    temp3 = (0.7, 1.0, 1.3)[i % 3]

    def pick(k, pool=H):
        pool = np.asarray(pool)
        if k > len(pool):
            other = np.setdiff1d(np.arange(V), pool)
            return rng.permutation(np.concatenate([pool, rng.choice(other, k - len(pool), replace=False)]))
        return rng.choice(pool, k, replace=False)

    def mid(raw, used, n=30, e=0.06, temp=1.0):
        """n tokens off the band with e about `e`: mass outside K"""
        ids = rng.choice(np.setdiff1d(np.arange(V), used), n, replace=False)
        raw[ids] = _raw_of(e * (1.0 + 0.05 * rng.random(n)), temp)

    raw = (REST + 0.5 * rng.standard_normal(V)).astype(np.float32)
    if name == "k_edge":                                   # the k-th token (and its neighbours) on hand-over ids
        m = 1 + i % 6
        band = pick(m + 3)
        raw[band] = _raw_of(np.exp(-0.35 * np.arange(m + 3)), temp3)
        return KProbe(name, raw, temp=temp3, top_k=m, top_p=(1.0, 0.999)[i % 2], aims=band[:m + 1])
    if name == "k_ties":                                   # a tie group at the k-th value over several CTAs
        ties = pick(5, cta_edges(V, cs) if cs >= 4 else H)
        rest = pick(4, np.setdiff1d(H, ties))
        raw[ties] = 10.0
        raw[rest[:2]] = (11.0, 10.5)
        raw[rest[2:]] = (9.5, 9.0)
        return KProbe(name, raw, temp=1.0, top_k=(3, 5, 7)[i % 3], aims=np.concatenate([ties, rest]))
    if name == "k_one":
        band = pick(6)
        raw[band] = _raw_of(np.exp(-0.3 * np.arange(6)), temp3)
        return KProbe(name, raw, temp=temp3, top_k=1, top_p=(1.0, 0.5)[i % 2], aims=band[:2])
    if name == "k_one_tie":                                # k = 1 keeps the whole argmax tie group
        ties = pick(3, cta_edges(V, cs) if cs >= 2 else H)
        other = pick(3, np.setdiff1d(H, ties))
        raw[ties] = 10.0
        raw[other] = (9.8, 9.5, 9.0)
        return KProbe(name, raw, temp=1.0, top_k=1, aims=np.concatenate([ties, other]))
    if name in ("k_vm1", "k_v", "k_gtv"):                  # k = V - 1 runs the top-k phases; k = V, V + 5 are off
        band = pick(7)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, 7)
        k = {"k_vm1": V - 1, "k_v": V, "k_gtv": V + 5}[name]
        return KProbe(name, raw, temp=temp3, top_k=k, top_p=(0.9, 0.6)[i % 2], aims=band)
    if name == "k_many":                                   # k beyond the tokens with non-negligible e
        band = pick(7)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, 7)
        if i % 2 == 0:
            raw[np.setdiff1d(np.arange(V), band)] = REST - 40.0      # e < 2^-32: all share key 0 with the k-th
            k = 20
        else:
            keep = rng.choice(np.setdiff1d(np.arange(V), band), 12, replace=False)
            mask = np.ones(V, bool)
            mask[band] = mask[keep] = False
            raw[mask] = -np.inf
            k = 15
        return KProbe(name, raw, temp=1.0, top_k=k, top_p=(1.0, 0.9)[(i // 2) % 2], aims=band)
    if name == "kp_inside":                                # the nucleus strictly inside K, crossing mid-gap over Z_K
        m = 1 + i % 4
        band = pick(8)
        raw[band] = _raw_of(np.exp(-0.35 * np.arange(8)), temp3)
        ee = _e64(raw, temp3)
        srt = np.sort(ee)[::-1]
        zk = srt[:6].sum()
        top_p = 0.5 * (srt[:m].sum() + srt[:m + 1].sum()) / zk
        return KProbe(name, raw, temp=temp3, top_k=6, top_p=top_p, aims=band[:m + 1])
    if name in ("kp_zk", "kp_all"):
        if name == "kp_zk":                                # need over Z keeps all of K, over Z_K only two tokens
            e_band = np.array([1.0, 0.75, 0.55])
        else:                                              # top-p keeps all of K
            e_band = np.array([1.0, 0.9, 0.8, 0.7, 0.6])
        band = pick(len(e_band))
        raw[band] = _raw_of(e_band, 1.0)
        mid(raw, band)
        zk = e_band.sum()
        top_p = 0.5 * (1.0 + 1.75) / zk if name == "kp_zk" else 0.95
        return KProbe(name, raw, temp=1.0, top_k=len(e_band), top_p=top_p, aims=band)
    if name == "minp_edge":                                # one token just above, one just below min_p
        mp = (0.2, 0.05, 0.3)[i % 3]
        band = pick(5)
        raw[band] = _raw_of([1.0, 0.5, mp * (1 + 2e-3), mp * (1 - 2e-3), 0.1 * mp], temp3)
        return KProbe(name, raw, temp=temp3, min_p=mp, aims=band[:4])
    if name == "minp_one":
        ties = pick(2, cta_edges(V, cs) if cs >= 2 else H)
        other = pick(3, np.setdiff1d(H, ties))
        raw[ties] = BAND
        raw[other] = _raw_of([0.999, 0.9, 0.5], 1.0)
        return KProbe(name, raw, temp=1.0, min_p=1.0, aims=np.concatenate([ties, other]))
    if name in ("mix_k", "mix_p", "mix_m"):                # all three filters; a different one binds
        band = pick(10)
        eb = np.exp(-0.25 * np.arange(10))
        raw[band] = _raw_of(eb, temp3)
        if name == "mix_k":
            k, top_p, mp = 3, 0.99, eb[5] * (1 - 1e-3)
        elif name == "mix_p":
            k, mp = 8, eb[6] * (1 - 1e-3)
            top_p = 0.5 * (eb[:2].sum() + eb[:3].sum()) / eb[:8].sum()
        else:
            k, mp = 8, eb[2] * (1 - 1e-3)
            top_p = 0.5 * (eb[:5].sum() + eb[:6].sum()) / eb[:8].sum()
        return KProbe(name, raw, temp=temp3, top_k=k, top_p=top_p, min_p=mp, aims=band[:5])
    if name == "greedy_kpm":                               # greedy ignores both filters
        raw = (2.0 + rng.standard_normal(V)).astype(np.float32)
        top = pick(2 if i % 2 else 1, cta_edges(V, cs) if cs >= 2 else H)
        raw[top] = 10.0
        return KProbe(name, raw, temp=0.0, top_k=3, top_p=0.5, min_p=0.5)
    raise ValueError(name)


class KLaunch:
    """B probe rows for one ``sample`` call and every row's reference; per-sequence state at row_map[b] of n_state
    rows.  ``off_rows``: rows whose top_k / min_p are zeroed (their reference follows)."""

    def __init__(self, V, cs, B, variants, *, rounds=len(STEPS), seed=0, offset=0, row_map=None, n_state=None,
                 off_rows=()):
        rng = np.random.default_rng(seed)
        self.V, self.cs, self.B = V, cs, B
        self.row_map = np.arange(B) if row_map is None else np.asarray(row_map)
        S = self.n_state = B if n_state is None else n_state
        self.probes = [make_kprobe(variants[(i + offset) % len(variants)], V, cs, i, rng) for i in range(B)]
        for b in off_rows:
            self.probes[b].top_k, self.probes[b].min_p = 0, 0.0
        self.refs = [FiltRef(p.raw, p.temp, p.top_p, p.top_k, p.min_p) if bb >= 0 else None
                     for p, bb in zip(self.probes, self.row_map)]
        self.logits = np.stack([p.raw for p in self.probes])
        self.temp = rng.uniform(0.5, 2.0, S).astype(np.float32)        # state rows no logits row maps to: junk
        self.top_p = rng.uniform(0.1, 1.0, S).astype(np.float32)
        self.top_k = rng.integers(1, 100, S).astype(np.int32)
        self.min_p = rng.uniform(0.0, 1.0, S).astype(np.float32)
        for p, bb in zip(self.probes, self.row_map):
            if bb >= 0:
                self.temp[bb], self.top_p[bb], self.min_p[bb] = p.temp, p.top_p, p.min_p
                self.top_k[bb] = min(p.top_k, 2 ** 31 - 1)
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
            if aim is not None and tok != aim:
                bad.append(f"{tag} row {b} {p.name}: aimed at {aim}, got {tok} (u={u:.7f}, err/bound {r:.3g})")
            elif tok not in allowed:
                bad.append(f"{tag} row {b} {p.name}: token {tok} not in {allowed[:8].tolist()} (err/bound {r:.3g})")
        return bad


# --------------------------------------------------------------------------- CPU: the reference
def test_filtref_without_filters_is_rowref():
    """top_k = 0, min_p = 0: the same must / may sets as the plain top-p reference"""
    rng = np.random.default_rng(3)
    for i in range(12):
        V = (1000, 3001)[i % 2]
        raw = (rng.standard_normal(V) * (1.0, 3.0)[i % 2]).astype(np.float32)
        temp, top_p = (0.7, 1.0, 1.5)[i % 3], (0.5, 0.9, 0.95)[i % 3]
        a, b = FiltRef(raw, temp, top_p), RowRef(raw, temp=temp, top_p=top_p)
        assert np.array_equal(a.must, b.must) and np.array_equal(a.may, b.may), i


def test_filtref_matches_sample_reference_where_unambiguous():
    """where must == may the kept set is what torch_ref.sample_reference can draw: every kept token gets a draw and
    nothing else does"""
    from bee2bee_b200.models import torch_ref
    rng = np.random.default_rng(4)
    checked = 0
    for i in range(24):
        V = 400
        raw = (rng.standard_normal(V) * 2.0).astype(np.float32)
        temp, top_p = (0.7, 1.0, 1.3)[i % 3], (1.0, 0.9, 0.6)[i % 3]
        top_k, min_p = (0, 5, 40, 1)[i % 4], (0.0, 0.02, 0.3)[(i // 4) % 3]
        ref = FiltRef(raw, temp, top_p, top_k, min_p)
        if (ref.must != ref.may).any():
            continue
        checked += 1
        lg = torch.from_numpy(raw)[None].repeat(4000, 1)
        g = torch.Generator().manual_seed(i)
        drawn = set(torch_ref.sample_reference(lg, None, temp, top_p, 1.0, g, top_k=top_k, min_p=min_p).tolist())
        assert drawn <= set(np.nonzero(ref.must)[0].tolist()), i
        likely = ref.must & (ref.e > 0.01 * ref.T_must)          # drawn about 40 times or more out of 4000
        assert set(np.nonzero(likely)[0].tolist()) <= drawn, i
    assert checked >= 16
    # defaults reproduce the call without the new arguments
    lg = torch.from_numpy((rng.standard_normal((3, 500)) * 2).astype(np.float32))
    a = torch_ref.sample_reference(lg, None, 0.8, 0.9, 1.0, torch.Generator().manual_seed(1))
    b = torch_ref.sample_reference(lg, None, 0.8, 0.9, 1.0, torch.Generator().manual_seed(1), top_k=0, min_p=0.0)
    assert torch.equal(a, b)


def test_filtref_matches_transformers_warpers():
    """the exact kept set is transformers' TopK -> TopP -> MinP chain on tie-free rows"""
    tr = pytest.importorskip("transformers")
    rng = np.random.default_rng(5)
    checked = 0
    for i in range(24):
        V = 700
        raw = (rng.standard_normal(V) * 2.5).astype(np.float32)
        temp, top_p = (0.7, 1.0, 1.3)[i % 3], (1.0, 0.9, 0.6, 0.95)[i % 4]
        top_k, min_p = (0, 7, 60)[i % 3], (0.0, 0.05, 0.2)[(i // 3) % 3]
        ref = FiltRef(raw, temp, top_p, top_k, min_p)
        if (ref.must != ref.may).any():
            continue
        checked += 1
        scores = torch.from_numpy(raw.astype(np.float64))[None] / temp
        if top_k > 0:
            scores = tr.TopKLogitsWarper(top_k)(None, scores)
        if top_p < 1.0:
            scores = tr.TopPLogitsWarper(top_p)(None, scores)
        if min_p > 0.0:
            scores = tr.MinPLogitsWarper(min_p)(None, scores)
        hf = torch.isfinite(scores[0]).numpy()
        assert np.array_equal(hf, ref.must), (i, np.nonzero(hf != ref.must))
        assert np.array_equal(ref.kept, ref.must), i
    assert checked >= 12


@pytest.mark.parametrize("V,cs", [(32000, 1), (32000, 8), (128256, 4), (151936, 8)])
def test_aimed_draws_allow_exactly_one_token(V, cs):
    """every aimed draw allows exactly its token, and every sampled probe kind gets aims"""
    L = KLaunch(V, cs, len(KVARIANTS), KVARIANTS, rounds=3, seed=V + cs)
    aimed = defaultdict(int)
    for t in range(3):
        for p, ref, d in zip(L.probes, L.refs, L.draws[t]):
            u, allowed, aim = d
            if aim is not None:
                assert allowed.tolist() == [aim], (p.name, t, aim, allowed[:8])
                aimed[p.name] += 1
            assert ref.point(u) in allowed, (p.name, t)
    for name in KVARIANTS:
        if name != "greedy_kpm":
            assert aimed[name] > 0, name


@pytest.mark.parametrize("mutant,names", [
    ("need_from_Z", ("kp_zk",)),
    ("ties_cut", ("k_ties", "k_one_tie")),
    ("k_minus_1", ("k_edge",)),
    ("minp_sum", ("minp_edge",)),
])
def test_probe_catches_reference_mutant(mutant, names):
    V, cs, B = 32000, 4, 9
    L = KLaunch(V, cs, B, names, rounds=len(STEPS), seed=11)
    hits = 0
    for t in range(len(L.steps)):
        for p, ref, d in zip(L.probes, L.refs, L.draws[t]):
            hits += ref.point(d[0], mutant) not in d[1]
            assert ref.point(d[0]) in d[1], (p.name, t)
    assert hits > 0


# --------------------------------------------------------------------------- GPU
def _ops():
    from bee2bee_b200 import ops
    return ops


def _i32(a, dev="cuda"):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).astype(np.uint32).view(np.int32))).to(dev)


def _run(L, tag, filters=True, row_map=None):
    """every round of L through ``sample``; returns the tokens per round and the failures"""
    ops = _ops()
    dev = "cuda"
    logits = torch.from_numpy(L.logits).to(dev)
    temp, top_p = torch.from_numpy(L.temp).to(dev), torch.from_numpy(L.top_p).to(dev)
    kw = {}
    if filters:
        kw = dict(top_k=torch.from_numpy(L.top_k).to(dev), min_p=torch.from_numpy(L.min_p).to(dev))
    rm = torch.from_numpy(L.row_map.astype(np.int32)).to(dev)
    out = torch.empty(L.n_state, dtype=torch.int32, device=dev)
    outs, bad = [], []
    for t, step in enumerate(L.steps):
        out.fill_(-1)
        ops.sample(logits, out, temperature=temp, top_p=top_p, seeds=_i32(L.seeds[t]),
                   step=_i32(np.array([step], np.uint64).astype(np.uint32)),
                   row_map=rm.data_ptr() if row_map else 0, **kw)
        got = out.cpu().numpy().copy()
        outs.append(got)
        if hasattr(L, "check"):
            bad += L.check(t, got, f"{tag} step {step:#x}")
    return outs, bad


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_filters_match_ref64_at_every_cluster_size(V):
    """every top-k / top-p / min-p probe at every cluster size V reaches; identical bytes on a repeat"""
    bad = []
    for cs, B in sorted(cluster_cases(V).items()):
        L = KLaunch(V, cs, B, KVARIANTS, seed=V + cs, offset=(V // 11 + 3 * cs) % len(KVARIANTS))
        a, fails = _run(L, f"V={V} cs={cs} B={B}")
        b, _ = _run(L, "repeat")
        bad += fails
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), f"V={V} cs={cs}: two identical launches differ"
    print("\nerr/bound per probe: " + "  ".join(f"{k}={v:.3f}" for k, v in sorted(MEASURED.items())))
    assert not bad, f"{len(bad)} failures:\n" + "\n".join(bad[:12])


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_zero_filters_change_nothing(V):
    """top_k and min_p passed as zeros give the tokens of the launch without them, on the plain sampler probes, at
    every cluster size"""
    for cs, B in sorted(cluster_cases(V).items()):
        L = Launch(V, cs, B, VARIANTS, rounds=3, seed=V + 7 * cs)
        L.top_k = np.zeros(L.n_state, np.int32)
        L.min_p = np.zeros(L.n_state, np.float32)
        ops, dev = _ops(), "cuda"
        logits = torch.from_numpy(L.logits).to(dev)
        temp, top_p, pen = (torch.from_numpy(a).to(dev) for a in (L.temp, L.top_p, L.pen))
        zk, zm = torch.zeros(L.n_state, dtype=torch.int32, device=dev), torch.zeros(L.n_state, device=dev)
        bad = []
        for t, step in enumerate(L.steps):
            res = []
            for kw in ({}, dict(top_k=zk, min_p=zm), dict(top_k=zk), dict(min_p=zm)):
                out = torch.full((L.n_state,), -1, dtype=torch.int32, device=dev)
                ops.sample(logits, out, seen=torch.from_numpy(L.seen).to(dev), temperature=temp, top_p=top_p,
                           rep_penalty=pen, seeds=_i32(L.seeds[t]),
                           step=_i32(np.array([step], np.uint64).astype(np.uint32)), **kw)
                res.append(out.cpu().numpy())
            assert all(np.array_equal(res[0], r) for r in res[1:]), f"V={V} cs={cs} step {step:#x}"
            bad += L.check(t, res[0], f"V={V} cs={cs} step {step:#x}")
        assert not bad, "\n".join(bad[:12])


@gpu
def test_row_map_mixes_off_and_on_rows():
    """one launch through row_map with skipped rows, some rows with both filters off and junk filters in the state
    rows no logits row maps to"""
    V, B, S = 128256, 12, 17
    row_map = np.array([5, 0, 16, 2, -1, 7, 1, 12, 3, -1, 9, 14])
    cs = int(_ops().native().sample_cluster_size(B, V))
    L = KLaunch(V, cs, B, KVARIANTS, rounds=4, seed=21, row_map=row_map, n_state=S, off_rows=(1, 5, 8, 11))
    outs, bad = _run(L, "row_map", row_map=True)
    free = [r for r in range(S) if r not in set(int(x) for x in row_map if x >= 0)]
    assert all((o[free] == -1).all() for o in outs)
    assert not bad, "\n".join(bad[:12])


@gpu
def test_refused_filter_tensors():
    """wrong dtype, device or length is refused before any launch"""
    ops, dev = _ops(), "cuda"
    V, B = 1000, 4
    logits = torch.randn(B, V, device=dev)
    temp = torch.ones(B, device=dev)
    out = torch.full((B,), -5, dtype=torch.int32, device=dev)
    bad_calls = [dict(top_k=torch.zeros(B, device=dev)), dict(top_k=torch.zeros(B, dtype=torch.int64, device=dev)),
                 dict(top_k=torch.zeros(B, dtype=torch.int32)), dict(top_k=torch.zeros(B - 1, dtype=torch.int32,
                                                                                     device=dev)),
                 dict(min_p=torch.zeros(B, dtype=torch.int32, device=dev)), dict(min_p=torch.zeros(B)),
                 dict(min_p=torch.zeros(B + 1, device=dev)), dict(min_p=torch.zeros(B, dtype=torch.float64, device=dev))]
    for kw in bad_calls:
        with pytest.raises(RuntimeError):
            ops.sample(logits, out, temperature=temp, **kw)
    torch.cuda.synchronize()
    assert (out == -5).all()


@gpu
def test_engine_top_k_beyond_int32_fails_no_request():
    """GpuRunner: a request with top_k = 2^31 admitted while another decodes; both finish (k >= V is off)"""
    from bee2bee_b200.engine.core import Engine, SamplingParams
    eng = Engine("tiny-llama", device="cuda:0", max_batch=4, max_seq_len=256, decode_burst=2)
    try:
        r1 = eng.submit([1, 5, 9, 33], SamplingParams(max_new_tokens=12, ignore_eos=True))
        eng.step()
        assert not r1.done.is_set()
        r2 = eng.submit([4, 4, 19], SamplingParams(max_new_tokens=12, ignore_eos=True, top_k=2 ** 31, seed=9))
        while not (r1.done.is_set() and r2.done.is_set()):
            eng.step()
    finally:
        eng.close()
    assert r1.error is None and r2.error is None
    assert len(r1.out_ids) == 12 and len(r2.out_ids) == 12


@gpu
@pytest.mark.parametrize("filt", [dict(top_k=1), dict(min_p=1.0)])
def test_engine_filters_reduce_to_greedy(filt):
    """GpuRunner at temperature 0.8 with top_k = 1 (or min_p = 1) produces the greedy sequence"""
    from bee2bee_b200.engine.core import Engine, SamplingParams
    prompts = [[1, 5, 9, 33, 2, 7, 8, 100], [4, 4, 19], [7, 3, 250, 11]]
    eng = Engine("tiny-llama", device="cuda:0", max_batch=4, max_seq_len=256, decode_burst=4)
    try:
        greedy = eng.generate(prompts, SamplingParams(max_new_tokens=12, temperature=0.0, ignore_eos=True))
        sampled = eng.generate(prompts, SamplingParams(max_new_tokens=12, temperature=0.8, ignore_eos=True, seed=3,
                                                       **filt))
        plain = eng.generate(prompts, SamplingParams(max_new_tokens=12, temperature=0.8, top_p=1.0, ignore_eos=True,
                                                     seed=3))
    finally:
        eng.close()
    assert sampled == greedy
    assert plain != greedy          # the filter, not the temperature, makes the sequence greedy
