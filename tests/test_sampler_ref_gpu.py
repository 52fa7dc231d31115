"""The fused sampler (``sample_kernel``) against a plain fp64 reference, at every cluster size the launcher picks, with
draws aimed at chosen tokens.

``launch_sample`` spreads one sequence over a cluster of cs = 1, 2, 4 or 8 CTAs (``sample_cluster_size``); CTA r owns
ids [r W, r W + W) with W = roundup128(ceil(V / cs)), and inside a CTA warp w owns a chunk of cw = roundup128(ceil(n / 32))
ids.  The sweep scans the batch size with the extension's own query so that every V runs at every cs it can reach on
the card at hand, and places its probe tokens on the ids where the kernel hands over: id 0 and V - 1, the first and last
id of every CTA slice and warp chunk, the 32-id steps of the draw loop, and the scalar tail of the last slice.

Reference (``RowRef``), one row at a time in fp64, following the kernel's stated semantics:
  * soft-cap, then repetition penalty (l > 0 ? l / pen : l * pen where the seen bit is set and pen != 1), then
    temperature; greedy when !(temp > 0): the argmax, ties to the lowest id;
  * otherwise e = exp(l - max), Z = sum e, need = min(top_p, 1) Z.  The nucleus is the smallest set of highest-e tokens
    whose mass reaches need, every token tied with the boundary token included, and at least the maximal tokens (so
    top_p = 0 is the argmax).  This is not HF's rule, which cuts a tie group by sort order: the kernel keeps or drops
    a whole radix bin, so tied tokens always share a fate;
  * the draw is the inverse CDF of the kept set in id order at u01 = (float(h >> 8) + 0.5f) / 2^24 (float32), with
    h = hash(seed ^ hash(step * 0x9E3779B9 + b)) in uint32 and b the LOGITS row (not the ``row_map`` state row).

The kernel is built with --use_fast_math and decides the kept set on a fixed-point radix histogram, so token-for-token
equality does not hold in general.  The reference therefore returns the set of tokens the kernel may return.  Error
model (per token j, in units where max e = 1):
  * eps_l: the transformed logit.  Approximate division / reciprocal and the fp32 products: |l| 2^-21; tanh.approx has
    an absolute error of 2^-10.99, so a soft-cap adds cap 2^-10.5 (times pen and 1 / temp).  Greedy allows the tokens
    within eps_l(j) + eps_l(argmax) of the max; of tokens with identical fp32 input (and seen bit) only the lowest id,
    since the kernel computes them bit for bit alike and its ties go to the lowest id.
  * eps_e: relative error of e: eps_l(j) + eps_l(argmax), the fp32 l - max and the __expf argument (|x| 2^-22), and
    ex2.approx (2^-21).
  * eps_m = 2 sum_j eps_e e_j + 2 V 2^-32: the histogram mass (the fx32 32.32 truncation loses < 2^-32 per token).
    must_keep = tokens whose mass possibly above them (every token with e > e_j (1 - 4 eps_e), its own tie group
    excepted) is < need - eps_m; may_keep = tokens with e >= e_b (1 - 2^-16 - 4 eps_e(b)), where e_b is the smallest e
    whose exact mass above is <= need + eps_m: the kept set is decided on a 22-bit key, exact up to one level-2 bin
    (a relative width of 2^-18 to 2^-17).
  * eps_c = 2^-17 T + 2 sum eps_e e over may_keep: the fp32 prefix sums of the draw (<= ~64 sequential terms per lane,
    then the shuffle, warp and cluster trees) and the error of every e.
  Token j in may_keep is allowed when [C_must(j), C_may(j) + e_j] meets [u T_must - eps_c, u T_may + eps_c], C_* the
  id-order prefix of e over the set and T_* its total.

Aimed draws: u01 is a pure function of (seed, step, b), so for a kept token k the test picks a seed whose u lies inside
the part of k's interval that no other token can reach (in its middle, or near one end so that a few percent of
misplaced mass moves the draw off k), and demands exactly k.  Seeds come from one table
of 2^20 candidates: seed = s ^ hash(step * 0x9E3779B9 + b) makes the draw hash(s).

Probe kinds: spread (K band tokens on hand-over ids), edge (top_p crosses mid-gap; one variant puts the crossing and
the next token in one level-1 bin), ties (sampled tie group at the nucleus boundary over several CTAs; greedy maxima in
several slices), penalty (seen tokens with positive and negative logits, pen 1.15 / 2.0 / 1.0, bits in the last partial
bitmap word), softcap (cap 30, logits +-60), flat (N(0, 1) x {1, 4}, membership only), limits (top_p 0, 1e-9, 1, 1.5;
temp 1e-3; -inf entries).  NaN or +inf inside the vocabulary is unspecified and not probed.

The CPU tests pin the reference against ``torch_ref``, check that every aimed draw allows exactly one token, and that
each reference-level mutant (one token too many, the crossing token dropped, ties to the higher id, a one-sided
penalty, the RNG keyed on the state row) leaves the allowed set on some draw of the probe meant to catch it."""
from __future__ import annotations

import functools
from collections import defaultdict

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

VOCABS = (1000, 32000, 50257, 128256, 151936, 256000)
REST, BAND = -10.0, 10.0            # logits of the bulk of the vocabulary and of the probe tokens
NO_SEED, PHI = 0x1234567, 0x9E3779B9
# the rounds of a launch: one step value each (the step product wraps near 2^31 and 2^32 - 1)
STEPS = (0, 1, 12345, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF, 2)
MAX_B = 160                         # batch sizes scanned for cluster sizes
# where in the window that only the aimed token can reach a draw is placed: near its ends a mutant that moves the
# kept total or a prefix by a few percent already lands on another token
AIM_AT = (0.5, 0.05, 0.95, 0.2, 0.8)

VARIANTS = ("spread1", "spread2", "spread7", "spread64", "spread300", "edge_wide", "edge_narrow", "ties_sampled",
            "ties_greedy", "pen_pos", "pen_neg", "pen_neg2", "pen_one", "pen_sampled", "flat", "lim_p0", "lim_p1e-9",
            "lim_p1", "lim_p1.5", "lim_t1e-3", "lim_ninf", "lim_one", "lim_one_greedy")
SOFTCAP_VARIANTS = ("cap_greedy", "cap_t1", "cap_t08_p1", "cap_seen", "cap_sat_greedy")
PLUMB_VARIANTS = ("edge_wide", "spread7", "ties_greedy", "edge_narrow", "pen_neg", "ties_sampled", "lim_one")
SOFTCAP = 30.0

# measured max(error / bound) per probe kind, the mean allowed-set size of the flat probes, and the cluster sizes run
MEASURED: dict = defaultdict(float)
FLAT_SIZES: list = []
CS_RUN: dict = defaultdict(set)


# --------------------------------------------------------------------------- RNG of the kernel
def hash_u32(x):
    x = np.atleast_1d(np.asarray(x, dtype=np.uint32)).copy()
    with np.errstate(over="ignore"):
        x ^= x >> np.uint32(16)
        x *= np.uint32(0x7FEB352D)
        x ^= x >> np.uint32(15)
        x *= np.uint32(0x846CA68B)
        x ^= x >> np.uint32(16)
    return x


def _inner(step, b):
    return hash_u32((int(step) * PHI + int(b)) & 0xFFFFFFFF)[0]


def _u_of_hash(h):
    """float32, as the kernel: (float(h >> 8) + 0.5f) * 2^-24 (the + 0.5 rounds for h >> 8 >= 2^23)"""
    return ((h >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)


def u01(seed, step, b):
    return float(_u_of_hash(hash_u32(np.uint32(seed) ^ _inner(step, b)))[0])


@functools.lru_cache(maxsize=None)
def _seed_table():
    s = np.arange(1 << 20, dtype=np.uint32)
    u = _u_of_hash(hash_u32(s)).astype(np.float64)
    order = np.argsort(u, kind="stable")
    return u[order], s[order]


def aim_seed(u_lo, u_hi, step, b, frac=0.5):
    """a seed whose draw for (step, b) lies strictly inside (u_lo, u_hi), as close to u_lo + frac (u_hi - u_lo) as the
    table allows"""
    us, ss = _seed_table()
    goal = u_lo + frac * (u_hi - u_lo)
    i = int(np.clip(np.searchsorted(us, goal), 1, us.size - 1))
    i = i if abs(us[i] - goal) < abs(us[i - 1] - goal) else i - 1
    if not u_lo < us[i] < u_hi:
        return None
    return int(ss[i] ^ _inner(step, b))


# --------------------------------------------------------------------------- fp64 reference
class RowRef:
    """The allowed tokens of one logits row (see the module docstring).  ``one_sided_penalty`` is a mutant."""

    def __init__(self, raw, seen=None, temp=0.0, top_p=1.0, pen=1.0, cap=0.0, one_sided_penalty=False):
        raw = np.asarray(raw, dtype=np.float32)
        V = raw.size
        temp, pen = float(np.float32(temp)), float(np.float32(pen))
        self.raw = raw
        self.top_p = min(float(np.float32(top_p)), 1.0)
        l = raw.astype(np.float64)
        if cap > 0:
            l = cap * np.tanh(l / cap)
        s = np.zeros(V, bool) if seen is None or pen == 1.0 else np.asarray(seen, bool)
        self.seen_eff = s
        with np.errstate(invalid="ignore"):
            pl = l / pen if one_sided_penalty else np.where(l > 0, l / pen, l * pen)
        l = np.where(s, pl, l)
        self.greedy = not temp > 0
        scale = 1.0 if self.greedy else 1.0 / temp
        l = l * scale
        fin = np.isfinite(l)
        dl = np.where(fin, np.abs(np.where(fin, l, 0.0)), 0.0) * 2.0 ** -21
        if cap > 0:
            dl = dl + np.where(fin, cap * 2.0 ** -10.5 * max(pen, 1.0) * scale, 0.0)
        self.l, self.dl = l, dl
        self.jmax = int(np.argmax(l))
        mx = l[self.jmax]
        if self.greedy:
            cand = np.nonzero(l + dl >= mx - dl[self.jmax])[0]
            key = (raw.view(np.uint32).astype(np.uint64) << np.uint64(1)) | s.astype(np.uint64)
            _, first = np.unique(key[cand], return_index=True)
            self.g_allowed = np.sort(cand[first])
            return
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

        A = gt(e)                                             # exact mass strictly above
        tie = suf[np.searchsorted(ea, e, side="left")] - A    # the token's own tie group
        a_plus = np.maximum(gt(e * (1.0 - 4.0 * eps)) - tie, 0.0)
        tiny = Z * 1e-12
        must = pos & ((a_plus < need - eps_m) | (a_plus <= tiny))
        cand = pos & (A <= need + eps_m)
        b = np.nonzero(cand)[0][np.argmin(e[cand])]
        may = (pos & (e >= e[b] * (1.0 - 2.0 ** -16 - 4.0 * eps[b]))) | must
        self.e, self.eps, self.must, self.may, self.pos = e, eps, must, may, pos
        self.kept = pos & ((A < need) | (A <= tiny))          # the exact rule (mutants and measurement)
        em, eM = e * must, e * may
        self.C_must, self.C_may = np.cumsum(em) - em, np.cumsum(eM) - eM
        self.T_must, self.T_may = em.sum(), eM.sum()
        self.eps_c = 2.0 ** -17 * self.T_may + 2.0 * (eps * eM).sum()

    def allowed(self, u):
        if self.greedy:
            return self.g_allowed
        lo, hi = u * self.T_must - self.eps_c, u * self.T_may + self.eps_c
        return np.nonzero(self.may & (self.C_may + self.e >= lo) & (self.C_must <= hi))[0]

    def window(self, k):
        """(u_lo, u_hi): draws strictly inside allow token k alone (empty when u_lo >= u_hi or k is not must_keep)"""
        if self.greedy or not self.must[k] or self.T_must <= 0:
            return 1.0, 0.0
        return ((self.C_may[k] + self.eps_c) / self.T_must, (self.C_must[k] + self.e[k] - self.eps_c) / self.T_may)

    def point(self, u, mutant=None):
        """the token of the exact rule at draw u, optionally under a reference-level mutant"""
        if self.greedy:
            ids = np.nonzero(self.l == self.l.max())[0]
            return int(ids[-1] if mutant == "ties_high" else ids[0])
        kept = self.kept.copy()
        if mutant == "keep_more":
            rest = self.pos & ~kept
            if rest.any():
                kept |= rest & (self.e == self.e[rest].max())
        elif mutant == "drop_crossing":
            low = self.e[kept].min()
            if (self.e[kept] > low).any():
                kept &= self.e > low
        c = np.cumsum(self.e * kept)
        return int(np.argmax(c > u * c[-1]))

    def ratio(self, token, u):
        """measured error / bound of the kernel's token"""
        if self.greedy:
            d = self.l[self.jmax] - self.l[token]
            return 0.0 if d <= 0 else d / max(self.dl[token] + self.dl[self.jmax], 1e-300)
        if not self.may[token]:
            return float("inf")
        c, t = self.C_may[token], u * self.T_may
        return max(0.0, c - t, t - c - self.e[token]) / self.eps_c


# --------------------------------------------------------------------------- kernel layout and probes
def _r128(x):
    return (x + 127) // 128 * 128


def cta_slices(V, cs):
    W = _r128(-(-V // cs))
    return [(min(V, r * W), min(V, min(V, r * W) + W)) for r in range(cs)]


def handover_ids(V, cs):
    """ids where the kernel hands over between CTAs, warps, 32-id draw steps and the scalar tail"""
    ids = {0, V - 1}
    for lo, hi in cta_slices(V, cs):
        n = hi - lo
        if n <= 0:
            continue
        ids.update((lo, hi - 1))
        cw = _r128(-(-n // 32))
        for w in range(32):
            c0 = min(n, w * cw)
            c1 = min(n, c0 + cw)
            if c1 > c0:
                ids.update(lo + c for c in (c0, c1 - 1, min(c0 + 31, c1 - 1), min(c0 + 32, c1 - 1)))
        ids.update(range(lo + 4 * (n // 4), hi))
    return np.array(sorted(ids))


def cta_edges(V, cs):
    return np.array(sorted({i for lo, hi in cta_slices(V, cs) if hi > lo for i in (lo, hi - 1)}))


class Probe:
    def __init__(self, name, raw, *, temp=0.0, top_p=1.0, pen=1.0, seen=None, aims=None):
        self.name, self.raw, self.temp, self.top_p, self.pen, self.seen = name, raw, temp, top_p, pen, seen
        self.aims = aims          # candidate tokens for aimed draws (None: random draws, membership only)
        self.kind = {"spread": "spread", "edge": "edge", "ties": "ties", "pen": "penalty", "cap": "softcap",
                     "flat": "flat", "lim": "limits"}[name.split("_")[0].rstrip("0123456789")]


def _e64(raw, temp):
    l = raw.astype(np.float64) / temp
    return np.exp(l - l.max())


def make_probe(name, V, cs, i, rng):
    H = handover_ids(V, cs)
    temp3 = (0.7, 1.0, 1.3)[i % 3]

    def pick(k, pool=H):
        if k > len(pool):
            other = np.setdiff1d(np.arange(V), pool)
            return rng.permutation(np.concatenate([pool, rng.choice(other, k - len(pool), replace=False)]))
        return rng.choice(pool, k, replace=False)

    raw = (REST + 0.5 * rng.standard_normal(V)).astype(np.float32)
    if name.startswith("spread") or name in ("lim_p0", "lim_p1e-9", "lim_p1", "lim_p1.5", "lim_t1e-3", "lim_ninf"):
        K = {"lim_p1": 64}.get(name, int(name[6:]) if name.startswith("spread") else 7)
        band = pick(K)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, K)
        temp, top_p = temp3, (0.9, 1.0, 0.6)[(i // 3) % 3]
        if name.startswith("lim"):
            temp, top_p = 1.0, {"lim_p0": 0.0, "lim_p1e-9": 1e-9, "lim_p1": 1.0, "lim_p1.5": 1.5}.get(name, 0.9)
        if name == "lim_t1e-3":
            temp = 1e-3
        if name == "lim_ninf":
            lo, hi = cta_slices(V, cs)[i % cs] if cs > 1 else (V // 3, V // 2)
            mask = rng.random(V) < 0.5
            mask[lo:hi] = True
            mask[band] = False
            raw[mask] = -np.inf
            top_p = (0.9, 1.0)[i % 2]
        return Probe(name, raw, temp=temp, top_p=top_p, aims=band)
    if name in ("edge_wide", "edge_narrow"):
        band = pick(8)                                   # band[r] has rank r
        if name == "edge_wide":
            m = 1 + i % 5
            e = np.exp(-0.35 * np.arange(8))
        else:
            # the crossing token (rank m) and the next one sit in one level-1 bin ([0.5 + k/128, 0.5 + (k+1)/128)),
            # three quarters and one quarter of the way up
            m = 1 + i % 4
            e = np.concatenate([1.0 - 0.08 * np.arange(m), [0.5 + 8.75 / 128, 0.5 + 8.25 / 128],
                                0.4 - 0.05 * np.arange(8 - m - 2)])
        raw[band] = (temp3 * np.log(e) + BAND).astype(np.float32)
        ee = _e64(raw, temp3)
        srt = np.sort(ee[band])[::-1]
        top_p = 0.5 * (srt[:m].sum() + srt[:m + 1].sum()) / ee.sum()
        return Probe(name, raw, temp=temp3, top_p=top_p, aims=band[:m + 1][::-1])
    if name == "ties_sampled":
        pool = cta_edges(V, cs) if cs >= 4 else H
        ties = pick(6, pool)
        others = pick(4, np.setdiff1d(H, ties))
        raw[ties] = 10.0
        raw[others[0]] = 11.0
        raw[others[1:]] = 9.0
        ee = _e64(raw, 1.0)
        top_p = (1.0 + 2.5 * np.exp(-1.0)) / ee.sum()
        return Probe(name, raw, temp=1.0, top_p=top_p, aims=np.append(ties, others[0]))
    if name == "ties_greedy":
        raw = (2.0 + rng.standard_normal(V)).astype(np.float32)
        pool = cta_edges(V, cs) if cs >= 2 else H
        ties = np.concatenate([pick(min(4, len(pool)), pool), pick(2)])
        raw[ties] = 10.0
        return Probe(name, raw)
    if name.startswith("pen_"):
        pen = (1.15, 2.0, 1.0)[i % 3] if name == "pen_sampled" else (1.0 if name == "pen_one" else (1.15, 2.0)[i % 2])
        seen = rng.random(V) < 0.01
        tail = V % 32
        if tail:
            seen[V - tail:] = True                           # every id of the last, partial bitmap word
        if name == "pen_sampled":
            band = pick(8)
            raw[band] = np.array([2.0, 1.2, 0.6, 0.2, -0.3, -0.8, -1.3, -2.0], np.float32)
            seen[band] = np.arange(8) % 2 == 0
            return Probe(name, raw, temp=1.0, top_p=(1.0, 0.9)[i % 2], pen=pen, seen=seen, aims=band)
        a = V - 1 - int(rng.integers(tail)) if tail and i % 2 == 0 else int(pick(1)[0])
        b = int(pick(1, np.setdiff1d(H, [a]))[0])
        if name in ("pen_pos", "pen_one"):
            raw = (2.0 + 0.5 * rng.standard_normal(V)).astype(np.float32)
            raw[a], raw[b] = 10.0, 9.0
        else:
            raw = (-5.0 + 0.5 * rng.standard_normal(V)).astype(np.float32)
            raw[a], raw[b] = (-1.0, -1.1) if name == "pen_neg" else (-1.1, -1.0)
        seen[a], seen[b] = True, False
        return Probe(name, raw, pen=pen, seen=seen)
    if name == "flat":
        raw = (rng.standard_normal(V) * (1.0, 4.0)[i % 2]).astype(np.float32)
        return Probe(name, raw, temp=temp3 + (0.2 if temp3 > 1 else 0.0), top_p=(0.9, 0.95, 1.0)[(i // 3) % 3])
    if name in ("lim_one", "lim_one_greedy"):
        raw = np.full(V, -np.inf, np.float32)
        k = pick(1)
        raw[k] = rng.uniform(-3.0, 3.0)
        return Probe(name, raw, temp=1.0 if name == "lim_one" else 0.0, top_p=0.9, aims=k)
    if name.startswith("cap_"):
        raw = rng.uniform(-60.0, 0.0, V).astype(np.float32)
        if name == "cap_sat_greedy":
            return Probe(name, rng.uniform(-60.0, 60.0, V).astype(np.float32))
        band = pick(5)
        raw[band] = np.array([60.0, 45.0, 38.0, 34.0, 31.0]) + rng.uniform(-0.5, 0.5, 5)
        if name == "cap_greedy":
            return Probe(name, raw)
        seen = None
        if name == "cap_seen":
            seen = np.zeros(V, bool)
            seen[band[0]] = True
        return Probe(name, raw, temp=0.8 if name == "cap_t08_p1" else 1.0,
                     top_p=0.95 if name == "cap_t1" else 1.0, pen=2.0 if seen is not None else 1.0, seen=seen,
                     aims=band)
    raise ValueError(name)


def pack_bits(bits):
    """bool [rows, V] -> int32 [rows, ceil(V / 32)] bitmap (bit i of word w = id 32 w + i)"""
    rows, V = bits.shape
    words = (V + 31) // 32
    padded = np.zeros((rows, words * 32), bool)
    padded[:, :V] = bits
    return np.packbits(padded, axis=1, bitorder="little").view(np.uint32).view(np.int32)


class Launch:
    """B probe rows for one ``sample`` call, ``rounds`` rounds of (step, seeds), and every row's reference.  Per-sequence
    state (temperature, top_p, penalty, seeds, seen) lives at state row row_map[b] of ``n_state`` rows."""

    def __init__(self, V, cs, B, variants, *, cap=0.0, rounds=len(STEPS), seed=0, offset=0, row_map=None,
                 n_state=None):
        rng = np.random.default_rng(seed)
        self.V, self.cs, self.B, self.cap = V, cs, B, cap
        self.row_map = np.arange(B) if row_map is None else np.asarray(row_map)
        S = self.n_state = B if n_state is None else n_state
        self.probes = [make_probe(variants[(i + offset) % len(variants)], V, cs, i, rng) for i in range(B)]
        self.refs = [RowRef(p.raw, p.seen, p.temp, p.top_p, p.pen, cap) if bb >= 0 else None
                     for p, bb in zip(self.probes, self.row_map)]
        self.logits = np.stack([p.raw for p in self.probes])
        self.temp = rng.uniform(0.5, 2.0, S).astype(np.float32)        # rows no logits row maps to: junk
        self.top_p = rng.uniform(0.1, 1.0, S).astype(np.float32)
        self.pen = rng.uniform(1.0, 3.0, S).astype(np.float32)
        seen = rng.random((S, V)) < 0.3
        for b, (p, bb) in enumerate(zip(self.probes, self.row_map)):
            if bb >= 0:
                self.temp[bb], self.top_p[bb], self.pen[bb] = p.temp, p.top_p, p.pen
                seen[bb] = False if p.seen is None else p.seen
        self.seen = pack_bits(seen)
        self.steps = STEPS[:rounds]
        self.seeds = rng.integers(0, 1 << 32, (rounds, S), dtype=np.uint64).astype(np.uint32)
        self.draws = []           # [round][b] = (u, allowed ids, aimed token or None)
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
        """failures of round t (``out_state``: out_tokens by state row)"""
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
            MEASURED[p.kind] = max(MEASURED[p.kind], r)
            if p.kind == "flat":
                FLAT_SIZES.append(len(allowed))
            if aim is not None and tok != aim:
                bad.append(f"{tag} row {b} {p.name}: aimed at {aim}, got {tok} (u={u:.7f}, err/bound {r:.3g})")
            elif tok not in allowed:
                bad.append(f"{tag} row {b} {p.name}: token {tok} not in {allowed[:8].tolist()} (err/bound {r:.3g})")
        return bad


# --------------------------------------------------------------------------- CPU: the reference and the probes
def test_ref64_matches_torch_ref_where_unambiguous():
    """on tie-free random logits the nucleus (where must_keep == may_keep) is torch_ref's top-p mask, and greedy with
    a penalty is torch_ref's pick"""
    from bee2bee_b200.models import torch_ref
    rng = np.random.default_rng(1)
    checked = 0
    for i in range(24):
        V = (1000, 3001, 4096)[i % 3]
        raw = (rng.standard_normal(V) * (1.0, 3.0)[i % 2]).astype(np.float32)
        temp, top_p = (0.7, 1.0, 1.5)[i % 3], (0.5, 0.9, 0.95, 0.99)[i % 4]
        ref = RowRef(raw, temp=temp, top_p=top_p)
        if (ref.must != ref.may).any():
            continue
        checked += 1
        keep = torch_ref.top_p_keep_mask(torch.from_numpy(raw)[None], temp, top_p)[0].numpy()
        assert np.array_equal(ref.must, keep), (i, np.nonzero(ref.must != keep))
        seen = rng.random(V) < 0.2
        g = RowRef(raw, seen=seen, temp=0.0, pen=1.3)
        exp = torch_ref.sample_reference(torch.from_numpy(raw)[None], torch.from_numpy(seen)[None], 0.0, 1.0, 1.3)
        assert g.g_allowed.tolist() == [int(exp[0])]
    assert checked >= 16


def test_u01_reproduces_the_float32_rounding():
    """h >> 8 >= 2^23: + 0.5 rounds to even in float32; the step product wraps in uint32"""
    h = np.array([0xFFFFFFFF, 0x80000000, 0x800000FF, 0x00000100], np.uint32)
    u = _u_of_hash(h)
    assert u.dtype == np.float32
    assert u[0] == np.float32(1.0)                          # (2^24 - 1) + 0.5 rounds up to 2^24
    assert u[1] == np.float32(0.5)                          # 2^23 + 0.5 rounds to 2^23
    assert u[3] == np.float32(1.5 / 2 ** 24)


@pytest.mark.parametrize("V,cs", [(1000, 1), (1000, 8), (32000, 2), (50257, 4), (50257, 8), (128256, 4)])
def test_aimed_draws_allow_exactly_one_token(V, cs):
    """every aimed draw of every probe allows exactly the aimed token; spread / edge / ties probes all get aims"""
    L = Launch(V, cs, len(VARIANTS), VARIANTS, rounds=3, seed=V + cs)
    Lc = Launch(V, cs, 8, SOFTCAP_VARIANTS, cap=SOFTCAP, rounds=3, seed=V + cs + 1)
    aimed = defaultdict(int)
    for launch in (L, Lc):
        for t in range(3):
            for p, d in zip(launch.probes, launch.draws[t]):
                u, allowed, aim = d
                if aim is not None:
                    assert allowed.tolist() == [aim], (p.name, t, aim, allowed[:8])
                    aimed[p.kind] += 1
    for kind in ("spread", "edge", "ties", "penalty", "limits", "softcap"):
        assert aimed[kind] > 0, kind


def test_handover_ids_cover_slices_warps_and_tail():
    for V, cs in ((50257, 8), (1000, 8), (128256, 4), (32000, 1)):
        H = set(handover_ids(V, cs).tolist())
        W = _r128(-(-V // cs))
        assert {0, V - 1} <= H
        for r in range(cs):
            if r * W < V:
                assert r * W in H and min(V, r * W + W) - 1 in H
        lo, hi = cta_slices(V, cs)[-1]
        assert set(range(lo + 4 * ((hi - lo) // 4), hi)) <= H


def _caught(launch, mutant, names):
    """does the reference-level mutant leave the allowed set on some draw of the probes ``names``?"""
    hits = 0
    for t in range(len(launch.steps)):
        for b, (p, ref, d) in enumerate(zip(launch.probes, launch.refs, launch.draws[t])):
            if d is None or p.name not in names:
                continue
            u, allowed, _ = d
            bb = int(launch.row_map[b])
            if mutant == "one_sided_penalty":
                tok = RowRef(p.raw, p.seen, p.temp, p.top_p, p.pen, launch.cap, one_sided_penalty=True).point(u)
            elif mutant == "rng_state_row":
                tok = ref.point(u01(launch.seeds[t, bb], launch.steps[t], bb))
            else:
                tok = ref.point(u, mutant)
            hits += tok not in allowed
    return hits


@pytest.mark.parametrize("mutant,names,cs", [
    ("keep_more", ("edge_wide", "edge_narrow"), 2),
    ("drop_crossing", ("edge_wide", "edge_narrow"), 4),
    ("ties_high", ("ties_greedy",), 8),
    ("one_sided_penalty", ("pen_neg", "pen_neg2", "pen_sampled"), 2),
    ("rng_state_row", PLUMB_VARIANTS, 4),
])
def test_probe_catches_reference_mutant(mutant, names, cs):
    V, B = 32000, 10
    row_map = np.array([4, 0, 9, 2, -1, 7, 1, 12, 3, 5]) if mutant == "rng_state_row" else None
    L = Launch(V, cs, B, names, rounds=4, seed=7, row_map=row_map, n_state=13 if row_map is not None else None)
    assert _caught(L, mutant, names) > 0
    # the correct rule stays inside the allowed set
    for t in range(4):
        for p, ref, d in zip(L.probes, L.refs, L.draws[t]):
            if d is not None:
                assert ref.point(d[0]) in d[1], (p.name, t)


# --------------------------------------------------------------------------- GPU
def _ops():
    from bee2bee_b200 import ops
    return ops


def cluster_cases(V):
    """{cs: batch} for every cluster size ``sample`` reaches at vocabulary V on this device (batch 1 .. MAX_B), the
    batch nearest 24 within each cluster size's range"""
    q = _ops().native().sample_cluster_size
    by = defaultdict(list)
    for B in range(1, MAX_B + 1):
        by[int(q(B, V))].append(B)
    assert 0 not in by, V
    return {cs: min(max(24, Bs[0]), Bs[-1]) for cs, Bs in by.items()}


def _i32(a, dev="cuda"):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).astype(np.uint32).view(np.int32))).to(dev)


def _step_tensor(step):
    return _i32(np.array([step], np.uint64).astype(np.uint32))


def _run_launch(L, tag, logits=None, vocab=0):
    """every round of L through ``sample``; checks tokens, the seen bitmap and identical bytes on a repeat"""
    ops = _ops()
    dev = "cuda"
    if logits is None:
        logits = torch.from_numpy(L.logits).to(dev)
    temp, top_p, pen = (torch.from_numpy(a).to(dev) for a in (L.temp, L.top_p, L.pen))
    seen0 = torch.from_numpy(L.seen).to(dev)
    out = torch.empty(L.n_state, dtype=torch.int32, device=dev)
    bad, outs = [], []
    for t, step in enumerate(L.steps):
        seeds, st = _i32(L.seeds[t]), _step_tensor(step)
        reps = []
        for _ in range(2 if t == 0 else 1):
            seen = seen0.clone()
            out.fill_(-1)
            ops.sample(logits, out, seen=seen, temperature=temp, top_p=top_p, rep_penalty=pen, seeds=seeds, step=st,
                       vocab=vocab, softcap=L.cap)
            reps.append((out.cpu().numpy().copy(), seen.cpu().numpy()))
        if len(reps) == 2:
            assert np.array_equal(reps[0][0], reps[1][0]) and np.array_equal(reps[0][1], reps[1][1]), \
                f"{tag}: two identical launches differ"
        got, seen_after = reps[0]
        bad += L.check(t, got, f"{tag} step {step:#x}")
        exp_seen = L.seen.copy().view(np.uint32)
        for b, bb in enumerate(L.row_map):
            tok = int(got[bb])
            if bb >= 0 and 0 <= tok < L.V:
                exp_seen[bb, tok >> 5] |= np.uint32(1 << (tok & 31))
        if not np.array_equal(seen_after.view(np.uint32), exp_seen):
            bad.append(f"{tag} step {step:#x}: seen bitmap is not the old bits plus the drawn tokens")
        outs.append(got)
    assert not bad, f"{len(bad)} failures:\n" + "\n".join(bad[:12])
    return outs


def _report():
    print("\nerr/bound per probe kind: " + "  ".join(f"{k}={v:.3f}" for k, v in sorted(MEASURED.items())))
    if FLAT_SIZES:
        print(f"flat: mean allowed-set size {np.mean(FLAT_SIZES):.1f} over {len(FLAT_SIZES)} draws")
    print("cluster sizes run: " + "  ".join(f"V={v}: {sorted(c)}" for v, c in sorted(CS_RUN.items())))


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_sweep_matches_ref64_at_every_cluster_size(V):
    """every probe kind, mixed greedy and sampled rows, at every cluster size V reaches; one soft-capped launch"""
    cases = cluster_cases(V)
    for cs, B in sorted(cases.items()):
        L = Launch(V, cs, B, VARIANTS, seed=V + cs, offset=(V // 7 + 5 * cs) % len(VARIANTS))
        _run_launch(L, f"V={V} cs={cs} B={B}")
        CS_RUN[V].add(cs)
    cs = max(cases)
    L = Launch(V, cs, cases[cs], SOFTCAP_VARIANTS, cap=SOFTCAP, rounds=4, seed=V + 100 + cs)
    _run_launch(L, f"V={V} cs={cs} softcap")
    _report()


@gpu
def test_cluster_sizes_reach_every_size():
    """the sweep's batch sizes reach cs = 1, 2, 4 and 8 over its vocabularies; too large a vocabulary is refused"""
    ops = _ops()
    reached = {V: set(cluster_cases(V)) for V in VOCABS}
    print("\ncluster sizes per vocabulary: " + "  ".join(f"V={v}: {sorted(c)}" for v, c in reached.items()))
    assert set().union(*reached.values()) == {1, 2, 4, 8}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms == 132:
        assert reached == {1000: {1, 2, 4, 8}, 32000: {1, 2, 4, 8}, 50257: {2, 4, 8}, 128256: {4, 8},
                           151936: {8}, 256000: {8}}
    assert ops.native().sample_cluster_size(1, 300000) == 0
    out = torch.full((1,), -3, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError):
        ops.sample(torch.zeros(1, 300000, device="cuda"), out)
    torch.cuda.synchronize()
    assert out.item() == -3


@gpu
@pytest.mark.parametrize("V,B", [(50257, 12), (500, 3)])
def test_padded_and_unaligned_rows_match(V, B):
    """ld > V with NaN and +inf in the padding, and a contiguous [B, V] tensor whose odd row stride takes the scalar
    load path, give the tokens of the same logits padded to an aligned ld (V = 500 at cs = 8 leaves CTAs empty)"""
    ops = _ops()
    cs = int(ops.native().sample_cluster_size(B, V))
    L = Launch(V, cs, B, PLUMB_VARIANTS, rounds=3, seed=V)
    base = _run_launch(L, f"V={V} contiguous")
    for ld in (_r128(V) + 4, V + 3):
        buf = np.full((B, ld), np.nan, np.float32)
        buf[:, V::2] = np.inf
        buf[:, :V] = L.logits
        padded = _run_launch(L, f"V={V} ld={ld}", logits=torch.from_numpy(buf).cuda(), vocab=V)
        for a, b in zip(base, padded):
            assert np.array_equal(a, b), f"ld={ld}: tokens differ from the contiguous rows"


@gpu
def test_row_map_history_ring_peer_tokens_and_flags():
    """row_map with a permutation and skipped rows: state rows it does not own keep their sentinels in out_tokens,
    peer_tokens, history, hist_pos and seen; the history ring wraps; the flag epoch rises by one per call (also when
    every row is skipped) and the done counter resets; the RNG is keyed on the logits row"""
    ops = _ops()
    dev = "cuda"
    V, B, S, stride = 32000, 10, 13, 8
    row_map = np.array([4, 0, 9, 2, -1, 7, 1, 12, 3, -1])
    cs = int(ops.native().sample_cluster_size(B, V))
    L = Launch(V, cs, B, PLUMB_VARIANTS, rounds=4, seed=3, row_map=row_map, n_state=S)
    owned = sorted(int(x) for x in row_map if x >= 0)
    free = [r for r in range(S) if r not in owned]
    rm = torch.from_numpy(row_map.astype(np.int32)).to(dev)
    temp, top_p, pen = (torch.from_numpy(a).to(dev) for a in (L.temp, L.top_p, L.pen))
    out = torch.full((S,), -77, dtype=torch.int32, device=dev)
    peer = torch.full((S,), -66, dtype=torch.int32, device=dev)
    hist = torch.full((S, stride), -55, dtype=torch.int32, device=dev)
    pos0 = np.full(S, 999, np.int32)
    pos0[owned] = [0, 7, 8, 13, 3 * stride + 5, 1, 6, 100][:len(owned)]
    hist_pos = torch.from_numpy(pos0.copy()).to(dev)
    flag, epoch, counter = (torch.tensor([v], dtype=torch.int32, device=dev) for v in (0, 41, 0))
    seen = torch.from_numpy(L.seen).to(dev)
    exp_hist = np.full((S, stride), -55, np.int32)
    exp_pos = pos0.copy()
    calls = 0

    def call(rmap, seeds, st, seeds_on=True):
        nonlocal calls
        seen.copy_(torch.from_numpy(L.seen))
        ops.sample(torch.from_numpy(L.logits).to(dev), out, seen=seen, temperature=temp, top_p=top_p, rep_penalty=pen,
                   seeds=seeds if seeds_on else None, step=st, peer_tokens=peer.data_ptr(), history=hist.data_ptr(),
                   hist_pos=hist_pos, hist_stride=stride, signal_flag=flag.data_ptr(), signal_epoch=epoch.data_ptr(),
                   done_counter=counter.data_ptr(), row_map=rmap.data_ptr())
        torch.cuda.synchronize()
        calls += 1
        assert epoch.item() == 41 + calls and flag.item() == epoch.item() and counter.item() == 0, \
            (calls, epoch.item(), flag.item(), counter.item())

    bad = []
    for t, step in enumerate(L.steps):
        call(rm, _i32(L.seeds[t]), _step_tensor(step))
        got = out.cpu().numpy()
        bad += L.check(t, got, f"row_map step {step:#x}")
        for bb in owned:
            exp_hist[bb, exp_pos[bb] % stride] = got[bb]
            exp_pos[bb] += 1
        assert np.array_equal(peer.cpu().numpy()[owned], got[owned])
        assert (got[free] == -77).all() and (peer.cpu().numpy()[free] == -66).all()
        assert np.array_equal(hist.cpu().numpy(), exp_hist), t
        assert np.array_equal(hist_pos.cpu().numpy(), exp_pos), t
        exp_seen = L.seen.copy().view(np.uint32)
        for bb in owned:
            exp_seen[bb, got[bb] >> 5] |= np.uint32(1 << (int(got[bb]) & 31))
        assert np.array_equal(seen.cpu().numpy().view(np.uint32), exp_seen), t
    assert not bad, "\n".join(bad[:12])

    # every row skipped: only the flag handoff moves
    before = [x.cpu().clone() for x in (out, peer, hist, hist_pos)]
    call(torch.full((B,), -1, dtype=torch.int32, device=dev), _i32(L.seeds[0]), _step_tensor(0))
    for a, x in zip(before, (out, peer, hist, hist_pos)):
        assert torch.equal(a, x.cpu())
    assert np.array_equal(seen.cpu().numpy(), L.seen)

    # no seeds and no step: seed 0x1234567, step 0
    out_ns = torch.full((S,), -77, dtype=torch.int32, device=dev)
    ops.sample(torch.from_numpy(L.logits).to(dev), out_ns, seen=torch.from_numpy(L.seen).to(dev), temperature=temp,
               top_p=top_p, rep_penalty=pen, row_map=rm.data_ptr())
    got = out_ns.cpu().numpy()
    for b, (ref, bb) in enumerate(zip(L.refs, row_map)):
        if bb >= 0:
            assert got[bb] in ref.allowed(u01(NO_SEED, 0, b)), (b, got[bb])
    assert (got[free] == -77).all()


@gpu
def test_mark_seen_ignores_out_of_range_ids():
    """duplicates set one bit; ids -1, V and V + 5 (inside the last bitmap word's padding) are ignored"""
    ops = _ops()
    V, rows = 1000, 3
    rng = np.random.default_rng(5)
    init = pack_bits(rng.random((rows, V)) < 0.1)
    ids = np.array([5, 5, 999, 992, -1, V, V + 5, 0, 31, 32, 999, 700, V + 5, -1], np.int32)
    seq = np.array([0, 0, 0, 1, 1, 1, 2, 2, 2, 2, 1, 0, 0, 2], np.int32)
    exp = init.copy().view(np.uint32)
    for i, s in zip(ids, seq):
        if 0 <= i < V:
            exp[s, i >> 5] |= np.uint32(1 << (int(i) & 31))
    seen = torch.from_numpy(init).cuda()
    ops.mark_seen(torch.from_numpy(ids).cuda(), torch.from_numpy(seq).cuda(), seen, V)
    assert np.array_equal(seen.cpu().numpy().view(np.uint32), exp)
