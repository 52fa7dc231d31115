"""Logit bias in the fused sampler (``sample_kernel``) against a plain reference, at every cluster size the launcher
picks, with draws aimed at chosen tokens; the refusals of the binding; and the engine that carries the bias.

Semantics (vLLM / OpenAI ``logit_bias``): a row's tables hold token ids and biases; for its first
n = min(bias_n, width) entries, l[id] = l[id] + b in fp32 (round to nearest) right after soft-cap, so the repetition
penalty's sign test sees the biased logit, then the presence / frequency penalties, temperature and the filters.  Ids
outside [0, V) are ignored; bias_n = 0 turns the bias off.  Greedy rows are biased too.

Reference: without soft-cap the bias is one exact fp32 addition, so the biased row is built in numpy float32 and handed
to the penalty test's references (``PenRef``, or ``FiltRef`` for rows with top-k or min-p), which treat their input as
the kernel's logits after soft-cap.  With soft-cap the kernel computes cap tanh(l / cap) + b; that is RowRef's soft-cap
of the logit l' = cap atanh(tanh(l / cap) + b / cap), so the capped probes keep every biased logit inside (-cap, cap)
and use ``RowRef`` on l' with its soft-cap error model.

Probes bias the ids where the kernel hands over (CTA slice edges, id 0 and V - 1), move the greedy argmax either way,
ban the argmax with -100 (greedy and sampled), force a token with +100, bias a seen id whose logit turns positive (the
repetition penalty's sign), combine the bias with presence / frequency penalties and with top-k / top-p / min-p, fill
the table to its width, give bias_n beyond the width (clamped), and put ids outside the vocabulary in the table.  Rows
with bias_n = 0 carry junk in their tables; entries past bias_n are junk too."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from test_sampler_penalty_ref_gpu import MEASURED, PenRef, PLaunch, penalise32
from test_sampler_ref_gpu import (AIM_AT, STEPS, VARIANTS, Launch, RowRef, aim_seed, cluster_cases, cta_edges,
                                  handover_ids, pack_bits, u01)
from test_sampler_topk_ref_gpu import FiltRef

gpu = pytest.mark.gpu

VOCABS = (32000, 128256, 151936)
REST, BAND = -10.0, 10.0
SOFTCAP = 30.0
WIDTH = 1024                  # LOGIT_BIAS_MAX: the width of the engine's tables
BVARIANTS = ("b_edges", "b_up", "b_down", "b_ban_greedy", "b_ban_sampled", "b_force", "b_seen_sign", "b_pf",
             "b_topk", "b_topp", "b_minp", "b_full", "b_clamp", "b_oob", "b_off")
CAP_VARIANTS = ("bc_sampled", "bc_greedy", "bc_seen")


# --------------------------------------------------------------------------- reference
def bias32(raw, ids, vals, mutant=None):
    """the row after the bias step in float32 (``mutant`` "every_id": the first bias is added to every id as well)"""
    l = np.asarray(raw, np.float32).copy()
    ids, vals = np.asarray(ids, np.int64), np.asarray(vals, np.float32)
    ok = (ids >= 0) & (ids < l.size)
    if mutant == "every_id" and ok.any():
        l = (l + vals[ok][0]).astype(np.float32)
        l[ids[ok]] = (np.asarray(raw, np.float32)[ids[ok]] + vals[ok]).astype(np.float32)
        return l
    l[ids[ok]] = (l[ids[ok]] + vals[ok]).astype(np.float32)
    return l


class BProbe:
    """One row: kernel input ``raw`` and its bias table entries (``ids``, ``vals``; ``n`` of them in use, None = all),
    plus the controls of the penalty and filter tests.  ``expect``: the one token a greedy row may return."""

    def __init__(self, name, raw, ids, vals, *, n=None, temp=0.0, top_p=1.0, pen=1.0, seen=None, counts=None,
                 pres=0.0, freq=0.0, top_k=0, min_p=0.0, aims=None, expect=None):
        self.name, self.raw, self.ids, self.vals = name, raw, np.asarray(ids, np.int64), np.asarray(vals, np.float32)
        self.n = len(self.ids) if n is None else n
        self.temp, self.top_p, self.pen, self.seen, self.counts = temp, top_p, pen, seen, counts
        self.pres, self.freq, self.top_k, self.min_p, self.aims, self.expect = pres, freq, top_k, min_p, aims, expect

    def used(self):
        k = min(self.n, WIDTH)
        return self.ids[:k], self.vals[:k]

    def ref(self, cap=0.0, mutant=None):
        ids, vals = self.used()
        if cap > 0:
            # cap tanh(l / cap) + b == cap tanh(l' / cap): RowRef's soft-cap of l'
            t = np.tanh(self.raw.astype(np.float64) / cap)
            t[ids] += vals.astype(np.float64) / cap
            assert np.abs(t).max() < 1.0, "a capped probe must keep its biased logits inside (-cap, cap)"
            return RowRef((cap * np.arctanh(t)).astype(np.float32), self.seen, self.temp, self.top_p, self.pen, cap)
        if mutant == "after_pen":        # the bias added after the penalties
            l = penalise32(self.raw, self.seen, self.counts, self.pen, self.pres, self.freq)
            l = bias32(l, ids, vals)
            return PenRef(l, temp=self.temp, top_p=self.top_p) if not (self.top_k or self.min_p) else \
                FiltRef(l, self.temp, self.top_p, self.top_k, self.min_p)
        lb = bias32(self.raw, ids, vals, mutant)
        if self.top_k or self.min_p:
            l = penalise32(lb, self.seen, self.counts, self.pen, self.pres, self.freq)
            return FiltRef(l, self.temp, self.top_p, self.top_k, self.min_p)
        return PenRef(lb, self.seen, self.counts, self.pres, self.freq, self.temp, self.top_p, self.pen)


def make_bprobe(name, V, cs, i, rng):
    H = handover_ids(V, cs)
    E = cta_edges(V, cs)
    temp3 = (0.7, 1.0, 1.3)[i % 3]

    def pick(k, pool=H, avoid=()):
        pool = np.setdiff1d(np.asarray(pool), np.asarray(avoid, np.int64))
        if k > len(pool):
            other = np.setdiff1d(np.arange(V), np.concatenate([pool, np.asarray(avoid, np.int64)]))
            return rng.permutation(np.concatenate([pool, rng.choice(other, k - len(pool), replace=False)]))
        return rng.choice(pool, k, replace=False)

    raw = (REST + 0.5 * rng.standard_normal(V)).astype(np.float32)
    if name == "b_edges":          # the bias lifts CTA edges, id 0 and V - 1 into the band
        band = np.unique(np.concatenate([[0, V - 1], pick(min(6, len(E)), E, (0, V - 1))]))
        vals = (BAND - raw[band] + rng.uniform(-1.0, 1.0, band.size)).astype(np.float32)
        return BProbe(name, raw, band, vals, temp=temp3, top_p=(1.0, 0.9)[(i // 3) % 2], aims=band)
    if name in ("b_up", "b_down", "b_ban_greedy"):     # greedy: the bias moves the argmax
        a, b = pick(2, E if cs >= 2 else H)
        raw[a], raw[b] = BAND, BAND - 0.5
        ids, vals = {"b_up": ([b], [0.75]), "b_down": ([a], [-0.75]), "b_ban_greedy": ([a], [-100.0])}[name]
        return BProbe(name, raw, ids, vals, expect=int(b))
    if name == "b_ban_sampled":    # -100 on the argmax of a sampled band: the rest is drawn
        band = pick(6)
        raw[band] = BAND - np.array([0.0, 0.3, 0.5, 0.8, 1.0, 1.4], np.float32)
        return BProbe(name, raw, band[:1], [-100.0], temp=temp3, top_p=(1.0, 0.95)[i % 2], aims=band[1:])
    if name == "b_force":          # +100 on a bulk token: it is the only one that can be drawn
        raw[pick(5)] = BAND
        t = pick(1, np.setdiff1d(np.arange(V), H))
        greedy = i % 2 == 1
        return BProbe(name, raw, t, [100.0], temp=0.0 if greedy else 1.0, aims=None if greedy else t,
                      expect=int(t[0]) if greedy else None)
    if name == "b_seen_sign":      # seen id at -1, biased to +1.5: the penalty divides (1.5 / 2 = 0.75)
        a, c = pick(2)
        raw = (-5.0 + 0.5 * rng.standard_normal(V)).astype(np.float32)
        raw[a], raw[c] = -1.0, (0.6, 1.0)[i % 2]      # a wins (0.75 > 0.6) / c wins (0.75 < 1.0)
        seen = rng.random(V) < 0.01
        seen[a], seen[c] = True, False
        return BProbe(name, raw, [a], [2.5], pen=2.0, seen=seen, expect=int(a if i % 2 == 0 else c))
    if name == "b_pf":             # bias and presence / frequency penalties on the same tokens
        band = pick(8)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, 8)
        counts = np.zeros(V, np.int32)
        counts[rng.choice(V, 200, replace=False)] = 1
        counts[band] = (0, 1, 2, 0, 3, 1, 0, 2)
        return BProbe(name, raw, band[::2], rng.uniform(-1.5, 1.5, 4), temp=temp3, counts=counts, pres=0.4,
                      freq=0.3, aims=band)
    if name in ("b_topk", "b_topp", "b_minp"):        # the bias reorders the top of the band under a filter
        band = pick(10)
        raw[band] = (temp3 * np.log(np.exp(-0.25 * np.arange(10))) + BAND).astype(np.float32)
        kw = {"b_topk": dict(top_k=3), "b_topp": dict(top_p=0.7), "b_minp": dict(min_p=0.3)}[name]
        return BProbe(name, raw, band[[5, 0, 2]], [1.3, -0.6, 0.4], temp=temp3, aims=band[:7], **kw)
    if name in ("b_full", "b_clamp"):  # WIDTH entries (the band among them); b_clamp gives bias_n beyond the width
        band = pick(6)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, 6)
        ids = rng.permutation(np.concatenate([band, rng.choice(np.setdiff1d(np.arange(V), band), WIDTH - 6,
                                                               replace=False)]))
        vals = rng.uniform(-2.0, 2.0, WIDTH).astype(np.float32)
        return BProbe(name, raw, ids, vals, n=WIDTH if name == "b_full" else WIDTH + 777, temp=temp3, aims=band)
    if name == "b_oob":            # ids outside the vocabulary are ignored
        band = pick(6)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, 6)
        ids = np.array([-1, band[0], V, -(1 << 31), band[1], V + 7, (1 << 31) - 1], np.int64)
        vals = np.array([100.0, 0.5, 100.0, 100.0, -0.7, -100.0, 100.0], np.float32)
        return BProbe(name, raw, ids, vals, temp=temp3, aims=band)
    if name == "b_off":            # bias_n = 0: the table row holds junk
        band = pick(6)
        raw[band] = BAND + rng.uniform(-1.0, 1.0, 6)
        return BProbe(name, raw, band, np.full(6, 50.0, np.float32), n=0, temp=temp3, top_p=0.9, aims=band)
    if name.startswith("bc_"):     # soft-capped launch: the bias reorders the capped band and keeps it inside the cap
        raw = rng.uniform(-60.0, 0.0, V).astype(np.float32)
        band = pick(5)
        raw[band] = np.array([60.0, 45.0, 38.0, 34.0, 31.0]) + rng.uniform(-0.5, 0.5, 5)
        vals = np.array([-3.0, 2.0, 3.5, -1.0, 0.0], np.float32)
        if name == "bc_greedy":
            return BProbe(name, raw, band, vals)
        seen = None
        if name == "bc_seen":
            seen = np.zeros(V, bool)
            seen[band[[0, 2]]] = True
        return BProbe(name, raw, band, vals, temp=1.0, top_p=0.95 if name == "bc_sampled" else 1.0,
                      pen=2.0 if seen is not None else 1.0, seen=seen, aims=band)
    raise ValueError(name)


class BLaunch(PLaunch):
    """B bias probes for one ``sample`` call (``PLaunch``'s checks); per-sequence state at row_map[b] of n_state rows,
    junk controls and junk bias tables in the state rows no logits row maps to.  ``plain``: rows whose bias is turned
    off (their tables keep junk)."""

    def __init__(self, V, cs, B, variants, *, cap=0.0, rounds=len(STEPS), seed=0, offset=0, row_map=None,
                 n_state=None, plain=()):
        rng = np.random.default_rng(seed)
        self.V, self.cs, self.B, self.cap = V, cs, B, cap
        self.row_map = np.arange(B) if row_map is None else np.asarray(row_map)
        S = self.n_state = B if n_state is None else n_state
        self.probes = [make_bprobe(variants[(i + offset) % len(variants)], V, cs, i, rng) for i in range(B)]
        for b in plain:
            self.probes[b].n, self.probes[b].expect = 0, None
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
        self.bias_ids = rng.integers(0, V, (S, WIDTH)).astype(np.int32)
        self.bias_vals = rng.uniform(-100.0, 100.0, (S, WIDTH)).astype(np.float32)
        self.bias_n = rng.integers(1, WIDTH, S).astype(np.int32)
        seen = rng.random((S, V)) < 0.3
        for p, bb in zip(self.probes, self.row_map):
            if bb >= 0:
                self.temp[bb], self.top_p[bb], self.pen[bb] = p.temp, p.top_p, p.pen
                self.top_k[bb], self.min_p[bb], self.pres[bb], self.freq[bb] = p.top_k, p.min_p, p.pres, p.freq
                self.counts[bb] = 0
                if p.counts is not None:
                    self.counts[bb, :V] = p.counts
                k = min(len(p.ids), WIDTH)
                self.bias_ids[bb, :k] = p.ids[:k].astype(np.int64).clip(-(1 << 31), (1 << 31) - 1)
                self.bias_vals[bb, :k] = p.vals[:k]
                self.bias_n[bb] = p.n
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


# --------------------------------------------------------------------------- CPU: the reference and the probes
def test_bias_reference_matches_sample_reference():
    """greedy picks and (where must == may) the kept set of the biased row equal torch_ref.sample_reference's with
    ``bias``, together with the repetition and presence / frequency penalties"""
    from bee2bee_b200.models import torch_ref
    rng = np.random.default_rng(4)
    checked = 0
    for i in range(24):
        V = 400
        raw = (rng.standard_normal(V) * 2.0).astype(np.float32)
        ids = rng.choice(V, 40, replace=False)
        vals = rng.uniform(-3.0, 3.0, 40).astype(np.float32)
        seen = rng.random(V) < 0.2
        counts = np.where(rng.random(V) < 0.3, rng.integers(1, 6, V), 0).astype(np.int32)
        pen, pres, freq = (1.0, 1.3)[i % 2], (0.0, 0.4)[(i // 2) % 2], (0.0, 0.3)[(i // 2) % 2]
        temp, top_p = (0.7, 1.0, 1.3)[i % 3], (1.0, 0.9, 0.6)[i % 3]
        bias = (torch.from_numpy(ids), torch.from_numpy(vals))
        args = (torch.from_numpy(raw)[None], torch.from_numpy(seen)[None])
        kw = dict(counts=torch.from_numpy(counts)[None], presence=pres, frequency=freq, bias=bias)
        g = BProbe("g", raw, ids, vals, seen=seen, pen=pen, counts=counts, pres=pres, freq=freq).ref()
        assert g.g_allowed.tolist() == [int(torch_ref.sample_reference(*args, 0.0, 1.0, pen, **kw)[0])], i
        ref = BProbe("s", raw, ids, vals, seen=seen, pen=pen, counts=counts, pres=pres, freq=freq, temp=temp,
                     top_p=top_p).ref()
        if (ref.must != ref.may).any():
            continue
        checked += 1
        n = 4000
        kw4 = dict(kw, counts=kw["counts"].repeat(n, 1))
        drawn = set(torch_ref.sample_reference(args[0].repeat(n, 1), args[1].repeat(n, 1), temp, top_p, pen,
                                               torch.Generator().manual_seed(i), **kw4).tolist())
        assert drawn <= set(np.nonzero(ref.must)[0].tolist()), i
        assert set(np.nonzero(ref.must & (ref.e > 0.01 * ref.T_must))[0].tolist()) <= drawn, i
    assert checked >= 10


def test_capped_bias_is_rowref_of_the_shifted_logit():
    """cap tanh(l' / cap) reproduces cap tanh(l / cap) + b to far below the soft-cap error bound"""
    rng = np.random.default_rng(2)
    p = make_bprobe("bc_sampled", 32000, 4, 0, rng)
    ids, vals = p.used()
    ref = p.ref(SOFTCAP)
    want = SOFTCAP * np.tanh(p.raw.astype(np.float64) / SOFTCAP)
    want[ids] += vals
    assert np.abs(ref.l - want).max() < SOFTCAP * 2.0 ** -16


@pytest.mark.parametrize("V,cs", [(32000, 1), (32000, 8), (128256, 4), (151936, 8)])
def test_aimed_draws_allow_exactly_one_token(V, cs):
    """every aimed draw allows exactly its token, every sampled probe gets aims, every greedy probe allows exactly its
    expected token, and the exact rule stays inside the allowed set"""
    aimed = {}
    for variants, cap in ((BVARIANTS, 0.0), (CAP_VARIANTS, SOFTCAP)):
        L = BLaunch(V, cs, 2 * len(variants), variants, cap=cap, rounds=3, seed=V + cs)
        for t in range(3):
            for p, ref, d in zip(L.probes, L.refs, L.draws[t]):
                u, allowed, aim = d
                if aim is not None:
                    assert allowed.tolist() == [aim], (p.name, t, aim, allowed[:8])
                    aimed[p.name] = aimed.get(p.name, 0) + 1
                if p.expect is not None:
                    assert allowed.tolist() == [p.expect], (p.name, allowed[:8])
                assert ref.point(u) in allowed, (p.name, t)
    for name in BVARIANTS + CAP_VARIANTS:
        if name not in ("b_up", "b_down", "b_ban_greedy", "b_seen_sign", "bc_greedy"):
            assert aimed.get(name, 0) > 0, name


def test_greedy_probes_need_the_bias():
    """without the bias the greedy probes would return another token (the bias is what the probe checks)"""
    rng = np.random.default_rng(8)
    for name, i in (("b_up", 0), ("b_down", 1), ("b_ban_greedy", 2), ("b_seen_sign", 4), ("b_force", 5)):
        p = make_bprobe(name, 32000, 2, i, rng)
        assert p.expect is not None
        plain = PenRef(p.raw, p.seen, None, temp=0.0, pen=p.pen)
        assert plain.g_allowed.tolist() != [p.expect], (name, i)


@pytest.mark.parametrize("mutant,names", [("after_pen", ("b_seen_sign", "b_pf")),
                                          ("every_id", ("b_ban_greedy", "b_ban_sampled", "b_edges"))])
def test_probe_catches_reference_mutant(mutant, names):
    """biasing after the penalties, or adding the bias to every id, leaves the allowed set on some probe"""
    V, cs, B = 32000, 4, 10
    L = BLaunch(V, cs, B, names, rounds=len(STEPS), seed=11)
    hits = 0
    for t in range(len(L.steps)):
        for p, ref, d in zip(L.probes, L.refs, L.draws[t]):
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


def _run(L, tag, row_map=False):
    """every round of L through ``sample`` with the launch's bias tables; checks tokens and identical bytes on a
    repeat of the first round"""
    ops, dev = _ops(), "cuda"
    logits = torch.from_numpy(L.logits).to(dev)
    st = {k: torch.from_numpy(getattr(L, k)).to(dev)
          for k in ("temp", "top_p", "pen", "top_k", "min_p", "pres", "freq", "bias_ids", "bias_vals", "bias_n")}
    rm = torch.from_numpy(L.row_map.astype(np.int32)).to(dev)
    out = torch.empty(L.n_state, dtype=torch.int32, device=dev)
    bad, outs = [], []
    for t, step in enumerate(L.steps):
        reps = []
        for _ in range(2 if t == 0 else 1):
            out.fill_(-1)
            ops.sample(logits, out, seen=torch.from_numpy(L.seen).to(dev), temperature=st["temp"], top_p=st["top_p"],
                       rep_penalty=st["pen"], top_k=st["top_k"], min_p=st["min_p"], seeds=_i32(L.seeds[t]),
                       step=_step(step), softcap=L.cap, counts=torch.from_numpy(L.counts).to(dev),
                       presence=st["pres"], frequency=st["freq"], bias_ids=st["bias_ids"], bias_vals=st["bias_vals"],
                       bias_n=st["bias_n"], row_map=rm.data_ptr() if row_map else 0)
            reps.append(out.cpu().numpy().copy())
        if len(reps) == 2:
            assert np.array_equal(reps[0], reps[1]), f"{tag}: two identical launches differ"
        bad += L.check(t, reps[0], f"{tag} step {step:#x}")
        outs.append(reps[0])
    return outs, bad


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_bias_matches_ref_at_every_cluster_size(V):
    """every bias probe at every cluster size V reaches, and a soft-capped launch at the largest"""
    bad = []
    cases = cluster_cases(V)
    for cs, B in sorted(cases.items()):
        L = BLaunch(V, cs, B, BVARIANTS, seed=V + cs, offset=(V // 11 + 5 * cs) % len(BVARIANTS))
        bad += _run(L, f"V={V} cs={cs} B={B}")[1]
    cs = max(cases)
    L = BLaunch(V, cs, cases[cs], CAP_VARIANTS, cap=SOFTCAP, rounds=4, seed=V + 100 + cs)
    bad += _run(L, f"V={V} cs={cs} softcap")[1]
    print("\nerr/bound per probe: " + "  ".join(f"{k}={v:.3f}" for k, v in sorted(MEASURED.items())))
    assert not bad, f"{len(bad)} failures:\n" + "\n".join(bad[:12])


@gpu
def test_row_map_mixes_biased_and_plain_rows():
    """one launch through row_map with skipped rows, rows whose bias is off (junk in their tables) and junk tables in
    the state rows no logits row maps to"""
    V, B, S = 128256, 12, 17
    row_map = np.array([5, 0, 16, 2, -1, 7, 1, 12, 3, -1, 9, 14])
    cs = int(_ops().native().sample_cluster_size(B, V))
    L = BLaunch(V, cs, B, BVARIANTS, rounds=4, seed=21, row_map=row_map, n_state=S, plain=(1, 5, 8, 11))
    outs, bad = _run(L, "row_map", row_map=True)
    free = [r for r in range(S) if r not in set(int(x) for x in row_map if x >= 0)]
    assert all((o[free] == -1).all() for o in outs)
    assert not bad, "\n".join(bad[:12])


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_zero_bias_counts_change_nothing(V):
    """bias_n = 0 with junk tables gives the tokens of the launch without the tables, on the plain sampler probes, at
    every cluster size"""
    ops, dev = _ops(), "cuda"
    rng = np.random.default_rng(V)
    for cs, B in sorted(cluster_cases(V).items()):
        L = Launch(V, cs, B, VARIANTS, rounds=3, seed=V + 7 * cs)
        logits = torch.from_numpy(L.logits).to(dev)
        temp, top_p, pen = (torch.from_numpy(a).to(dev) for a in (L.temp, L.top_p, L.pen))
        ids = torch.from_numpy(rng.integers(0, V, (L.n_state, WIDTH)).astype(np.int32)).to(dev)
        vals = torch.from_numpy(rng.uniform(-100, 100, (L.n_state, WIDTH)).astype(np.float32)).to(dev)
        zero = torch.zeros(L.n_state, dtype=torch.int32, device=dev)
        bad = []
        for t, step in enumerate(L.steps):
            res = []
            for kw in ({}, dict(bias_ids=ids, bias_vals=vals, bias_n=zero)):
                out = torch.full((L.n_state,), -1, dtype=torch.int32, device=dev)
                ops.sample(logits, out, seen=torch.from_numpy(L.seen).to(dev), temperature=temp, top_p=top_p,
                           rep_penalty=pen, seeds=_i32(L.seeds[t]), step=_step(step), **kw)
                res.append(out.cpu().numpy())
            assert np.array_equal(res[0], res[1]), f"V={V} cs={cs} step {step:#x}"
            bad += L.check(t, res[0], f"V={V} cs={cs} step {step:#x}")
        assert not bad, "\n".join(bad[:12])


@gpu
def test_refused_bias_tensors():
    """wrong dtype, device, layout, row count or width, and an incomplete set of tables, are refused before any
    launch"""
    ops, dev = _ops(), "cuda"
    V, B, W = 1000, 4, 16
    logits = torch.randn(B, V, device=dev)
    temp = torch.ones(B, device=dev)
    out = torch.full((B,), -5, dtype=torch.int32, device=dev)
    ids, vals = ops.logit_bias_table(B, W, dev)
    n = torch.zeros(B, dtype=torch.int32, device=dev)
    good = dict(bias_ids=ids, bias_vals=vals, bias_n=n)
    bad_calls = [dict(good, bias_ids=ids.long()), dict(good, bias_vals=vals.double()), dict(good, bias_n=n.float()),
                 dict(good, bias_ids=ids.cpu()), dict(good, bias_vals=vals.cpu()), dict(good, bias_n=n.cpu()),
                 dict(good, bias_ids=torch.zeros(W, B, dtype=torch.int32, device=dev).t()),       # column-major
                 dict(good, bias_vals=torch.zeros(B, 2 * W, device=dev)[:, ::2]),                 # strided rows
                 dict(good, bias_ids=ids[:B - 1], bias_vals=vals[:B - 1]),                        # too few rows
                 dict(good, bias_n=torch.zeros(B + 1, dtype=torch.int32, device=dev)),
                 dict(good, bias_vals=torch.zeros(B, W + 4, device=dev)),                        # widths differ
                 dict(good, bias_ids=ids.reshape(-1), bias_vals=vals.reshape(-1)),                # 1-D tables
                 dict(bias_ids=ids, bias_vals=vals), dict(bias_n=n), dict(bias_ids=ids, bias_n=n)]
    for kw in bad_calls:
        with pytest.raises(RuntimeError):
            ops.sample(logits, out, temperature=temp, **kw)
    torch.cuda.synchronize()
    assert (out == -5).all()
    ops.sample(logits, out, temperature=temp, **good)
    torch.cuda.synchronize()
    assert (out >= 0).all()


# --------------------------------------------------------------------------- GPU: the engine
def _engine(max_batch=4, **kw):
    from bee2bee_b200.engine.core import Engine
    return Engine("tiny-llama", device="cuda:0", max_batch=max_batch, max_seq_len=256, decode_burst=4, **kw)


def _greedy(**kw):
    from bee2bee_b200.engine.core import SamplingParams
    return SamplingParams(max_new_tokens=12, temperature=0.0, top_p=1.0, repetition_penalty=1.0, ignore_eos=True,
                          **kw)


@gpu
def test_engine_forces_and_bans_tokens():
    """greedy with {t: +100} and the penalties off generates t every step (also when t is the last id); {g: -100} on
    the unbiased first token g changes the first token"""
    eng = _engine()
    try:
        V = eng.cfg.vocab_size
        prompt = [1, 5, 9, 33, 2, 7]
        plain = eng.generate([prompt], _greedy())[0]
        for t in (17, V - 1, 0):
            assert eng.generate([prompt], _greedy(logit_bias={t: 100.0}))[0] == [t] * 12, t
        g = plain[0]
        banned = eng.generate([prompt], _greedy(logit_bias={g: -100.0}))[0]
        assert banned[0] != g
        with pytest.raises(ValueError):
            eng.submit(prompt, _greedy(logit_bias={V: 1.0}))
    finally:
        eng.close()


@gpu
def test_engine_biased_neighbour_and_reused_slot_leave_plain_requests_unchanged():
    """a plain request decoding beside a biased one gets the tokens it gets beside a plain one; a slot freed by a
    biased request and taken by a plain one carries no bias (prefill and decode)"""
    prompts = ([1, 5, 9, 33, 2, 7], [4, 4, 19, 4, 4])
    outs = []
    for bias in ({}, {3: 9.0, 40: -100.0, 200: 100.0}):
        eng = _engine()
        try:
            from bee2bee_b200.engine.core import SamplingParams
            ra = eng.submit(prompts[0], SamplingParams(max_new_tokens=16, temperature=0.8, ignore_eos=True, seed=1))
            rb = eng.submit(prompts[1], _greedy(logit_bias=bias))
            while not (ra.done.is_set() and rb.done.is_set()):
                eng.step()
        finally:
            eng.close()
        assert ra.error is None and rb.error is None
        outs.append((list(ra.out_ids), list(rb.out_ids)))
    assert outs[0][0] == outs[1][0]
    assert outs[1][1] == [200] * 12 and outs[0][1] != outs[1][1]

    eng = _engine(max_batch=1, prefix_cache=False)       # every request prefills its whole prompt
    try:
        plain = eng.generate([prompts[1]], _greedy())[0]
        assert eng.generate([prompts[1]], _greedy(logit_bias={200: 100.0}))[0] == [200] * 12
        assert int(eng.runner.sampler_i32[2, 0]) == 1
        assert eng.generate([prompts[1]], _greedy())[0] == plain
        assert int(eng.runner.sampler_i32[2, 0]) == 0
    finally:
        eng.close()
