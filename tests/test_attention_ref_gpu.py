"""Both paged-attention kernels against a plain fp64 reference, with inputs that turn a one-key mask error into an O(1)
change of the output.

Random q / K / V give diffuse attention: including or dropping one key of n moves the output by about |v| / n, far
inside any bf16 tolerance.  The probe inputs here put, for every query row, one target key ~17 nats above all others
(``q = b * u_t``, ``K[j] = a * u_j``, a * b = 32), so the output is ~V[t] when the target is visible and something else
when it is masked.  Probe kinds (t(p) = target of the query at absolute position p, w = window):

    diag      t = p                          visible
    future    t = p + 1                      masked (the last query's target is the slot at kv_len)
    win_in    t = p - w + 1                  visible
    win_out   t = p - w                      masked
    first     t = max(0, p - w + 1) or 0     visible; often a tile other rows of the block cannot see
    ramp_up   each 64-key tile's max beats the previous one by 8 nats: a lazy rescale on every tile
    ramp_down the maximum sits in the first visible tile
    random    plain random q / K / V
    softcap   random scores of +-40 (cap 5) or +-120 (cap 50): tanh saturates
    split_edge  (split-KV decode) head g targets the first or last key of one split's share of the tiles

Every cache slot no sequence may see holds finite poison whose score beats every probe (K[0] = 1024 against q[0] = 1)
and whose value is 64; gap and inactive q rows hold finite garbage; the split-KV workspace is NaN before each call;
``out`` starts as a sentinel that every row the call must not write keeps, bit for bit.

Error model (``tolerance``): the reference reads the same bf16 q / K / V in fp64, so the kernels' errors are
  * the bf16 rounding of the output: <= 2^-8 |out| per element;
  * on the tensor-core kernel, the bf16 rounding of P before the PV product.  The row sum l uses the unrounded P, so the
    error is sum_j (p~_j - p_j) v_j / l <= 2^-8 max|v_visible|, i.e. c = 2 in units of 2^-9;
  * fp32 scores, exp and accumulation: relative ~1e-5 at the largest scores used here (256), far below one 2^-9 unit.
The CUDA-core kernel keeps P in fp32, so it gets c = 1; the tensor-core kernel c = 2.

The CPU tests at the top pin the reference against SDPA and prove that every probe separates its mask mutant by at
least 20x the tolerance."""
from __future__ import annotations

import math
from collections import defaultdict

import pytest
import torch

gpu = pytest.mark.gpu

PAGE = 64                 # tokens per KV page (csrc/attention.cu)
A_K, B_Q = 8.0, 4.0       # probe key / query norms: target score a * b = 32 (x cos 0.97 from the per-head jitter)
POISON_K0 = 1024.0        # K[0] of every slot no sequence may see; every active q row has q[0] = 1
POISON_V = 64.0
SENTINEL = -7.5           # out rows the call must not write keep this value
RAMP_STEP = 4.0           # ramp_up: K[1] = RAMP_STEP * tile against q[1] = 2 -> +8 nats per tile (> 8 ln 2 = 5.55)
C_TC, C_CC = 2.0, 1.0     # the error model's c (units of 2^-9 max|v_visible|) per kernel
MASK_KINDS = ("diag", "future", "win_in", "win_out", "first")
KINDS = MASK_KINDS + ("ramp_up", "ramp_down", "random", "softcap")
KV_LENS = (1, 63, 64, 65, 128, 129, 1000, 2049)

# measured max(|out - ref| / bound) per (kernel, probe kind), printed at the end of each GPU test (pytest -s shows it)
MEASURED: dict = defaultdict(float)


# --------------------------------------------------------------------------- fp64 reference
def attn_ref64(q, kc, vc, bt, q_start, q_len, kv_len, n_kv, window=0, cap=0.0, *, causal_shift=0, window_shift=0,
               kvlen_shift=0, apply_cap=True):
    """The kernels' stated semantics in fp64.  q [T, n_q, D] (pre-scaled), K/V cache [pages, 64, n_kv, D], block table
    [seqs, max_pages]; q_start / q_len / kv_len are int lists.  Key kvpos is visible to the query at
    qpos = kv_len - q_len + i iff kvpos <= qpos, kvpos < kv_len and (window <= 0 or kvpos > qpos - window); scores are
    q.k, then cap * tanh(s / cap), then the mask, softmax, PV.  A row that sees no key is 0.  The keyword arguments
    mutate the mask (for the discrimination checks).  Returns (out [T, n_q, D] fp64, zero where no row is written,
    written [T] bool, vmax [T, n_q] = max |v| over the keys the row sees)."""
    T, n_q, D = q.shape
    G = n_q // n_kv
    out = torch.zeros(T, n_q, D, dtype=torch.float64, device=q.device)
    vmax = torch.zeros(T, n_q, dtype=torch.float64, device=q.device)
    written = torch.zeros(T, dtype=torch.bool, device=q.device)
    w = window + window_shift if window > 0 else 0
    for s, (q0, ql, kl) in enumerate(zip(q_start, q_len, kv_len)):
        if ql <= 0:
            continue
        written[q0:q0 + ql] = True
        pages = bt[s].long()
        kpos = torch.arange(pages.numel() * PAGE, device=q.device)
        qpos = torch.arange(kl - ql, kl, device=q.device)[:, None]
        vis = (kpos[None] <= qpos + causal_shift) & (kpos[None] < kl + kvlen_shift)
        if w > 0:
            vis &= kpos[None] > qpos - w
        for h in range(n_kv):
            k = kc[pages, :, h].reshape(-1, D).double()
            v = vc[pages, :, h].reshape(-1, D).double()
            qq = q[q0:q0 + ql, h * G:(h + 1) * G].double()                 # [ql, G, D]
            sc = torch.einsum("igd,jd->igj", qq, k)
            if cap > 0 and apply_cap:
                sc = cap * torch.tanh(sc / cap)
            sc = sc.masked_fill(~vis[:, None, :], float("-inf"))
            p = torch.softmax(sc, -1).nan_to_num(0.0)                        # no visible key -> 0
            out[q0:q0 + ql, h * G:(h + 1) * G] = torch.einsum("igj,jd->igd", p, v)
            vrow = v.abs().amax(-1)
            vmax[q0:q0 + ql, h * G:(h + 1) * G] = torch.where(vis, vrow[None], 0.0).amax(-1)[:, None]
    return out, written, vmax


def tolerance(ref, vmax, c):
    """per-element bound 2^-8 |ref| + c 2^-9 max|v_visible| (see the module docstring)"""
    return 2.0 ** -8 * ref.abs() + c * 2.0 ** -9 * vmax[..., None]


# --------------------------------------------------------------------------- probe inputs
class Case:
    """One batch of probe inputs: paged K/V cache with poison, block table, ragged q with garbage gap rows.
    ``targets(seq, pos)`` gives the split_edge kind's target keys."""

    def __init__(self, seqs, G, n_kv, D, kind, window=0, cap=0.0, seed=0, targets=None):
        self.G, self.n_kv, self.D, self.window, self.cap, self.kind = G, n_kv, D, window, cap, kind
        self.n_q = n_q = G * n_kv
        self.q_len = [ql for ql, _ in seqs]
        self.kv_len = [kl for _, kl in seqs]
        gen = torch.Generator().manual_seed(seed)
        rnd = lambda *shape: torch.randn(*shape, generator=gen)  # noqa: E731
        S = len(seqs)

        # token rows: a gap of s % 3 rows before each sequence, one own (never written) row for a q_len == 0 sequence,
        # two rows past the last sequence
        self.q_start, row = [], 0
        for ql, _ in seqs:
            row += len(self.q_start) % 3
            self.q_start.append(row)
            row += max(ql, 1)
        self.T = T = row + 2

        # pages: the block table covers the slot at kv_len too (the mutated kv_len mask reads it); entries past a
        # sequence's last page point to a shared poison page; a few more pages belong to no sequence at all
        self.max_pages = max(kl // PAGE + 1 for kl in self.kv_len) + 1
        own = [(kl + PAGE - 1) // PAGE for kl in self.kv_len]
        n_pages = 1 + sum(own) + 3
        perm = torch.randperm(n_pages, generator=gen).int()
        bt = torch.full((S, self.max_pages), int(perm[0]), dtype=torch.int32)
        nxt = 1
        for s, n in enumerate(own):
            bt[s, :n] = perm[nxt:nxt + n]
            nxt += n
        self.bt = bt
        kc = torch.zeros(n_pages, PAGE, n_kv, D)
        kc[..., 0] = POISON_K0
        vc = torch.full((n_pages, PAGE, n_kv, D), POISON_V)
        q = rnd(T, n_q, D) * 4.0                                     # finite garbage in every row no sequence owns
        for s, (ql, kl) in enumerate(seqs):
            K, V, Q = self._fill(kind, ql, kl, rnd, s, targets)
            pos = torch.arange(kl)
            slot = (bt[s, pos // PAGE].long() * PAGE + pos % PAGE)
            kc.view(-1, n_kv, D)[slot] = K
            vc.view(-1, n_kv, D)[slot] = V
            if ql > 0:
                q[self.q_start[s]:self.q_start[s] + ql] = Q
        self.q, self.kc, self.vc = q.to(torch.bfloat16), kc.to(torch.bfloat16), vc.to(torch.bfloat16)

    def _fill(self, kind, ql, kl, rnd, s, targets):
        G, n_kv, D, w = self.G, self.n_kv, self.D, self.window
        V = rnd(kl, n_kv, D)
        Q = torch.zeros(ql, n_kv, G, D)
        if kind in MASK_KINDS or kind == "split_edge":
            u = rnd(kl + 1, n_kv, D)
            u[..., 0] = 0.0
            u = u / u.norm(dim=-1, keepdim=True)
            K = A_K * u[:kl] + 0.02 * rnd(kl, n_kv, D)
            K[..., 0] = 0.0
            pos = torch.arange(kl - ql, kl)[:, None].expand(ql, G)
            tgt = targets(s, pos) if kind == "split_edge" else probe_target(kind, pos, kl, w)
            jit = rnd(ql, n_kv, G, D) / math.sqrt(D)                   # per-head jitter: heads of a group differ
            jit[..., 0] = 0.0
            for h in range(n_kv):
                d = u[tgt, h] + 0.25 * jit[:, h]                          # [ql, G, D]
                Q[:, h] = B_Q * d / d.norm(dim=-1, keepdim=True)
        elif kind in ("ramp_up", "ramp_down"):
            tile = (torch.arange(kl) // PAGE).float()
            K = 0.3 * rnd(kl, n_kv, D)
            K[..., 0] = 0.0
            K[..., 1] = (RAMP_STEP * tile if kind == "ramp_up" else -tile)[:, None]
            Q = rnd(ql, n_kv, G, D) / math.sqrt(D)
            Q[..., 1] = 2.0
        elif kind == "random":
            K = rnd(kl, n_kv, D)
            K[..., 0] = 0.0
            Q = 0.3 * rnd(ql, n_kv, G, D)
        elif kind == "softcap":
            std = 40.0 if self.cap <= 5.0 else 120.0                   # score std: tanh saturates at either cap
            a = math.sqrt(std / math.sqrt(D - 1))
            K = a * rnd(kl, n_kv, D)
            K[..., 0] = 0.0
            Q = a * rnd(ql, n_kv, G, D)
        else:
            raise ValueError(kind)
        Q[..., 0] = 1.0
        return K, V, Q.reshape(ql, n_kv * G, D)

    def ref(self, **mut):
        return attn_ref64(self.q, self.kc, self.vc, self.bt, self.q_start, self.q_len, self.kv_len, self.n_kv,
                          self.window, self.cap, **mut)

    def to(self, device):
        for name in ("q", "kc", "vc", "bt"):
            setattr(self, name, getattr(self, name).to(device))
        return self


def probe_target(kind, pos, kl, w):
    """target key of the query at absolute position ``pos`` (see the module docstring); rows for which the kind has
    no target of its own (win_* before the window reaches key 0) fall back to the diagonal or the future key"""
    if kind == "diag":
        return pos
    if kind == "future":
        return pos + 1
    if kind == "first":
        return (pos - w + 1).clamp(min=0) if w > 0 else torch.zeros_like(pos)
    if kind == "win_in":
        return torch.where(pos - w + 1 >= 0, pos - w + 1, pos) if w > 0 else pos
    if kind == "win_out":
        return torch.where(pos - w >= 0, pos - w, pos + 1) if w > 0 else pos + 1
    raise ValueError(kind)


def split_ranges(kernel, kl, window, splits):
    """[first key, last key] of every non-empty split share of a decode query's tiles, by the kernel's partition"""
    kv_lo = max(0, kl - window) if window > 0 else 0
    t_lo, t_hi = kv_lo // PAGE, (kl + PAGE - 1) // PAGE
    nt = t_hi - t_lo
    out = []
    for k in range(splits):
        if kernel == "tc":
            per = (nt + splits - 1) // splits
            a = min(t_hi, t_lo + k * per)
            b = min(t_hi, a + per)
        else:
            a, b = t_lo + nt * k // splits, t_lo + nt * (k + 1) // splits
        if b > a:
            out.append((max(a * PAGE, kv_lo), min(b * PAGE, kl) - 1))
    return out


# --------------------------------------------------------------------------- CPU: the reference and the probes
def _sdpa_ref(case):
    """the same attention through torch SDPA (fp64, explicit boolean mask, K/V gathered per sequence)"""
    F = torch.nn.functional
    out = torch.zeros(case.T, case.n_q, case.D, dtype=torch.float64)
    for s, (q0, ql, kl) in enumerate(zip(case.q_start, case.q_len, case.kv_len)):
        if ql == 0:
            continue
        k = case.kc[case.bt[s].long()].reshape(-1, case.n_kv, case.D)[:kl].double()
        v = case.vc[case.bt[s].long()].reshape(-1, case.n_kv, case.D)[:kl].double()
        k = k.repeat_interleave(case.G, 1).transpose(0, 1)
        v = v.repeat_interleave(case.G, 1).transpose(0, 1)
        qq = case.q[q0:q0 + ql].double().transpose(0, 1)
        qpos = torch.arange(kl - ql, kl)[:, None]
        kpos = torch.arange(kl)[None]
        m = kpos <= qpos
        if case.window > 0:
            m &= kpos > qpos - case.window
        out[q0:q0 + ql] = F.scaled_dot_product_attention(qq, k, v, attn_mask=m, scale=1.0).transpose(0, 1)
    return out


@pytest.mark.parametrize("G,n_kv,D,window,seqs", [
    (1, 2, 64, 0, [(5, 70), (3, 3), (1, 130)]),
    (4, 2, 64, 20, [(17, 80), (0, 40), (2, 200)]),
    (3, 1, 128, 0, [(40, 40), (9, 129)]),
    (2, 3, 64, 65, [(64, 300), (1, 1), (30, 64)]),
])
def test_ref64_matches_sdpa(G, n_kv, D, window, seqs):
    case = Case(seqs, G, n_kv, D, "random", window=window, seed=1)
    ref, written, _ = case.ref()
    exp = _sdpa_ref(case)
    assert written.sum().item() == sum(case.q_len)
    assert torch.allclose(ref, exp, rtol=1e-10, atol=1e-10), (ref - exp).abs().max()


# (probe kind, window, mask mutation, rows the mutation must expose)
_MUTANTS = [
    ("diag", 0, dict(causal_shift=-1), "all"),
    ("diag", 20, dict(causal_shift=-1), "all"),
    ("future", 0, dict(causal_shift=1, kvlen_shift=1), "all"),
    ("future", 20, dict(causal_shift=1, kvlen_shift=1), "all"),
    ("win_in", 20, dict(window_shift=-1), "windowed"),
    ("win_out", 20, dict(window_shift=1), "windowed"),
    ("first", 20, dict(window_shift=-1), "windowed"),
    ("win_in", 64, dict(window_shift=-1), "windowed"),
    ("win_out", 64, dict(window_shift=1), "windowed"),
    ("softcap", 0, dict(apply_cap=False), "long"),
]
# the mask probes run uncapped and at cap 50 (a cap of 5 bends every probe score to within 10 nats, so the soft-cap
# probe covers it); the soft-cap probe at caps 5 and 50
_MUTANT_CASES = [(k, w, m, r, c) for k, w, m, r in _MUTANTS for c in ((5.0, 50.0) if k == "softcap" else (0.0, 50.0))]


@pytest.mark.parametrize("kind,window,mut,rows,cap", _MUTANT_CASES,
                         ids=[f"{k}-w{w}-{'-'.join(m)}-cap{int(c)}" for k, w, m, _, c in _MUTANT_CASES])
def test_probe_discriminates_mask_mutant(kind, window, mut, rows, cap):
    """the correct reference and a one-key mask mutant differ by >= 20x the (loosest) tolerance on every probed row"""
    seqs = [(5, 70), (1, 1), (3, 3), (1, 130), (70, 200), (0, 50), (4, 64), (2, 2049)]
    case = Case(seqs, 2, 2, 64, kind, window=window, cap=cap, seed=3)
    ref, written, vmax = case.ref()
    mref, _, _ = case.ref(**mut)
    ratio = ((mref - ref).abs() / tolerance(ref, vmax, C_TC)).amax(dim=(1, 2))   # per row
    probed = 0
    for s, (q0, ql, kl) in enumerate(zip(case.q_start, case.q_len, case.kv_len)):
        for i in range(ql):
            p = kl - ql + i
            if rows == "windowed" and p - window < 0:
                continue
            if rows == "long" and min(p + 1, window or p + 1) < 32:
                continue
            probed += 1
            assert ratio[q0 + i] >= 20.0, (s, i, p, ratio[q0 + i].item())
    assert probed >= 20


def test_probe_scores_single_out_the_target():
    """a * b = 32 at D = 64: over 2049 keys the target's score beats every other visible key by > 10 nats"""
    case = Case([(3, 2049), (64, 1000)], 2, 1, 64, "diag", seed=5)
    for s, (q0, ql, kl) in enumerate(zip(case.q_start, case.q_len, case.kv_len)):
        k = case.kc[case.bt[s].long()].reshape(-1, 64)[:kl].double()
        sc = case.q[q0:q0 + ql].double() @ k.T                                       # [ql, G, kl]
        pos = torch.arange(kl - ql, kl)
        top = sc[torch.arange(ql), :, pos]                                             # [ql, G]
        vis = torch.arange(kl)[None] <= pos[:, None]
        other = sc.masked_fill(~vis[:, None] | (torch.arange(kl)[None, None] == pos[:, None, None]), -1e9).amax(-1)
        assert (top - other).min() > 10.0, (top - other).min()


def test_ramp_inputs_force_a_rescale_on_every_tile():
    """ramp_up: every visible 64-key tile's max beats the previous tile's by more than 8 ln 2 nats, the tensor-core
    kernel's lazy-rescale threshold (2^8 in the exp2 domain); ramp_down: the maximum sits in the first visible tile"""
    for kind in ("ramp_up", "ramp_down"):
        case = Case([(3, 2049), (70, 200), (1, 129)], 2, 1, 64, kind, window=0, seed=7)
        for s, (q0, ql, kl) in enumerate(zip(case.q_start, case.q_len, case.kv_len)):
            k = case.kc[case.bt[s].long()].reshape(-1, 64)[:kl].double()
            sc = case.q[q0:q0 + ql].double() @ k.T
            for i in range(ql):
                p = kl - ql + i
                tmax = torch.stack([sc[i, :, t * PAGE:min(p + 1, (t + 1) * PAGE)].amax(-1) for t in range(p // PAGE + 1)])
                if tmax.shape[0] < 2:
                    continue
                if kind == "ramp_up":
                    assert (tmax[1:] - tmax[:-1]).min() > 8 * math.log(2), (s, i)
                else:
                    assert (tmax[0] > tmax[1:]).all(), (s, i)


def test_poison_fills_every_slot_no_sequence_sees():
    """slots past kv_len, pages outside every block table and the page of the unused block-table entries hold poison;
    the block table holds no out-of-range or negative entry"""
    case = Case([(5, 70), (0, 64), (1, 129)], 2, 2, 64, "diag", seed=9)
    n_pages = case.kc.shape[0]
    assert case.bt.min() >= 0 and case.bt.max() < n_pages
    seen = torch.zeros(n_pages, PAGE, dtype=torch.bool)
    for s, kl in enumerate(case.kv_len):
        pos = torch.arange(kl)
        seen[case.bt[s, pos // PAGE].long(), pos % PAGE] = True
    assert (case.kc[~seen][..., 0] == POISON_K0).all() and (case.vc[~seen] == POISON_V).all()
    assert (case.kc[seen][..., 0] == 0).all()


# --------------------------------------------------------------------------- GPU: kernels against the reference
def _ops():
    from bee2bee_b200 import ops
    return ops


def run_kernel(kernel, case, *, splits=1, decode=False, fill_ws=True):
    """one attention call on ``kernel``: "tc" = tensor-core (default dispatch for prefill, use_tc=1 for decode), "cc" =
    CUDA-core (tc_min_q 0 for prefill, use_tc=0 for decode), "auto" = the default dispatch"""
    ops = _ops()
    dev = case.q.device
    out = torch.full((case.T, case.n_q * case.D), SENTINEL, dtype=torch.bfloat16, device=dev)
    i32 = lambda xs: torch.tensor(xs, dtype=torch.int32, device=dev)  # noqa: E731
    max_q = max(case.q_len)
    ws = None
    if splits > 1:
        R = _attn_rows(case.G)
        ws = torch.full((len(case.q_len) * case.n_kv * splits * R * (case.D + 2),), float("nan"), device=dev)
    kw = dict(max_q=max_q, n_q=case.n_q, n_kv=case.n_kv, head_dim=case.D, window=case.window, softcap=case.cap,
              splits=splits, ws=ws)
    args = (case.q.view(case.T, -1), case.kc, case.vc, out, case.bt, i32(case.q_start), i32(case.q_len),
            i32(case.kv_len))
    if decode:
        ops.attention(*args, use_tc={"tc": 1, "cc": 0, "auto": -1}[kernel], **kw)
    elif kernel == "cc":
        old = ops.get_attn_tc_min_q()
        ops.set_attn_tc_min_q(0)
        try:
            ops.attention(*args, **kw)
        finally:
            ops.set_attn_tc_min_q(old)
    else:
        if kernel == "tc":
            assert 0 < ops.get_attn_tc_min_q() <= max_q
        ops.attention(*args, **kw)
    torch.cuda.synchronize()
    return out.view(case.T, case.n_q, case.D)


def _attn_rows(G):
    """rows of one decode CTA's workspace partial (attn_rows(G, 1) in csrc/attention.cu)"""
    r = (G + 3) // 4 * 4
    return next(x for x in (4, 8, 16, 32, 64) if r <= x)


def check_case(kernel, case, out, tag):
    """out matches the reference within the error model, rows the call must not write keep the sentinel"""
    ref, written, vmax = case.ref()
    o = out.double()
    assert torch.isfinite(o[written]).all(), f"{tag}: non-finite output"
    untouched = out[~written]
    assert (untouched == SENTINEL).all(), f"{tag}: wrote {(untouched != SENTINEL).any(-1).any(-1).sum().item()} rows it does not own"
    bound = tolerance(ref, vmax, C_TC if kernel == "tc" else C_CC)
    ratio = ((o - ref).abs() / bound)[written]
    worst = ratio.max().item()
    key = (kernel, case.kind)
    MEASURED[key] = max(MEASURED[key], worst)
    if worst > 1.0:
        idx = (ratio == ratio.max()).nonzero()[0].tolist()
        rows = written.nonzero()[:, 0]
        t = rows[idx[0]].item()
        raise AssertionError(f"{tag}: |out - ref| / bound = {worst:.3f} at token {t}, head {idx[1]}, dim {idx[2]}: "
                             f"out {o[t, idx[1], idx[2]].item():.5f} ref {ref[t, idx[1], idx[2]].item():.5f}")


def _report(kernel):
    print("\n" + "  ".join(f"{k[0]}/{k[1]}={v:.3f}" for k, v in sorted(MEASURED.items()) if k[0] == kernel))


def _qb(kernel, G, D):
    """query rows per CTA block: 128 / G on the tensor-core kernel, 64 / G (32 / G at D = 256) on the CUDA-core one"""
    return 128 // G if kernel == "tc" else (32 if D == 256 else 64) // G


def _prefill_cases():
    cases = []
    windows = (0, 1, 63, 64, 65, 100, 5000)
    i = 0
    for kernel in ("tc", "cc"):
        for G in (1, 2, 4, 8, 16):
            for D in (64, 128, 256):
                cases.append((kernel, G, D, windows[i % len(windows)], (0.0, 50.0)[(i // 2) % 2], i))
                i += 1
    for G, D in ((3, 64), (5, 128), (7, 256), (12, 128)):            # groups the tensor-core kernel refuses
        cases.append(("auto", G, D, windows[i % len(windows)], (0.0, 50.0)[i % 2], i))
        i += 1
    return cases


@gpu
@pytest.mark.parametrize("kernel,G,D,window,cap,idx", _prefill_cases(),
                         ids=[f"{k}-G{g}-D{d}-w{w}-cap{int(c)}" for k, g, d, w, c, _ in _prefill_cases()])
def test_prefill_probes_match_ref64(kernel, G, D, window, cap, idx):
    """ragged prefill batch: q_len QB - 1, QB and QB + 1 for this kernel's query block, a q_len == 0 sequence, a
    one-token chunk, chunks on top of cached context starting mid-page, gaps between the q_start ranges; every probe
    kind, then the random kind twice for identical bytes"""
    kern = "cc" if kernel == "auto" else kernel
    QB = _qb(kern, G, D)
    qls = [QB - 1, QB, QB + 1, 0, 1, 2 * QB + 3]
    seqs = []
    for j, ql in enumerate(qls):
        kl = KV_LENS[(idx + 3 * j) % len(KV_LENS)]
        seqs.append((ql, kl if kl >= ql else ql + 29))
    n_kv = 1 if G * D >= 2048 else 2
    for kind in KINDS:
        c = (5.0 if idx % 2 == 0 else 50.0) if kind == "softcap" else cap
        if kind in ("win_in", "win_out") and window == 0:
            continue
        case = Case(seqs, G, n_kv, D, kind, window=window, cap=c, seed=idx * 31 + KINDS.index(kind)).to("cuda")
        out = run_kernel(kernel, case)
        check_case(kern, case, out, f"{kernel} {kind}")
        if kind == "random":
            assert torch.equal(out, run_kernel(kernel, case)), "two identical calls differ"
    _report(kern)


@gpu
@pytest.mark.parametrize("kernel", ["tc", "cc"])
@pytest.mark.parametrize("G", [1, 4, 16])
@pytest.mark.parametrize("window", [65, 100, 127])
def test_window_edge_probes_match_ref64(kernel, G, window):
    """full query blocks over cached contexts of every page offset: the window's lower edge crosses tile boundaries at
    many alignments, so a tile that the first query of a block sees whole but the last does not (the tensor-core
    kernel's unpredicated-tile shortcut) is always there"""
    QB = _qb(kernel, G, 128)
    seqs = [(3 * QB, 3 * QB + ctx) for ctx in (0, 17, 64, 100, 333, 1000)]
    for kind in ("win_in", "win_out"):
        case = Case(seqs, G, 1, 128, kind, window=window, seed=window + G).to("cuda")
        check_case(kernel, case, run_kernel(kernel, case), f"{kernel} {kind}")
    _report(kernel)


def _decode_cases():
    cases = []
    i = 0
    for kernel in ("tc", "cc"):
        for splits in (1, 2, 3, 5, 16, 64):
            G = (1, 2, 4, 8, 16)[i % 5]
            D = (64, 128, 256)[i % 3]
            cases.append((kernel, G, D, splits, (0, 100, 63, 1, 65, 5000)[i % 6], (0.0, 50.0)[(i // 3) % 2]))
            i += 1
        cases.append((kernel, 16, 128, 5, 64, 50.0))                 # split-KV at G = 16
    cases += [("auto", 3, 128, 3, 100, 0.0), ("auto", 12, 64, 16, 0, 50.0), ("auto", 6, 256, 1, 65, 0.0)]
    return cases


@gpu
@pytest.mark.parametrize("kernel,G,D,splits,window,cap", _decode_cases(),
                         ids=[f"{k}-G{g}-D{d}-s{s}-w{w}-cap{int(c)}" for k, g, d, s, w, c in _decode_cases()])
def test_decode_probes_match_ref64(kernel, G, D, splits, window, cap):
    """decode (one query per sequence), split-KV with splits beyond the tile count included, an inactive sequence
    (q_len 0) whose row must keep the sentinel; with splits, heads target the first / last key of each split's share"""
    kern = "cc" if kernel == "auto" else kernel
    seqs = [(1, kl) for kl in KV_LENS] + [(0, 500)]
    n_kv = 1 if G * D >= 2048 else 2
    kinds = KINDS + (("split_edge",) if splits > 1 else ())
    for kind in kinds:
        c = (5.0 if splits % 2 else 50.0) if kind == "softcap" else cap
        if kind in ("win_in", "win_out") and window == 0:
            continue

        def edge(s, pos):
            rng = split_ranges(kern, seqs[s][1], window, splits)
            t = torch.empty_like(pos)
            for g in range(pos.shape[1]):
                a, b = rng[(g // 2 + s) % len(rng)]
                t[:, g] = a if g % 2 == 0 else b
            return t

        case = Case(seqs, G, n_kv, D, kind, window=window, cap=c, seed=splits * 7 + len(kind), targets=edge).to("cuda")
        out = run_kernel(kernel, case, splits=splits, decode=True)
        check_case(kern, case, out, f"{kernel} splits={splits} {kind}")
        if kind == "random":
            assert torch.equal(out, run_kernel(kernel, case, splits=splits, decode=True)), "two identical calls differ"
    _report(kern)


@gpu
@pytest.mark.parametrize("kernel", ["tc", "cc"])
@pytest.mark.parametrize("splits", [1, 4])
def test_split_decode_leaves_inactive_rows_alone(kernel, splits):
    """q_len == 0 sequences own no output row: with split-KV the merge pass must not write out[q_start] for them (it
    would write whatever the workspace holds, NaN here)"""
    seqs = [(1, 700), (0, 300), (1, 65), (0, 2049), (1, 1)]
    case = Case(seqs, 4, 2, 128, "random", seed=11).to("cuda")
    out = run_kernel(kernel, case, splits=splits, decode=True)
    check_case(kernel, case, out, f"{kernel} splits={splits}")


@gpu
@pytest.mark.parametrize("max_q", [15, 16])
def test_tc_min_q_switch(max_q):
    """with tc_min_q = 16 a batch of max_q 15 runs on the CUDA-core kernel and one of 16 on the tensor-core kernel:
    each output is bitwise the one of the forced kernel and matches the reference"""
    ops = _ops()
    seqs = [(max_q, 300), (5, 5), (0, 10), (max_q - 2, 129)]
    case = Case(seqs, 4, 2, 128, "diag", window=100, seed=13).to("cuda")
    old = ops.get_attn_tc_min_q()
    ops.set_attn_tc_min_q(16)
    try:
        out = run_kernel("auto", case)
    finally:
        ops.set_attn_tc_min_q(old)
    expect = "tc" if max_q >= 16 else "cc"
    ops.set_attn_tc_min_q(2)
    try:
        forced = run_kernel(expect, case)
    finally:
        ops.set_attn_tc_min_q(old)
    assert torch.equal(out, forced)
    check_case(expect, case, out, f"tc_min_q=16 max_q={max_q}")


@gpu
@pytest.mark.parametrize("what", ["G32", "ragged_group", "head_dim96", "small_ws_tc", "small_ws_cc"])
def test_host_refuses_unsupported_launches(what):
    """unsupported layouts and a too-small split workspace raise a Python error before any launch (out untouched)"""
    ops = _ops()
    dev = "cuda"
    n_q, n_kv, D, splits, use_tc = 4, 2, 128, 1, -1
    if what == "G32":
        n_q, n_kv, D = 32, 1, 64
    elif what == "ragged_group":
        n_q, n_kv = 6, 4
    elif what == "head_dim96":
        D = 96
    else:
        splits, use_tc = 4, (1 if what == "small_ws_tc" else 0)
    S, T = 2, 4
    q = torch.randn(T, n_q * D, device=dev).to(torch.bfloat16)
    kc = torch.zeros(4, PAGE, n_kv, D, device=dev, dtype=torch.bfloat16)
    out = torch.full_like(q, SENTINEL)
    bt = torch.zeros(S, 2, dtype=torch.int32, device=dev)
    qs = torch.tensor([0, 1], dtype=torch.int32, device=dev)
    ql = torch.ones(S, dtype=torch.int32, device=dev)
    kvl = torch.tensor([10, 70], dtype=torch.int32, device=dev)
    R = _attn_rows(max(1, n_q // n_kv))
    ws = torch.zeros(S * n_kv * splits * R * (D + 2) - 1, device=dev) if splits > 1 else None
    with pytest.raises(RuntimeError):
        ops.attention(q, kc, kc, out, bt, qs, ql, kvl, max_q=1, n_q=n_q, n_kv=n_kv, head_dim=D, splits=splits, ws=ws,
                      use_tc=use_tc)
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()
