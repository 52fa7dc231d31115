"""Inference engine: request queue, continuous batching over fixed batch slots, paged-KV
admission control, token streaming.  The reference runs one blocking
``model.generate`` per request inside the event loop (no batching, no KV management,
/root/reference/bee2bee/services.py:85-116, api.py:229); here requests are only *enqueued*
by the asyncio side and a scheduler thread drives the GPU:

    admit (pages available?) -> prefill burst -> decode burst of N graph replays -> read tokens
    -> EOS / max_new_tokens / stop handling -> free slots -> repeat

Backends: ``GpuRunner`` (hand-written sm_90a kernels; one per GPU, pieces over NVLink) or
``TorchRunner`` (plain PyTorch; CPU plumbing configuration and numerical oracle).
"""
from __future__ import annotations

import itertools
import os
import collections
import queue
import re
import statistics
import threading
import time
from dataclasses import dataclass, field, fields
from typing import Callable, Dict, List, Mapping, Optional, Sequence

import numpy as np
import torch

from ..models.config import ModelConfig, resolve_config, split_layers
from ..models.torch_ref import SequenceSampler, TorchPiece
from ..models.weights import load_or_init
from .kv import PAGE, PageAllocator


LOGIT_BIAS_MAX = 1024       # entries one request's logit_bias may hold (the width of the sampler's bias tables)
LOGIT_BIAS_LIMIT = 100.0    # |bias| bound, as in OpenAI's API


def parse_logit_bias(obj: Optional[Mapping]) -> Dict[int, float]:
    """A request's ``logit_bias`` as the engine takes it: int token id -> float bias.  On the wire it is a JSON object
    whose keys are decimal strings (OpenAI's shape); int keys are taken as they are.  None or an empty map = off.
    Raises ``ValueError`` for a key that is not a decimal integer, for two keys that name the same id ("5" and "05")
    and for a value that is not a number; ranges are checked by ``SamplerControls.validate``."""
    if obj is None:
        return {}
    if not isinstance(obj, Mapping):
        raise ValueError(f"logit_bias must be a map of token id -> bias, got {type(obj).__name__}")
    out: Dict[int, float] = {}
    for k, v in obj.items():
        if isinstance(k, str) and re.fullmatch(r"[+-]?[0-9]+", k):
            tid = int(k)
        elif isinstance(k, (int, np.integer)) and not isinstance(k, bool):
            tid = int(k)
        else:
            raise ValueError(f"logit_bias keys must be integer token ids, got {k!r}")
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)):
            raise ValueError(f"logit_bias[{k!r}] must be a number, got {v!r}")
        if tid in out:
            raise ValueError(f"logit_bias names token id {tid} twice")
        out[tid] = float(v)
    return out


@dataclass(kw_only=True)
class SamplerControls:
    """A sequence's sampling controls: the request carries them (``SamplingParams``), the replicated plan hands them
    to every rank (``runner.SeqInit``), and the sampler applies them per sequence."""
    temperature: float = 0.7
    top_p: float = 0.95                # reference streaming default (hf.py:103)
    repetition_penalty: float = 1.15   # reference streaming default (hf.py:95)
    top_k: int = 0                     # keep the k most likely tokens (ties kept) before top-p; 0 = off
    min_p: float = 0.0                 # after top-p keep tokens with p >= min_p * p_max; 0 = off
    presence_penalty: float = 0.0      # subtracted from every token generated so far (prompt excluded); 0 = off
    frequency_penalty: float = 0.0     # times the token's generated count, subtracted too; 0 = off
    # token id -> bias added to its logit after soft-cap, before the penalties; empty = off.  -100 makes a token
    # negligible, not impossible.
    logit_bias: Mapping[int, float] = field(default_factory=dict)

    def validate(self, vocab_size: Optional[int] = None) -> None:
        """Raise ``ValueError`` for a control outside the range the sampler defines; with ``vocab_size``, also for a
        ``logit_bias`` id outside the vocabulary."""
        if not self.top_k >= 0:
            raise ValueError(f"top_k must be >= 0 (0 = off), got {self.top_k}")
        if not 0.0 <= self.min_p <= 1.0:
            raise ValueError(f"min_p must lie in [0, 1] (0 = off), got {self.min_p}")
        for name in ("presence_penalty", "frequency_penalty"):
            v = getattr(self, name)
            if not -2.0 <= v <= 2.0:          # also refuses NaN and +-inf
                raise ValueError(f"{name} must be a finite value in [-2, 2] (0 = off), got {v}")
        if len(self.logit_bias) > LOGIT_BIAS_MAX:
            raise ValueError(f"logit_bias holds {len(self.logit_bias)} entries; at most {LOGIT_BIAS_MAX} are allowed")
        for k, v in self.logit_bias.items():
            if isinstance(k, bool) or not isinstance(k, (int, np.integer)):
                raise ValueError(f"logit_bias keys must be integer token ids, got {k!r}")
            if k < 0 or (vocab_size is not None and k >= vocab_size):
                raise ValueError(f"logit_bias id {k} lies outside the vocabulary"
                                 + (f" of {vocab_size} ids" if vocab_size is not None else ""))
            if (isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating))
                    or not -LOGIT_BIAS_LIMIT <= v <= LOGIT_BIAS_LIMIT):     # also refuses NaN and +-inf
                raise ValueError(f"logit_bias[{k}] must be a finite value in [-100, 100], got {v}")

    def controls(self) -> Dict[str, object]:
        """The controls alone, as keyword arguments for another ``SamplerControls``."""
        return {f.name: getattr(self, f.name) for f in fields(SamplerControls)}


@dataclass(kw_only=True)
class SamplingParams(SamplerControls):
    max_new_tokens: int = 32
    seed: Optional[int] = None
    stop_token_ids: Sequence[int] = ()
    ignore_eos: bool = False
    timeout_s: Optional[float] = None  # deadline from submission; an overdue request is retired ("timeout") at the next
                                       # burst boundary and frees its slot + pages (default: B2B_REQUEST_TIMEOUT_S, 0 = none)


@dataclass
class Request:
    rid: int
    prompt_ids: List[int]
    params: SamplingParams
    on_token: Optional[Callable[[int], None]] = None
    out_ids: List[int] = field(default_factory=list)
    slot: int = -1
    done: threading.Event = field(default_factory=threading.Event)
    finish_reason: str = ""
    error: Optional[str] = None
    t_submit: float = 0.0
    t_first: float = 0.0
    t_done: float = 0.0
    consumed: int = 0          # tokens already taken from the history ring
    cancelled: bool = False    # set by Engine.cancel(): retired at the next burst boundary

    @property
    def ttft_ms(self) -> float:
        return (self.t_first - self.t_submit) * 1e3 if self.t_first else 0.0

    def wait(self, timeout: Optional[float] = None) -> "Request":
        if not self.done.wait(timeout):
            raise TimeoutError(f"request {self.rid} timed out")
        if self.error:
            raise RuntimeError(self.error)
        return self


# =========================================================================== CPU / oracle backend
class TorchRunner:
    """Same interface as GpuRunner, plain PyTorch ops, dense per-slot KV.  Optionally a chain of
    pieces connected by ``hop`` callables (the loopback p2p transport in the CPU config)."""

    def __init__(self, cfg: ModelConfig, model: str = "", pieces: int = 1, device="cpu", dtype=torch.float32,
                 max_batch: int = 8, seed: int = 0, hop: Optional[Callable[[int, torch.Tensor], torch.Tensor]] = None):
        self.cfg, self.device, self.dtype, self.max_batch = cfg, torch.device(device), dtype, max_batch
        ranges = split_layers(cfg.n_layers, pieces)
        self.pieces: List[TorchPiece] = []
        for i, r in enumerate(ranges):
            first, last = i == 0, i == len(ranges) - 1
            t = load_or_init(model, cfg, r, first, last, device=self.device, dtype=dtype, seed=seed)
            self.pieces.append(TorchPiece(cfg, r, first, last, t))
        self.hop = hop
        self.cache: Dict[int, List[dict]] = {}
        self.state: Dict[int, dict] = {}
        self.kernel_launches = 0
        self.hist_len = 1 << 30

    def _forward(self, slot: int, ids: List[int], pos0: int) -> torch.Tensor:
        x = torch.tensor([ids], device=self.device)
        positions = torch.arange(pos0, pos0 + len(ids), device=self.device)[None]
        caches = self.cache.setdefault(slot, [p.new_cache() for p in self.pieces])
        for i, p in enumerate(self.pieces):
            x = p.forward(x, positions, caches[i], logits_last_only=True)
            if self.hop is not None and i + 1 < len(self.pieces):
                x = self.hop(i, x)
        return x[0, -1]

    def prefill(self, seqs) -> None:
        with torch.no_grad():
            for s in seqs:
                self.cache.pop(s.slot, None)
                sampler = SequenceSampler(s, self.cfg.vocab_size, s.prompt,
                                          torch.Generator().manual_seed(int(s.seed) & 0x7FFFFFFF))
                tok = sampler.draw(self._forward(s.slot, list(s.prompt), 0))
                self.state[s.slot] = dict(sampler=sampler, pos=len(s.prompt), hist=[tok])

    def decode(self, n_steps: int) -> None:
        with torch.no_grad():
            for _ in range(n_steps):
                for slot, st in self.state.items():
                    if not st.get("active", True):
                        continue
                    logits = self._forward(slot, [st["hist"][-1]], st["pos"])
                    st["pos"] += 1
                    st["hist"].append(st["sampler"].draw(logits))

    def sync(self) -> None:
        pass

    def tokens_of(self, slot: int, start: int, count: int) -> List[int]:
        return self.state[slot]["hist"][start:start + count]

    def release(self, slots) -> None:
        for b in slots:
            self.state.pop(b, None)
            self.cache.pop(b, None)

    def close(self) -> None:
        self.state.clear()
        self.cache.clear()


# ============================================================================================ engine
class Engine:
    """Scheduler + backend.  Thread-safe ``submit``; ``start()`` spawns the scheduler thread."""

    def __init__(self, model: str = "tiny-llama", cfg: Optional[ModelConfig] = None, device: Optional[str] = None,
                 pieces: int = 1, max_batch: int = 8, max_seq_len: int = 2048, max_prefill_tokens: int = 2048,
                 decode_burst: int = 8, seed: int = 0, runner=None, groups: int = 1, rank: int = 0, world: int = 1,
                 control_group=None, plan_sync: bool = False, plan_group=None, quant: str = "bf16",
                 overlap_prefill: bool = True, prefix_cache: bool = True):
        self.model = model
        # plan_sync: rank 0 owns the request queue and broadcasts every newly arrived request to the
        # follower ranks at the top of each step (serving); False = every rank is fed identical
        # requests by its caller (SPMD benchmark / tests)
        self.plan_sync, self.plan_group = plan_sync, plan_group
        # overlap_prefill: when none of the newly admitted requests streams tokens to a callback, the decode burst is
        # enqueued right behind the prefill and the first tokens are read together with the burst's (one read-back, no
        # pipeline drain between prefill and decode: piece 0's embed kernel waits per group for the prefill chunks that
        # hold its sequences).  Streaming requests keep the early first-token read-back (TTFT).
        self.overlap_prefill = overlap_prefill
        self._first_pending = False
        self.cfg = cfg or resolve_config(model)
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        if self.cfg.rope_theta <= 0:
            # learned absolute positions (GPT-2): a sequence may not outgrow the position table; submit() trims prompts
            # and the generation budget to this length
            max_seq_len = min(max_seq_len, self.cfg.max_position)
        self.max_batch, self.max_seq_len, self.decode_burst = max_batch, max_seq_len, max(1, decode_burst)
        self.rank, self.world, self.control_group = rank, world, control_group
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        if runner is not None:
            self.runner = runner
        elif self.device.type == "cuda":
            from .runner import GpuRunner
            if pieces > 1 and world == 1:
                raise ValueError("multi-GPU pieces run one process per GPU (SPMD): launch with torchrun and pass "
                                 "rank/world, see bench.py / bee2bee_b200.parallel.launch")
            self.runner = GpuRunner(self.cfg, model, rank, world, self.device, max_batch=max_batch, groups=groups,
                                    max_seq_len=max_seq_len, max_prefill_tokens=max_prefill_tokens, seed=seed,
                                    control_group=control_group, quant=quant)
        else:
            self.runner = TorchRunner(self.cfg, model, pieces=pieces, device=self.device, max_batch=max_batch, seed=seed)
        self.gpu = self.device.type == "cuda"
        pages_per_seq = (max_seq_len + PAGE - 1) // PAGE
        # prefix cache: only the paged GPU backend can share KV pages between sequences (the CPU oracle keeps a dense
        # cache per slot)
        self.alloc = PageAllocator(getattr(self.runner, "num_pages", 1 + max_batch * pages_per_seq),
                                   prefix_cache=self.gpu and prefix_cache)
        self._ids = itertools.count(1)
        self._waiting: "queue.Queue[Request]" = queue.Queue()
        self._pending: List[Request] = []
        self._running: Dict[int, Request] = {}
        self._free_slots = list(range(max_batch - 1, -1, -1))
        self._lock = threading.Lock()
        self._cancelled: List[int] = []            # rids cancelled since the last step (rank 0 -> plan broadcast)
        self._wake = threading.Event()
        self._stop = False
        self.broken: Optional[str] = None          # set once the mesh aborted (MeshStalled): the engine refuses new work
        self.default_timeout_s = float(os.environ.get("B2B_REQUEST_TIMEOUT_S", "0") or 0)   # 0 = requests have no deadline
        self._thread: Optional[threading.Thread] = None
        self.host_ms = {"prefill": 0.0, "decode": 0.0, "collect": 0.0}     # host wall time per scheduler phase
        self._ttfts: "collections.deque[float]" = collections.deque(maxlen=4096)   # submit -> first token, ms
        self.stats = {"requests": 0, "tokens": 0, "prefill_tokens": 0, "steps": 0, "busy_s": 0.0,
                      "started": time.time()}

    # ------------------------------------------------------------------ public
    def submit(self, prompt_ids: Sequence[int], params: Optional[SamplingParams] = None,
               on_token: Optional[Callable[[int], None]] = None) -> Request:
        params = params or SamplingParams()
        params.validate(self.cfg.vocab_size)
        ids = list(prompt_ids)[-(self.max_seq_len - 1):] or [max(self.cfg.bos_token_id, 0)]
        budget = self.max_seq_len - len(ids)
        if params.max_new_tokens > budget:
            params = SamplingParams(**{**params.__dict__, "max_new_tokens": max(1, budget)})
        r = Request(next(self._ids), ids, params, on_token, t_submit=time.time())
        if self.broken:
            # reference semantics for a lost peer: the provider disappears and the caller is told at once
            # (/root/reference/bee2bee/p2p_runtime.py:396-410) -- no request may queue behind a dead mesh
            r.error = self.broken
            r.finish_reason = "error"
            r.t_done = time.time()
            r.done.set()
            return r
        self._waiting.put(r)
        self._wake.set()
        return r

    def generate(self, prompts: Sequence[Sequence[int]], params: Optional[SamplingParams] = None) -> List[List[int]]:
        """Blocking helper: run to completion (drives the scheduler inline if no thread is running)."""
        reqs = [self.submit(p, params) for p in prompts]
        if self._thread is None:
            while not all(r.done.is_set() for r in reqs):
                try:
                    self.step()
                except Exception as e:
                    self._note_failure(e)
                    self._fail_all(f"engine error: {e!r}")
                    raise
        return [r.wait().out_ids for r in reqs]

    def cancel(self, req: Request, reason: str = "cancelled") -> None:
        """Abandon a request (client disconnected, stop word hit, wait timed out): it stops occupying its batch slot
        and KV pages at the next burst boundary instead of decoding to ``max_new_tokens``.  Thread-safe; on a serving
        mesh the cancellation travels to the follower ranks with the next plan broadcast.  The reference leaks its
        generate thread in the same situation (/root/reference/bee2bee/hf.py:107-136)."""
        if req.done.is_set():
            return
        req.cancelled = True          # retired (finish_reason "cancelled") at the next burst boundary, on every rank
        with self._lock:
            self._cancelled.append(req.rid)
        self._wake.set()

    def start(self) -> None:
        if self._thread is None:
            self._stop = False
            self._thread = threading.Thread(target=self._loop, name="b2b-engine", daemon=True)
            self._thread.start()

    def stop(self) -> None:
        self._stop = True
        self._wake.set()
        if self._thread is not None:
            self._thread.join(timeout=10)
            self._thread = None
        if self.world > 1 and self.plan_sync and self.rank == 0:
            try:                                   # release the followers blocked in the plan broadcast
                self._sync_plan([])
            except Exception:
                pass

    def close(self) -> None:
        self.stop()
        self.runner.close()

    def metrics(self) -> Dict[str, float]:
        up = max(1e-9, time.time() - self.stats["started"])
        busy = max(1e-9, self.stats["busy_s"])
        return {"requests": self.stats["requests"], "tokens_generated": self.stats["tokens"],
                "prefill_tokens": self.stats["prefill_tokens"], "decode_steps": self.stats["steps"],
                "tokens_per_s": self.stats["tokens"] / busy, "running": len(self._running),
                "waiting": self._waiting.qsize() + len(self._pending), "kv_utilization": self.alloc.utilization(),
                "healthy": self.broken is None, "cancelled": self.stats.get("cancelled", 0),
                "timeouts": self.stats.get("timeouts", 0), "prefix_cache": self.alloc.cache_stats(),
                "prefix_cache_hit_tokens": self.stats.get("prefix_cache_hit_tokens", 0), "uptime_s": up, "h2d_bytes": self.h2d_bytes + getattr(self.runner, "h2d_bytes", 0),
                "d2h_bytes": self.d2h_bytes, "native_launches": getattr(self.runner, "kernel_launches", 0),
                "host_ms": dict(self.host_ms),
                "ttft_ms": ({"count": len(self._ttfts), "p50": statistics.median(self._ttfts),
                             "p90": sorted(self._ttfts)[int(0.9 * (len(self._ttfts) - 1))]} if self._ttfts else {}),
                "trace": __import__("bee2bee_b200.utils.tracing", fromlist=["TRACER"]).TRACER.summary()}

    # --------------------------------------------------------------- scheduler
    def _loop(self) -> None:
        while not self._stop:
            try:
                worked = self.step()
            except Exception as e:  # keep serving: fail the in-flight requests, not the node
                worked = True
                self._note_failure(e)                 # first: waiters woken by _fail_all must already see `broken`
                self._fail_all(f"engine error: {e!r}")
            if not worked:
                self._wake.wait(0.05)
                self._wake.clear()

    def _sync_plan(self, fresh: List[Request], cancelled: Optional[List[int]] = None) -> Optional[List[Request]]:
        """Replicated control plane: rank 0 broadcasts the requests that arrived since the last step
        (ids, prompt, sampling params); followers materialise mirror Request objects so that every
        rank takes identical admission / retirement decisions.  Returns None once rank 0 shuts down."""
        import torch.distributed as dist

        box = [None]
        if self.rank == 0:
            box[0] = {"stop": self._stop, "new": [(r.rid, r.prompt_ids, dict(r.params.__dict__)) for r in fresh],
                      "cancel": list(cancelled or [])}
        dist.broadcast_object_list(box, src=0, group=self.plan_group)
        plan = box[0]
        if plan["stop"]:
            self._stop = True
            return None
        self._plan_cancel = list(plan.get("cancel") or [])
        if self.rank == 0:
            return fresh
        out = []
        for rid, ids, sp in plan["new"]:
            sp["stop_token_ids"] = tuple(sp.get("stop_token_ids") or ())
            out.append(Request(rid, list(ids), SamplingParams(**sp), t_submit=time.time()))
        return out

    def follow_forever(self) -> None:
        """Follower ranks of a serving mesh: mirror rank 0 until it stops."""
        while not self._stop:
            if not self.step():
                time.sleep(0.002)

    def _note_failure(self, exc: Exception) -> None:
        from .runner import MeshStalled

        if isinstance(exc, MeshStalled):
            self.broken = f"mesh unavailable: {exc}"
            while True:                      # nobody may wait on a queue that will never be served
                try:
                    r = self._waiting.get_nowait()
                except queue.Empty:
                    break
                r.error, r.finish_reason, r.t_done = self.broken, "error", time.time()
                r.done.set()

    def _fail_all(self, msg: str) -> None:
        victims = list(self._running.values()) + self._pending
        try:
            self.runner.release(list(self._running.keys()))
        except Exception:
            pass
        for b in self._running:
            self.alloc.invalidate(b)            # a failed burst may have left half-written KV pages behind
            self.alloc.release(b)
            self._free_slots.append(b)
        self._running.clear()
        self._pending.clear()
        for r in victims:          # wake the waiters last: they may inspect the engine state right away
            r.error = msg
            r.t_done = time.time()
            r.done.set()

    def step(self) -> bool:
        """One scheduler iteration: retire cancelled requests, admit + prefill, then one decode burst.
        Returns False when idle."""
        from .runner import SeqInit

        t0 = time.time()
        fresh: List[Request] = []
        while True:
            try:
                fresh.append(self._waiting.get_nowait())
            except queue.Empty:
                break
        self._expire_overdue()
        with self._lock:
            cancelled, self._cancelled = self._cancelled, []
        if self.world > 1 and self.plan_sync:
            fresh = self._sync_plan(fresh, cancelled)
            if fresh is None:
                return False
            cancelled = self._plan_cancel
        self._pending.extend(fresh)
        if cancelled:
            self._retire_cancelled(set(cancelled))
        admitted: List[Request] = []
        still: List[Request] = []
        for r in self._pending:
            need = len(r.prompt_ids) + r.params.max_new_tokens
            if self._free_slots and self.alloc.can_allocate(need, r.prompt_ids):
                r.slot = self._free_slots.pop()
                self.alloc.allocate(r.slot, need, r.prompt_ids)
                admitted.append(r)
            else:
                still.append(r)
        self._pending = still
        if admitted:
            seqs = [SeqInit(slot=r.slot, prompt=r.prompt_ids, pages=self.alloc.owned(r.slot),
                            # k >= vocab already means off; the clamp keeps any k a client sends inside int32
                            **{**r.params.controls(), "top_k": min(int(r.params.top_k), self.cfg.vocab_size)},
                            seed=r.params.seed if r.params.seed is not None else (r.rid * 2654435761) & 0x7FFFFFFF,
                            cached=self.alloc.cached_tokens(r.slot))
                    for r in admitted]
            for r in admitted:          # after the whole admission round: requests of one round never share with each other
                self.alloc.commit(r.slot, r.prompt_ids)
            from ..utils.tracing import TRACER
            th = time.perf_counter()
            # the admitted requests are "running" from here on, so that a failing prefill is cleaned up by
            # _fail_all (slots, pages, waiters) instead of leaking them
            for r in admitted:
                self._running[r.slot] = r
            try:
                with TRACER.range(f"prefill[{len(seqs)} seqs]", getattr(self.runner, "stream", None),
                                  device_timed=self.gpu):
                    self.runner.prefill(seqs)
            except Exception as e:
                self._fail_all(f"prefill failed: {e!r}")
                raise
            self.host_ms["prefill"] += (time.perf_counter() - th) * 1e3
            for r in admitted:
                self.stats["prefill_tokens"] += len(r.prompt_ids) - self.alloc.cached_tokens(r.slot)
                self.stats["prefix_cache_hit_tokens"] = self.stats.get("prefix_cache_hit_tokens", 0) + self.alloc.cached_tokens(r.slot)
                self.stats["requests"] += 1
            if self.overlap_prefill and not any(r.on_token is not None for r in admitted):
                self._first_pending = True
            else:
                self._collect(first=True)
        if not self._running:
            if admitted:
                self.stats["busy_s"] += time.time() - t0
            return bool(admitted) or bool(cancelled)
        # a request whose first token (sampled by the prefill) has not been collected yet still owes one token less
        remaining = min(r.params.max_new_tokens - len(r.out_ids) - (1 if r.consumed == 0 else 0)
                        for r in self._running.values())
        n = max(1, min(self.decode_burst, remaining, getattr(self.runner, "hist_len", 1 << 30)))
        th = time.perf_counter()
        self.runner.decode(n)
        tc = time.perf_counter()
        self.host_ms["decode"] += (tc - th) * 1e3
        self.stats["steps"] += n
        self._collect(steps=n, include_first=self._first_pending)   # blocks on the device-side "burst complete on every rank" condition
        self._first_pending = False
        self.host_ms["collect"] += (time.perf_counter() - tc) * 1e3
        self.stats["busy_s"] += time.time() - t0
        return True

    def _expire_overdue(self) -> None:
        """Deadline check (rank 0 / single rank decides; the cancellation then travels with the plan like any other):
        queued and running requests whose ``timeout_s`` has passed are cancelled with finish_reason "timeout"."""
        if self.rank != 0 or (self.world > 1 and not self.plan_sync):
            return          # replicated (SPMD) submission without a plan broadcast: a wall-clock decision would diverge
        now = time.time()
        for r in list(self._pending) + list(self._running.values()):
            limit = r.params.timeout_s if r.params.timeout_s is not None else self.default_timeout_s
            if limit and limit > 0 and not r.cancelled and now - r.t_submit > limit:
                r.finish_reason = "timeout"
                self.cancel(r, "timeout")
                self.stats["timeouts"] = self.stats.get("timeouts", 0) + 1

    def _retire_cancelled(self, rids) -> None:
        """Burst boundary (the device is idle): drop cancelled requests from the queue / free their slot + pages."""
        keep = []
        for r in self._pending:
            if r.rid in rids:
                r.cancelled = True
                r.finish_reason = r.finish_reason or "cancelled"
                r.t_done = time.time()
                r.done.set()
            else:
                keep.append(r)
        self._pending = keep
        gone = [b for b, r in self._running.items() if r.rid in rids]
        if gone:
            self.runner.release(gone)
            for b in gone:
                r = self._running.pop(b)
                self.alloc.release(b)
                self._free_slots.append(b)
                r.cancelled = True
                r.finish_reason = r.finish_reason or "cancelled"
                r.t_done = time.time()
                r.done.set()
            self.stats["cancelled"] = self.stats.get("cancelled", 0) + len(gone)

    def _fetch_window(self, width: int, first: bool = False) -> torch.Tensor:
        """[max_batch, width] newest tokens of every slot, starting at each request's read cursor.  One kernel on
        every rank (runner.fetch_window): it waits on rank 0's sampler / prefill flags and gathers from rank 0's ring
        -- follower ranks read both through their NVLink mapping -- so every rank sees the same tokens and takes the
        same scheduling decisions without a broadcast."""
        cur = [0] * self.max_batch
        for b, r in self._running.items():
            cur[b] = r.consumed
        win = self.runner.fetch_window(cur, width, first=first)      # the runner counts the cursor / wait-list bytes
        self.d2h_bytes += win.numel() * 4
        return win

    def _collect(self, first: bool = False, steps: int = 0, include_first: bool = False) -> None:
        """Pull freshly produced tokens for every running request, stream them, retire finished ones.
        ``include_first``: requests admitted by the last prefill have not had their first token read yet -- their window
        is one token longer (first token + the burst)."""
        width = 1 if first else steps + (1 if include_first else 0)
        if self.gpu:
            win = self._fetch_window(width, first=first)
        finished: List[int] = []
        now = time.time()
        eos = list(self.cfg.eos_ids)
        if self.gpu:
            win = win.numpy()
        for b, r in list(self._running.items()):
            have = 1 if first and r.consumed == 0 else steps + (1 if (include_first and r.consumed == 0) else 0)
            if first and r.consumed > 0:
                continue
            row = win[b, :have] if self.gpu else np.asarray(self.runner.tokens_of(b, r.consumed, have), dtype=np.int64)
            r.consumed += len(row)
            if r.finish_reason or len(row) == 0:
                if r.finish_reason:
                    finished.append(b)
                continue
            # whole-window bookkeeping (a per-token Python loop cost ~10 ms per burst at 256 sequences x 20 tokens)
            take = min(len(row), r.params.max_new_tokens - len(r.out_ids))
            stop_at = -1
            if not r.params.ignore_eos or r.params.stop_token_ids:
                hit = np.zeros(take, dtype=bool)
                if not r.params.ignore_eos:
                    hit |= np.isin(row[:take], eos)
                if r.params.stop_token_ids:
                    hit |= np.isin(row[:take], list(r.params.stop_token_ids))
                nz = np.flatnonzero(hit)
                if nz.size:
                    stop_at = int(nz[0])
                    take = stop_at + 1
            new = row[:take].tolist()
            if new and not r.t_first:
                r.t_first = now
                if r.t_submit:
                    self._ttfts.append((r.t_first - r.t_submit) * 1e3)
            r.out_ids.extend(new)
            self.stats["tokens"] += len(new)
            if r.on_token is not None and not r.cancelled:
                for tok in new:
                    try:
                        r.on_token(tok)
                    except Exception:
                        pass
            if stop_at >= 0:
                r.finish_reason = "stop"
            elif len(r.out_ids) >= r.params.max_new_tokens:
                r.finish_reason = "length"
            if r.finish_reason:
                finished.append(b)
        if finished:
            self.runner.release(finished)
            for b in finished:
                r = self._running.pop(b)
                self.alloc.release(b)
                self._free_slots.append(b)
                r.t_done = time.time()
                r.done.set()
