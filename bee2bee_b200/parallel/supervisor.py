"""Supervised engine: the serving front (mesh node, HTTP sidecar) stays in ITS OWN process; the engine -- one worker
process per GPU piece, or one CPU worker -- runs as a child process group that can die and be restarted.

Why: a GPU rank that *stalls* is survivable in-process (bounded flag waits -> ``MeshStalled`` -> the engine marks itself
broken, ``engine/runner.py``), but a rank that *dies* takes its NVLink neighbours' CUDA contexts with it (they store into
its freed memory), and a broken CUDA context cannot be repaired from inside the process that owns it.  The reference's
semantics for a lost peer are "drop it, the next ``pick_provider`` skips it" (/root/reference/bee2bee/p2p_runtime.py:396-410)
and a human restarts the node; here the supervisor does both: while the group is down the service reports unhealthy (the
mesh routes around it), in-flight requests fail at once, a fresh group is spawned (new rendezvous port, fresh IPC
buffers) and the provider becomes healthy again without the front process ever touching a GPU.

    front process                                   worker group (generation g)
    SupervisedEngine.submit / cancel / metrics  <-- loopback socket, length-prefixed JSON -->  rank 0: Engine + scheduler
    monitor thread: child exit codes, "broken"                                                 ranks 1..W-1: follow_forever

``SupervisedEngine`` has the ``Engine`` surface the services use (``submit``, ``generate``, ``cancel``, ``metrics``,
``broken``, ``cfg``, ``start`` / ``stop`` / ``close``).  Enable with ``B2B_SUPERVISED=1`` (``hf.load_model_and_tokenizer``)
or ``serve-hf --supervised``.
"""
from __future__ import annotations

import argparse
import json
import os
import queue
import secrets
import select
import signal
import socket
import struct
import subprocess
import sys
import threading
import time
from typing import Callable, Dict, List, Optional, Sequence

_HDR = struct.Struct("!I")
_MAX_MSG = 64 << 20


def send_msg(sock: socket.socket, obj: dict, lock: Optional[threading.Lock] = None) -> None:
    data = json.dumps(obj, default=str).encode()
    frame = _HDR.pack(len(data)) + data
    if lock is None:
        sock.sendall(frame)
    else:
        with lock:
            sock.sendall(frame)


def _recv_exact(sock: socket.socket, n: int) -> bytes:
    buf = bytearray()
    while len(buf) < n:
        chunk = sock.recv(n - len(buf))
        if not chunk:
            raise ConnectionError("peer closed the control channel")
        buf.extend(chunk)
    return bytes(buf)


def recv_msg(sock: socket.socket) -> dict:
    (n,) = _HDR.unpack(_recv_exact(sock, _HDR.size))
    if n > _MAX_MSG:
        raise ConnectionError(f"oversized control frame ({n} bytes)")
    return json.loads(_recv_exact(sock, n))


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


# ================================================================================================ front side
class SupervisedEngine:
    def __init__(self, model: str, device: str = "cpu", world: int = 1, engine_kw: Optional[dict] = None,
                 max_restarts: int = 5, ready_timeout_s: float = 900.0, python: Optional[str] = None):
        from ..engine.core import Request            # noqa: F401  (the front only needs the dataclasses, never torch.cuda)
        from ..models.config import resolve_config

        self.model, self.device, self.world = model, str(device), max(1, int(world))
        self.engine_kw = dict(engine_kw or {})
        self.cfg = resolve_config(model)
        self.max_restarts, self.ready_timeout_s = max_restarts, ready_timeout_s
        self.python = python or sys.executable
        self.broken: Optional[str] = "starting"
        self.restarts = 0
        self.generation = 0
        self._token = secrets.token_hex(16)
        self._srv = socket.socket()
        self._srv.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        self._srv.bind(("127.0.0.1", 0))
        self._srv.listen(4)
        self._srv.settimeout(0.5)
        self._addr = self._srv.getsockname()
        self._lock = threading.RLock()               # group state (procs, connection, live requests)
        self._send_lock = threading.Lock()
        self._conn: Optional[socket.socket] = None
        self._procs: List[subprocess.Popen] = []
        self._live: Dict[int, "Request"] = {}
        self._ids = iter(range(1, 1 << 62))
        self._metrics_q: "queue.Queue[dict]" = queue.Queue()
        self._closing = False
        self._ready = threading.Event()
        self._restarting = False
        self._last_error = ""
        try:
            self._bring_up()
        except Exception:
            self._kill_group()
            self._srv.close()
            raise
        self._monitor = threading.Thread(target=self._monitor_loop, name="b2b-supervisor", daemon=True)
        self._monitor.start()

    # ------------------------------------------------------------------ group life cycle
    def _spawn(self) -> None:
        port = _free_port()
        # the workers import this package by name whatever the front's working directory is
        pkg_parent = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        pypath = pkg_parent + (os.pathsep + os.environ["PYTHONPATH"] if os.environ.get("PYTHONPATH") else "")
        base = dict(os.environ, B2B_SUP_TOKEN=self._token, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                    WORLD_SIZE=str(self.world), PYTHONPATH=pypath)
        self._procs = []
        for r in range(self.world):
            env = dict(base, RANK=str(r), LOCAL_RANK=str(r))
            cmd = [self.python, "-m", "bee2bee_b200.parallel.supervisor", "--worker", "--connect",
                   f"{self._addr[0]}:{self._addr[1]}", "--model", self.model, "--device", self.device, "--rank", str(r),
                   "--world", str(self.world), "--engine-kw", json.dumps(self.engine_kw)]
            self._procs.append(subprocess.Popen(cmd, env=env, start_new_session=True))

    def _accept_rank0(self) -> socket.socket:
        """rank 0 of the new generation dials in and authenticates; give up as soon as any child has exited"""
        deadline = time.time() + self.ready_timeout_s
        while time.time() < deadline and not self._closing:
            dead = [p for p in self._procs if p.poll() is not None]
            if dead:
                raise RuntimeError(f"worker exited with code {dead[0].returncode} during start-up")
            try:
                conn, _ = self._srv.accept()
            except socket.timeout:
                continue
            conn.settimeout(10.0)
            try:
                hello = recv_msg(conn)
            except Exception:
                conn.close()
                continue
            if hello.get("op") != "hello" or hello.get("token") != self._token:
                conn.close()
                continue
            conn.settimeout(None)
            return conn
        raise RuntimeError("worker group did not come up in time")

    def _bring_up(self) -> None:
        self._ready.clear()
        self._spawn()
        conn = self._accept_rank0()
        # the engine build (weights, graphs) happens after the hello: wait for "ready"
        deadline = time.time() + self.ready_timeout_s
        while True:
            if time.time() > deadline:
                raise RuntimeError("engine did not become ready in time")
            dead = [p for p in self._procs if p.poll() is not None]
            if dead:
                raise RuntimeError(f"worker exited with code {dead[0].returncode} while building the engine")
            if not select.select([conn], [], [], 1.0)[0]:
                continue                                 # (frames are read whole once the first byte is there)
            msg = recv_msg(conn)
            if msg.get("op") == "ready":
                break
            if msg.get("op") == "broken":
                raise RuntimeError(f"engine failed to start: {msg.get('error')}")
        conn.settimeout(None)
        with self._lock:
            self._conn = conn
            self.generation += 1
            self.broken = None
        self._reader = threading.Thread(target=self._reader_loop, args=(conn, self.generation), daemon=True,
                                        name=f"b2b-supervisor-rx{self.generation}")
        self._reader.start()
        self._ready.set()

    def _kill_group(self) -> None:
        for p in self._procs:
            if p.poll() is None:
                try:
                    os.killpg(p.pid, signal.SIGTERM)          # exact process groups we started (start_new_session)
                except (ProcessLookupError, PermissionError):
                    pass
        t0 = time.time()
        for p in self._procs:
            try:
                p.wait(timeout=max(0.1, 5.0 - (time.time() - t0)))
            except subprocess.TimeoutExpired:
                try:
                    os.killpg(p.pid, signal.SIGKILL)
                except (ProcessLookupError, PermissionError):
                    pass
                p.wait(timeout=10)
        self._procs = []

    def _fail_live(self, why: str) -> None:
        with self._lock:
            live, self._live = self._live, {}
        for r in live.values():
            r.error = why
            r.finish_reason = "error"
            r.t_done = time.time()
            r.done.set()

    def _restart(self, why: str) -> None:
        with self._lock:
            if self._closing or self._restarting:
                return                                   # a restart is already in progress
            self._restarting = True
            self.broken = f"engine group down: {why}"
            self._ready.clear()
            conn, self._conn = self._conn, None
        try:
            self._last_error = why
            if conn is not None:
                try:
                    conn.close()
                except OSError:
                    pass
            self._fail_live(f"engine group restarted: {why}")
            self._kill_group()
            if self.restarts >= self.max_restarts:
                self.broken = f"engine group down for good after {self.restarts} restarts: {why}"
                return
            self.restarts += 1
            try:
                self._bring_up()
            except Exception as exc:                     # could not come back: stay unhealthy, the monitor tries again
                self._kill_group()
                self.broken = f"engine group down: restart failed: {exc}"
        finally:
            self._restarting = False

    def _monitor_loop(self) -> None:
        while not self._closing:
            time.sleep(0.2)
            if self._closing:
                return
            if self._ready.is_set():
                dead = [p for p in self._procs if p.poll() is not None]
                if dead:
                    self._restart(f"rank process {dead[0].pid} exited with code {dead[0].returncode}")
            elif self.broken and not self._restarting and self.restarts < self.max_restarts and not self._procs:
                time.sleep(1.0)                          # back off, then try to bring the group up again
                self._restart(self._last_error or "retry")

    # ------------------------------------------------------------------ channel
    def _reader_loop(self, conn: socket.socket, generation: int) -> None:
        try:
            while True:
                msg = recv_msg(conn)
                op = msg.get("op")
                if op == "token":
                    r = self._live.get(msg["id"])
                    if r is not None:
                        if not r.t_first:
                            r.t_first = time.time()
                        r.out_ids.append(int(msg["tok"]))
                        if r.on_token is not None:
                            r.on_token(int(msg["tok"]))
                elif op == "done":
                    with self._lock:
                        r = self._live.pop(msg["id"], None)
                    if r is not None:
                        if r.on_token is None:
                            r.out_ids = [int(t) for t in msg.get("out_ids", [])]
                        r.finish_reason = msg.get("finish_reason", "")
                        r.error = msg.get("error")
                        r.t_first = r.t_first or (r.t_submit + msg.get("ttft_ms", 0.0) / 1e3)
                        r.t_done = time.time()
                        r.done.set()
                elif op == "metrics":
                    self._metrics_q.put(msg.get("data", {}))
                elif op == "broken":
                    threading.Thread(target=self._restart, args=(f"engine reported: {msg.get('error')}",),
                                     daemon=True).start()
                    return
        except Exception as exc:
            if not self._closing and generation == self.generation and self._ready.is_set():
                threading.Thread(target=self._restart, args=(f"control channel lost: {exc}",), daemon=True).start()

    def _send(self, obj: dict) -> None:
        conn = self._conn
        if conn is None:
            raise RuntimeError(self.broken or "engine group is not running")
        send_msg(conn, obj, self._send_lock)

    # ------------------------------------------------------------------ Engine surface
    @property
    def healthy(self) -> bool:
        return self.broken is None

    def worker_pids(self) -> List[int]:
        return [p.pid for p in self._procs]

    def start(self) -> None:                             # the worker's scheduler thread is started by the worker
        return None

    def stop(self) -> None:
        return None

    def submit(self, prompt_ids: Sequence[int], params=None, on_token: Optional[Callable[[int], None]] = None):
        from ..engine.core import Request, SamplingParams

        params = params or SamplingParams()
        params.validate(self.cfg.vocab_size)      # refused here, as by Engine.submit, rather than inside the worker
        r = Request(next(self._ids), list(prompt_ids), params, on_token, t_submit=time.time())
        if self.broken:
            r.error, r.finish_reason, r.t_done = self.broken, "error", time.time()
            r.done.set()
            return r
        with self._lock:
            self._live[r.rid] = r
        try:
            p = dict(params.__dict__)
            p["stop_token_ids"] = list(p.get("stop_token_ids") or ())
            p["logit_bias"] = dict(p.get("logit_bias") or {})          # JSON turns its int keys into strings
            self._send({"op": "submit", "id": r.rid, "prompt_ids": r.prompt_ids, "params": p,
                        "stream": on_token is not None})
        except Exception as exc:
            with self._lock:
                self._live.pop(r.rid, None)
            r.error, r.finish_reason, r.t_done = f"engine group unreachable: {exc}", "error", time.time()
            r.done.set()
        return r

    def generate(self, prompts: Sequence[Sequence[int]], params=None) -> List[List[int]]:
        reqs = [self.submit(p, params) for p in prompts]
        return [r.wait().out_ids for r in reqs]

    def cancel(self, req, reason: str = "cancelled") -> None:
        if req.done.is_set():
            return
        req.cancelled = True
        try:
            self._send({"op": "cancel", "id": req.rid, "reason": reason})
        except Exception:
            pass

    def metrics(self) -> Dict[str, object]:
        out: Dict[str, object] = {}
        if self._ready.is_set():
            try:
                while not self._metrics_q.empty():
                    self._metrics_q.get_nowait()
                self._send({"op": "metrics"})
                out = self._metrics_q.get(timeout=5.0)
            except Exception:
                out = {}
        out.setdefault("tokens_per_s", 0.0)
        out.update(healthy=self.healthy, supervised=True, restarts=self.restarts, generation=self.generation,
                   worker_pids=self.worker_pids())
        return out

    def wait_healthy(self, timeout: float = 600.0) -> bool:
        t0 = time.time()
        while time.time() - t0 < timeout:
            if self.healthy:
                return True
            time.sleep(0.05)
        return self.healthy

    def close(self) -> None:
        self._closing = True
        try:
            if self._conn is not None:
                send_msg(self._conn, {"op": "shutdown"}, self._send_lock)
        except Exception:
            pass
        t0 = time.time()
        while time.time() - t0 < 5.0 and any(p.poll() is None for p in self._procs):
            time.sleep(0.05)
        self._kill_group()
        self._fail_live("engine closed")
        for s in (self._conn, self._srv):
            try:
                if s is not None:
                    s.close()
            except OSError:
                pass
        self._conn = None
        self.broken = "closed"


# =============================================================================================== worker side
def _worker(a: argparse.Namespace) -> int:
    host, port = a.connect.rsplit(":", 1)
    kw = json.loads(a.engine_kw)
    sock: Optional[socket.socket] = None
    if a.rank == 0:
        sock = socket.create_connection((host, int(port)), timeout=30)
        sock.settimeout(None)
        send_msg(sock, {"op": "hello", "token": os.environ.get("B2B_SUP_TOKEN", ""), "rank": 0, "pid": os.getpid()})
    try:
        if a.world > 1:
            from .launch import build_engine
            eng = build_engine(a.model, a.rank, a.world, **kw)
        else:
            from ..engine.core import Engine
            eng = Engine(a.model, device=a.device, **kw)
    except Exception as exc:
        if sock is not None:
            send_msg(sock, {"op": "broken", "error": f"engine build failed: {exc!r}"})
        raise
    if a.rank != 0:
        try:
            eng.follow_forever()
        finally:
            eng.runner.close()
        return 0
    from ..engine.core import SamplingParams

    eng.start()
    send_msg(sock, {"op": "ready", "pid": os.getpid()})
    live: Dict[int, object] = {}
    toks: "queue.Queue[tuple]" = queue.Queue()
    reported_broken = False
    try:
        while True:
            ready, _, _ = select.select([sock], [], [], 0.002 if live else 0.05)
            if ready:
                msg = recv_msg(sock)
                op = msg.get("op")
                if op == "submit":
                    p = dict(msg["params"])
                    p["stop_token_ids"] = tuple(p.get("stop_token_ids") or ())
                    p["logit_bias"] = {int(k): v for k, v in (p.get("logit_bias") or {}).items()}
                    rid = msg["id"]
                    cb = (lambda t, i=rid: toks.put((i, int(t)))) if msg.get("stream") else None
                    live[rid] = eng.submit(msg["prompt_ids"], SamplingParams(**p), on_token=cb)
                elif op == "cancel":
                    r = live.get(msg["id"])
                    if r is not None:
                        eng.cancel(r, msg.get("reason", "cancelled"))
                elif op == "metrics":
                    send_msg(sock, {"op": "metrics", "data": eng.metrics()})
                elif op == "shutdown":
                    break
            finished = [(i, r) for i, r in live.items() if r.done.is_set()]      # BEFORE draining: their tokens are queued
            while True:
                try:
                    i, t = toks.get_nowait()
                except queue.Empty:
                    break
                send_msg(sock, {"op": "token", "id": i, "tok": t})
            for i, r in finished:
                send_msg(sock, {"op": "done", "id": i, "out_ids": [int(t) for t in r.out_ids], "ttft_ms": r.ttft_ms,
                                "finish_reason": r.finish_reason, "error": r.error})
                del live[i]
            if eng.broken and not reported_broken:
                reported_broken = True
                send_msg(sock, {"op": "broken", "error": eng.broken})
    except ConnectionError:
        pass                                              # the front went away: nothing left to serve
    finally:
        try:
            eng.close()
        except Exception:
            pass
    return 0


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="engine worker of a SupervisedEngine (not meant to be started by hand)")
    ap.add_argument("--worker", action="store_true", required=True)
    ap.add_argument("--connect", required=True)
    ap.add_argument("--model", required=True)
    ap.add_argument("--device", default="cpu")
    ap.add_argument("--rank", type=int, default=0)
    ap.add_argument("--world", type=int, default=1)
    ap.add_argument("--engine-kw", default="{}")
    return _worker(ap.parse_args(argv))


if __name__ == "__main__":
    sys.exit(main())
