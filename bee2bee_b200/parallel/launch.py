"""Multi-GPU serving launcher: ``serve-hf --pieces N`` on a H100 box.

Rank 0 is the process the user started (mesh node + HTTP sidecar + scheduler); ranks 1..N-1
are spawned as ``python -m bee2bee_b200.parallel.launch --follower`` subprocesses, one per GPU.
All ranks join one ``torch.distributed`` world (NCCL for barriers / IPC-handle exchange /
token-window broadcast, a gloo group for the plan objects); the token path between the pieces
is the fused NVLink handoff (``parallel.mesh``), never a collective.
"""
from __future__ import annotations

import argparse
import datetime
import os
import socket
import subprocess
import sys
from typing import List, Optional


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def build_engine(model: str, rank: int, world: int, **engine_kw):
    """Join the world described by the environment and build this rank's SPMD engine."""
    import torch
    import torch.distributed as dist

    from ..engine.core import Engine

    torch.cuda.set_device(rank)
    if not dist.is_initialized():
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"),
                                timeout=datetime.timedelta(hours=12))
    plan_group = dist.new_group(backend="gloo", timeout=datetime.timedelta(hours=12))
    engine_kw.setdefault("groups", world)
    mb = engine_kw.get("max_batch", 8 * world)
    engine_kw["max_batch"] = max(world, (mb // world) * world)
    return Engine(model, device=f"cuda:{rank}", rank=rank, world=world, plan_sync=True, plan_group=plan_group,
                  **engine_kw)


def spawn_followers(model: str, world: int, engine_kw: dict, port: Optional[int] = None) -> List[subprocess.Popen]:
    """Start ranks 1..world-1 and export the rendezvous env for rank 0 (this process)."""
    import json

    port = port or _free_port()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), WORLD_SIZE=str(world), RANK="0", LOCAL_RANK="0")
    procs = []
    for r in range(1, world):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, "-m", "bee2bee_b200.parallel.launch", "--follower", "--model",
                                       model, "--world", str(world), "--rank", str(r), "--engine-kw",
                                       json.dumps(engine_kw)], env=env))
    return procs


def main(argv=None) -> None:
    import json

    ap = argparse.ArgumentParser()
    ap.add_argument("--follower", action="store_true")
    ap.add_argument("--model", required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--engine-kw", default="{}")
    a = ap.parse_args(argv)
    eng = build_engine(a.model, a.rank, a.world, **json.loads(a.engine_kw))
    try:
        eng.follow_forever()
    finally:
        eng.runner.close()


if __name__ == "__main__":
    main()
