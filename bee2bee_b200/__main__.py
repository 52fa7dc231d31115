"""``bee2bee`` command line (parity: /root/reference/bee2bee/__main__.py:30-123).

Same verbs and options (``serve-ollama``, ``serve-hf``, ``serve-hf-remote``, ``register``)
plus what a H100 deployment needs: ``--pieces`` (layer pieces = GPUs), ``config``,
``topology``, ``bench``.  ``register``'s handshake test really connects and measures a ping
round-trip (the reference sleeps 1.5 s and prints success).
"""
from __future__ import annotations

import asyncio
import json
import os
import sys
import time

import click

try:
    from dotenv import load_dotenv

    load_dotenv()
except Exception:  # pragma: no cover
    pass

from .config import get_bootstrap_url, load_config, set_bootstrap_url, save_config


def _configure_logging() -> None:
    try:
        from loguru import logger

        logger.remove()
        logger.add(sys.stderr, level=os.getenv("LOG_LEVEL", "INFO"))
        log_dir = os.environ.get("BEE2BEE_LOG_DIR")
        if log_dir is not None or os.access(".", os.W_OK):
            logger.add(os.path.join(log_dir or ".", "bee2bee.log"), rotation="10 MB", level="DEBUG")
    except Exception:
        pass


@click.group()
def cli():
    """Bee2Bee on H100: peer-mesh inference over NVLink."""
    _configure_logging()


def _serve(**kw):
    from .p2p_runtime import run_p2p_node

    try:
        asyncio.run(run_p2p_node(**kw))
    except KeyboardInterrupt:
        pass


@cli.command("serve-ollama")
@click.option("--model", default="llama3", help="Ollama model name")
@click.option("--host", default="0.0.0.0", help="Bind host")
@click.option("--port", default=0, type=int, help="Bind port")
@click.option("--public-host", default=None, help="Public IP/Hostname")
@click.option("--region", default="Auto", help="Region name")
@click.option("--api-port", default=8000, type=int, help="FastAPI port for local access")
@click.option("--pieces", default=1, type=int, help="layer pieces (GPUs) for the embedded engine")
@click.option("--random-weights", is_flag=True, help="embedded engine: allow random-init weights when no checkpoint exists")
def serve_ollama(model, host, port, public_host, region, api_port, pieces, random_weights):
    """Serve a model with the Ollama API shape (daemon if reachable, else the embedded engine)."""
    if random_weights:
        os.environ["B2B_ALLOW_RANDOM_WEIGHTS"] = "1"
    _serve(host=host, port=port, bootstrap_link=get_bootstrap_url(), model_name=model, backend="ollama",
           announce_host=public_host, region=region, api_port=api_port, service_kw={"pieces": pieces})


@cli.command("serve-hf")
@click.option("--model", default="distilgpt2", help="HF model name / preset / local directory")
@click.option("--port", default=0, type=int, help="Bind port")
@click.option("--region", default="Auto", help="Region name")
@click.option("--api-port", default=8000, type=int, help="FastAPI port")
@click.option("--pieces", default=1, type=int, help="split the model into this many layer pieces (one GPU each)")
@click.option("--max-batch", default=None, type=int, help="concurrent sequences (continuous batching)")
@click.option("--max-seq-len", default=None, type=int, help="context budget per sequence")
@click.option("--random-weights", is_flag=True, help="allow random-init weights when --model is not a local checkpoint "
                                                     "directory (benchmarks / smoke tests: the node serves noise)")
@click.option("--supervised", is_flag=True, help="run the engine (one worker process per GPU piece) as a restartable child "
                                                 "group: a dead rank is replaced without restarting this node")
def serve_hf(model, port, region, api_port, pieces, max_batch, max_seq_len, random_weights, supervised):
    """Serve a Hugging Face model on the native engine with built-in FastAPI."""
    if random_weights:
        os.environ["B2B_ALLOW_RANDOM_WEIGHTS"] = "1"      # inherited by the follower ranks of --pieces N
    if supervised:
        os.environ["B2B_SUPERVISED"] = "1"                # hf.load_model_and_tokenizer puts the engine behind the supervisor
    kw = {}
    if max_batch:
        kw["max_batch"] = max_batch
    if max_seq_len:
        kw["max_seq_len"] = max_seq_len
    _serve(port=port, bootstrap_link=get_bootstrap_url(), model_name=model, backend="hf", region=region,
           api_port=api_port, pieces=pieces, service_kw=kw)


@cli.command("serve-hf-remote")
@click.option("--model", default="meta-llama/Llama-2-7b-hf", help="HF model name")
@click.option("--token", required=True, help="HF API Token")
@click.option("--region", default="Cloud", help="Region name")
@click.option("--api-port", default=8000, type=int, help="FastAPI port")
def serve_hf_remote(model, token, region, api_port):
    """Serve via the HF Inference API with a local FastAPI proxy."""
    os.environ["HUGGING_FACE_HUB_TOKEN"] = token
    _serve(bootstrap_link=get_bootstrap_url(), model_name=model, backend="hf_remote", region=region,
           api_port=api_port, token=token)


async def _handshake(addr: str, timeout: float = 5.0) -> float:
    """Connect, exchange hello, measure one ping round trip (ms)."""
    from .p2p_runtime import P2PNode

    probe = P2PNode(host="127.0.0.1", port=0, transport="inproc" if addr.startswith("inproc://") else "ws")
    await probe.start()
    try:
        await probe._connect_peer(addr)
        t0 = time.time()
        while time.time() - t0 < timeout:
            for info in probe.peers.values():
                if info.get("last_pong_at"):
                    return float(info.get("last_pong_ms") or 0.0)
            await asyncio.sleep(0.05)
        raise TimeoutError("no pong")
    finally:
        await probe.stop()


@cli.command()
@click.option("--node-url", default=None, help="Specific Node URL to register")
@click.option("--network", default="connectit", help="Network name")
@click.option("--region", prompt="Node Region", default="US-West")
@click.option("--test/--no-test", default=True, help="Run handshake test")
def register(node_url, network, region, test):
    """Register a node manually or via handshake test."""
    from .p2p_runtime import P2PNode
    from .registry import RegistryClient

    async def _reg() -> int:
        click.echo("Bee2Bee Node Registration")
        target, peer_id, node = node_url, f"ext-{os.urandom(4).hex()}", None
        if not target:
            node = P2PNode(host="127.0.0.1", port=0)
            await node.start()
            target, peer_id = node.addr, node.peer_id
        click.echo(f"Target Region: {region}")
        click.echo(f"Node Address: {target}")
        ok = True
        if test:
            try:
                rtt = await _handshake(target)
                click.echo(f"Handshake OK ({rtt:.2f} ms round trip)")
            except Exception as exc:
                ok = False
                click.echo(f"Handshake FAILED: {exc}")
        reg = RegistryClient()
        synced = False
        if ok:
            synced = await reg.sync_node(peer_id=peer_id, address=target,
                                         models=["manual-entry" if node_url else "system-test"],
                                         tag=f"cli-{network}", region=region)
        if synced:
            click.echo("Node Registered Successfully!")
        elif ok and not reg.enabled:
            click.echo("Registry unavailable (offline mode): row recorded in $BEE2BEE_HOME/registry.json")
        elif ok:
            click.echo("Registry rejected the registration")
        if node is not None:
            await node.stop()
        return 0 if ok else 1

    sys.exit(asyncio.run(_reg()))


@cli.command()
@click.option("--host", default="0.0.0.0", help="Bind host")
@click.option("--port", default=None, type=int, help="HTTP port (default: $API_PORT or 3000)")
@click.option("--seed", "seeds", multiple=True, help="Node address or join link to dial at start-up (repeatable; "
              "default: $BEE2BEE_SEEDS)")
def gateway(host, port, seeds):
    """Web gateway: /api/p2p/{register,generate,status,global_metrics} + a minimal chat page
    (the reference's Express app + bridge, app/api/index.js / bridge.js)."""
    from .gateway import main as gateway_main

    gateway_main(host=host, port=port, seeds=list(seeds) or None)


@cli.command("config")
@click.argument("key", required=False)
@click.argument("value", required=False)
def config_cmd(key, value):
    """Show the config, or set KEY VALUE (e.g. ``config bootstrap_url ws://host:4003``)."""
    cfg = load_config()
    if key is None:
        click.echo(json.dumps(cfg, indent=2))
        return
    if value is None:
        click.echo(json.dumps(cfg.get(key)))
        return
    if key == "bootstrap_url":
        set_bootstrap_url(value)
    else:
        cfg[key] = value
        save_config(cfg)
    click.echo(f"{key} = {load_config().get(key)!r}")


@cli.command()
@click.option("--model", default=None, help="also print how this model (preset / alias / local directory) is cut into pieces")
@click.option("--pieces", default=0, type=int, help="number of pieces (GPUs) for --model; default: the GPUs of this box")
def topology(model, pieces):
    """Print the local NVLink topology table (devices, peer access) and, with --model, the piece plan."""
    import torch

    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    out = {"devices": n, "names": [torch.cuda.get_device_name(i) for i in range(n)], "can_access_peer": []}
    if n:
        from . import ops

        C = ops.native()
        out["can_access_peer"] = [[bool(i == j or C.can_access_peer(i, j)) for j in range(n)] for i in range(n)]
    if model:
        from .models.config import UNITS_PER_LAYER, piece_units, resolve_config, unit_layers

        cfg = resolve_config(model)
        kinds = ("attention block (QKV, attention, O-proj)", "gate/up GEMM", "down GEMM")
        plan = piece_units(cfg, pieces or max(1, n))
        out["model"] = {"name": cfg.name, "layers": cfg.n_layers, "hidden": cfg.hidden_size, "ffn": cfg.ffn_size,
                        "vocab": cfg.vocab_size}
        out["pieces"] = [{"piece": i, "units": [u0, u1], "n_units": u1 - u0,
                          "layers": [min(unit_layers((u0, u1))), max(unit_layers((u0, u1)))],
                          "head_gemm_of": kinds[u0 % UNITS_PER_LAYER], "tail_gemm_of": kinds[(u1 - 1) % UNITS_PER_LAYER],
                          "extras": (["embedding"] if i == 0 else []) + (["lm_head", "sampler"] if i == len(plan) - 1 else [])}
                         for i, (u0, u1) in enumerate(plan)]
    click.echo(json.dumps(out, indent=2))


@cli.command(context_settings={"ignore_unknown_options": True})
@click.argument("args", nargs=-1, type=click.UNPROCESSED)
def bench(args):
    """Run the headline benchmark (forwards to bench.py at the repo root)."""
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.exit(subprocess.call([sys.executable, os.path.join(root, "bench.py"), *args]))


if __name__ == "__main__":
    cli()
