"""Legacy coordinator/worker protocol (parity: /root/reference/bee2bee/node.py:38-294,
constants in protocol.py).  The reference ships only the *worker* half -- its coordinator no
longer exists, so nothing can drive it.  Here:

* ``TaskExecutor``  executes every task kind the reference worker understands
  (``layer_forward``, ``layer_forward_train``, ``layer_backward``, ``hf_load/infer/unload``,
  ``onnx_load/infer/unload``, ``hf_part_load/forward``) -- dense layers on the GPU when present,
  ``hf_part_*`` generalised from DistilBERT to decoder LMs with a per-session KV cache, hidden
  states accepted/returned as binary payloads (JSON lists still accepted for wire compat);
* ``node_client`` / ``run_node``  the reconnecting WebSocket worker (REGISTER -> INFO -> TASK loop);
* ``Coordinator``  the missing other half: worker registry + ``run_pipeline`` /
  ``run_train_step`` / ``run_hf_pipeline`` built on TASK/RESULT frames, so the protocol
  constants that have no implementation anywhere in the reference are actually usable.

On a H100 mesh the product path does not use any of this (pieces hand off over NVLink);
it is kept for surface parity and as a CPU-cluster fallback.
"""
from __future__ import annotations

import asyncio
import json
import platform
from typing import Any, Dict, List, Optional

import numpy as np

from . import protocol as P
from .model import (Layer, dense_backward_device, dense_forward_device, deserialize_layer, layer_backward,
                    layer_forward, layer_forward_train, serialize_layer)
from .utils import new_id

try:
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("bee2bee")


def gather_resources() -> Dict[str, Any]:
    import psutil

    mem = psutil.virtual_memory()
    res: Dict[str, Any] = {"os": platform.system(), "cpu_count": psutil.cpu_count(logical=True),
                           "memory_gb": round(mem.total / (1024 ** 3), 2), "gpu": False}
    try:
        import torch

        if torch.cuda.is_available():
            res["gpu"] = True
            res["gpus"] = [{"name": torch.cuda.get_device_name(i),
                            "memory_gb": round(torch.cuda.get_device_properties(i).total_memory / (1024 ** 3), 1)}
                           for i in range(torch.cuda.device_count())]
    except Exception:
        pass
    return res


class TaskError(Exception):
    pass


class TaskExecutor:
    """Stateless dispatch + the worker-side state (train caches, loaded models)."""

    def __init__(self, device: Optional[str] = None):
        try:
            import torch

            self.device = device or ("cuda" if torch.cuda.is_available() else "cpu")
        except Exception:
            self.device = "cpu"
        self.caches: Dict[str, Dict[str, Any]] = {}
        self.models: Dict[str, Dict[str, Any]] = {}

    # ---- dense layers (K12) -------------------------------------------------------------
    def _t_layer_forward(self, p):
        layer = deserialize_layer(p["layer"])
        x = np.asarray(p["x"], dtype=np.float32)
        if self.device.startswith("cuda"):
            y, _ = dense_forward_device(layer.W, layer.b, layer.activation, x, self.device)
            return {"output": y.cpu().numpy().tolist()}
        return {"output": layer_forward(layer, x).tolist()}

    def _t_layer_forward_train(self, p):
        layer = deserialize_layer(p["layer"])
        x = np.asarray(p["x"], dtype=np.float32)
        cache_id = p.get("cache_id") or new_id("cache")
        if self.device.startswith("cuda"):
            y, z = dense_forward_device(layer.W, layer.b, layer.activation, x, self.device)
            self.caches[cache_id] = {"x": x, "z": z.cpu().numpy(), "layer": layer}
            return {"output": y.cpu().numpy().tolist(), "cache_id": cache_id}
        y, z = layer_forward_train(layer, x)
        self.caches[cache_id] = {"x": x, "z": z, "layer": layer}
        return {"output": y.tolist(), "cache_id": cache_id}

    def _t_layer_backward(self, p):
        cache = self.caches.pop(p.get("cache_id"), None)
        if cache is None:
            raise TaskError("cache_missing")
        up = np.asarray(p["upstream_grad"], dtype=np.float32)
        layer: Layer = cache["layer"]
        if self.device.startswith("cuda"):
            gX, gW, gb = dense_backward_device(layer.W, layer.activation, cache["x"], cache["z"], up, self.device)
            gX, gW, gb = gX.cpu().numpy(), gW.cpu().numpy(), gb.cpu().numpy()
        else:
            gX, gW, gb = layer_backward(layer, cache["x"], cache["z"], up)
        return {"dX": gX.tolist(), "gW": gW.tolist(), "gb": gb.tolist()}

    # ---- whole-model HF tasks ---------------------------------------------------------------
    def _t_hf_load(self, p):
        from .hf import load_model_and_tokenizer

        name = p.get("model_name")
        if not name:
            raise TaskError("model_name_missing")
        model_id = p.get("model_id") or new_id("hf")
        mdl, tok, dev = load_model_and_tokenizer(name, max_batch=4, max_seq_len=512)
        self.models[model_id] = {"kind": "hf", "model": mdl, "tok": tok, "device": dev}
        return {"model_id": model_id}

    def _t_hf_infer(self, p):
        from .hf import generate_text

        ent = self.models.get(p.get("model_id"))
        if not ent or ent["kind"] != "hf":
            raise TaskError("model_not_loaded")
        txt = generate_text(ent["model"], ent["tok"], ent["device"], p.get("prompt") or "",
                            int(p.get("max_new_tokens", 32)), temperature=float(p.get("temperature", 0.7)))
        return {"text": txt}

    def _t_unload(self, p):
        self.models.pop(p.get("model_id"), None)
        return {"ok": True}

    # ---- ONNX (optional dependency, as in the reference) ----------------------------------
    def _t_onnx_load(self, p):
        try:
            import onnxruntime as ort  # type: ignore
        except Exception:
            raise TaskError("onnx_support_missing")
        model_id = p.get("model_id") or new_id("onnx")
        self.models[model_id] = {"kind": "onnx", "session": ort.InferenceSession(p.get("path"))}
        return {"model_id": model_id}

    def _t_onnx_infer(self, p):
        ent = self.models.get(p.get("model_id"))
        if not ent or ent["kind"] != "onnx":
            raise TaskError("onnx_model_not_loaded")
        feeds = {k: np.asarray(v) for k, v in (p.get("inputs") or {}).items()}
        out = ent["session"].run(None, feeds)
        return {"outputs": [o.tolist() if hasattr(o, "tolist") else o for o in out]}

    # ---- partitioned model: layer range [start, end) ------------------------------------------
    def _t_hf_part_load(self, p):
        from .models.config import resolve_config

        name = p.get("model_name", "distilgpt2")
        cfg = resolve_config(name)
        start, end = int(p.get("start", 0)), int(p.get("end", cfg.n_layers))
        model_id = p.get("model_id") or new_id("hfpart")
        device = str(p.get("device") or self.device)
        if device.startswith("cuda") and cfg.norm == "rms" and cfg.glu:
            # H100 data plane: the layer range runs on the hand-written kernels with a paged KV cache, and hop payloads
            # may stay in device memory (hidden_ref: cudaMemcpyPeerAsync / CUDA IPC instead of JSON lists)
            import torch
            from .engine.tokenizer import load_tokenizer
            from .parallel.gpu_piece import GpuPieceHost

            if device == "cuda":
                device = f"cuda:{torch.cuda.current_device()}"
            host = GpuPieceHost(name, start, end, device=device, max_tokens=int(p.get("max_tokens", 512)),
                                max_seq_len=int(p.get("max_seq_len", 1024)))
            tok = load_tokenizer(name, cfg.vocab_size, cfg.eos_token_id, cfg.bos_token_id)
            self.models[model_id] = {"kind": "hf_part_gpu", "host": host, "tok": tok, "cfg": cfg}
            return {"model_id": model_id, "start": start, "end": min(end, cfg.n_layers), "device": device,
                    "backend": "b200-native"}
        from .hf import build_layer_partial

        piece, tok, dev = build_layer_partial(name, start, end, device="cpu")
        self.models[model_id] = {"kind": "hf_part", "piece": piece, "tok": tok, "sessions": {}, "cfg": cfg}
        return {"model_id": model_id, "start": start, "end": min(end, cfg.n_layers)}

    def _t_hf_part_forward(self, p):
        import torch

        from .parallel.cpu_pipeline import decode_tensor, encode_tensor

        ent = self.models.get(p.get("model_id"))
        if ent and ent["kind"] == "hf_part_gpu":
            return self._hf_part_forward_gpu(ent, p)
        if not ent or ent["kind"] != "hf_part":
            raise TaskError("model_not_loaded")
        piece, tok = ent["piece"], ent["tok"]
        session = p.get("session")
        cache = ent["sessions"].setdefault(session, piece.new_cache()) if session else None
        if p.get("text") is not None:
            ids = tok.encode(p["text"])
            x = torch.tensor([ids])
        elif p.get("hidden_b64") is not None:
            x = decode_tensor(p["hidden_b64"])
        elif p.get("hidden") is not None:
            x = torch.tensor(np.asarray(p["hidden"], dtype=np.float32))
        elif p.get("ids") is not None:
            x = torch.tensor([list(p["ids"])])
        else:
            raise TaskError("no_input")
        T = x.shape[1]
        pos0 = int(p.get("pos0", 0))
        pos = torch.arange(pos0, pos0 + T)[None]
        with torch.no_grad():
            y = piece.forward(x, pos, cache)
        if p.get("binary", False):
            return {"hidden_b64": encode_tensor(y)}
        return {"hidden": y.float().numpy().tolist()}

    def _hf_part_forward_gpu(self, ent, p):
        """hf_part_forward on a GPU-resident piece.  Input: text / ids (first piece), ``hidden_ref`` (device-resident
        payload of the previous hop: peer copy over NVLink, same or other process), or the legacy hidden / hidden_b64
        frames.  Output: ``hidden_ref`` when ``keep_on_device`` (the frame then carries ~100 bytes), else the legacy
        encodings; the last piece returns the logits of the final position."""
        import torch

        from .parallel.cpu_pipeline import decode_tensor, encode_tensor
        from .parallel.gpu_piece import release_buffer

        host, tok = ent["host"], ent["tok"]
        ids, hidden = None, None
        if p.get("text") is not None:
            ids = tok.encode(p["text"])
        elif p.get("ids") is not None:
            ids = [int(t) for t in p["ids"]]
        elif p.get("hidden_ref") is not None:
            hidden = host.load_hidden_ref(p["hidden_ref"])
            if p.get("release_ref", True):
                release_buffer(p["hidden_ref"].get("ref", ""))
        elif p.get("hidden_b64") is not None:
            hidden = host.load_hidden_host(decode_tensor(p["hidden_b64"]))
        elif p.get("hidden") is not None:
            hidden = host.load_hidden_host(torch.tensor(np.asarray(p["hidden"], dtype=np.float32)))
        else:
            raise TaskError("no_input")
        res = host.forward(p.get("session"), ids=ids, hidden=hidden, pos0=p.get("pos0"),
                           keep_on_device=bool(p.get("keep_on_device")))
        if "hidden_ref" in res:
            return {"hidden_ref": res["hidden_ref"]}
        y = res["logits"][None] if "logits" in res else res["hidden"][None]          # [1, T, H] / [1, 1, V]
        if p.get("binary", False):
            return {"hidden_b64": encode_tensor(y.cpu())}
        return {"hidden": y.float().cpu().numpy().tolist()}

    DISPATCH = {
        P.TASK_LAYER_FORWARD: "_t_layer_forward", P.TASK_LAYER_FORWARD_TRAIN: "_t_layer_forward_train",
        P.TASK_LAYER_BACKWARD: "_t_layer_backward", P.HF_LOAD: "_t_hf_load", P.HF_INFER: "_t_hf_infer",
        P.HF_UNLOAD: "_t_unload", P.ONNX_LOAD: "_t_onnx_load", P.ONNX_INFER: "_t_onnx_infer",
        P.ONNX_UNLOAD: "_t_unload", P.HF_PART_LOAD: "_t_hf_part_load", P.HF_PART_FORWARD: "_t_hf_part_forward",
    }

    def execute(self, payload: Dict[str, Any]) -> Dict[str, Any]:
        kind = payload.get("kind")
        name = self.DISPATCH.get(kind)
        if name is None:
            raise TaskError(f"unknown_task:{kind}")
        return getattr(self, name)(payload)


async def handle_task_frame(executor: TaskExecutor, data: Dict[str, Any]) -> Dict[str, Any]:
    """TASK frame -> RESULT / ERROR frame (compute runs off-loop)."""
    task_id = data.get("task_id")
    try:
        res = await asyncio.get_running_loop().run_in_executor(None, executor.execute, data.get("payload") or {})
        return P.msg(P.RESULT, task_id=task_id, **res)
    except Exception as exc:
        return P.msg(P.ERROR, task_id=task_id, error=str(exc))


async def node_client(coordinator_url: str, node_name: Optional[str] = None, price: float = 0.0,
                      max_reconnects: Optional[int] = None) -> None:
    """Worker loop: REGISTER, then serve TASK frames; reconnect with capped exponential back-off
    (the reference retries every 2 s forever)."""
    from .transport import connect

    executor = TaskExecutor()
    attempt = 0
    while max_reconnects is None or attempt <= max_reconnects:
        try:
            conn = await connect(coordinator_url)
            attempt = 0
            await conn.send(json.dumps(P.msg(P.REGISTER, node_id=new_id("node"), name=node_name or platform.node(),
                                             resources=gather_resources(), price=price)))
            async for raw in conn:
                try:
                    data = json.loads(raw)
                except ValueError:
                    continue
                t = data.get("type")
                if t == P.INFO:
                    logger.info(f"registered as {data.get('node_id')}")
                elif t == P.PING:
                    await conn.send(json.dumps(P.msg(P.PONG, ts=data.get("ts"))))
                elif t == P.TASK:
                    await conn.send(json.dumps(await handle_task_frame(executor, data)))
        except asyncio.CancelledError:
            raise
        except Exception as exc:
            logger.debug(f"coordinator link lost: {exc}")
        attempt += 1
        await asyncio.sleep(min(30.0, 2.0 * (1.5 ** min(attempt, 8))))


def run_node(coordinator_url: str, node_name: Optional[str] = None, price: float = 0.0) -> None:
    asyncio.run(node_client(coordinator_url, node_name, price))


# ===================================================================================== coordinator
class Coordinator:
    """Minimal coordinator: accepts worker registrations and drives them with TASK frames."""

    def __init__(self, host: str = "127.0.0.1", port: int = 0, transport: str = "ws", name: str = "coordinator"):
        self.host, self.port, self.transport, self.name = host, port, transport, name
        self.workers: Dict[str, Dict[str, Any]] = {}
        self._pending: Dict[str, asyncio.Future] = {}
        self.hop_log: List[Dict[str, Any]] = []        # per hop of the last hf pipeline: on-device or framed, frame size
        self._server = None
        self.addr = ""

    async def start(self) -> str:
        from .transport import InProcHub, ws_listen

        if self.transport == "inproc":
            self.addr = InProcHub.listen(self.name, self._on_worker)
        else:
            self._server = await ws_listen(self.host, self.port, self._on_worker)
            self.port = self._server.port
            self.addr = f"ws://{self.host}:{self.port}"
        return self.addr

    async def stop(self) -> None:
        from .transport import InProcHub

        for w in self.workers.values():
            try:
                await w["conn"].close()
            except Exception:
                pass
        self.workers.clear()
        if self._server is not None:
            await self._server.close()
        if self.addr.startswith("inproc://"):
            InProcHub.unlisten(self.name)

    async def _on_worker(self, conn) -> None:
        node_id = None
        try:
            async for raw in conn:
                data = json.loads(raw)
                t = data.get("type")
                if t == P.REGISTER:
                    node_id = data.get("node_id") or new_id("node")
                    self.workers[node_id] = {"conn": conn, "name": data.get("name"), "resources": data.get("resources"),
                                             "price": data.get("price", 0.0)}
                    await conn.send(json.dumps(P.msg(P.INFO, node_id=node_id)))
                elif t in (P.RESULT, P.ERROR):
                    fut = self._pending.pop(data.get("task_id"), None)
                    if fut is not None and not fut.done():
                        fut.set_result(data)
        except Exception:
            pass
        finally:
            if node_id:
                self.workers.pop(node_id, None)

    def list_nodes(self) -> List[Dict[str, Any]]:
        return [{"node_id": k, "name": v["name"], "resources": v["resources"], "price": v["price"]}
                for k, v in self.workers.items()]

    async def wait_for_workers(self, n: int, timeout: float = 10.0) -> None:
        t0 = asyncio.get_running_loop().time()
        while len(self.workers) < n:
            if asyncio.get_running_loop().time() - t0 > timeout:
                raise TimeoutError(f"{len(self.workers)}/{n} workers registered")
            await asyncio.sleep(0.02)

    async def submit(self, node_id: str, payload: Dict[str, Any], timeout: float = 120.0) -> Dict[str, Any]:
        w = self.workers.get(node_id)
        if w is None:
            raise KeyError(node_id)
        task_id = new_id("task")
        fut = asyncio.get_running_loop().create_future()
        self._pending[task_id] = fut
        await w["conn"].send(json.dumps(P.msg(P.TASK, task_id=task_id, payload=payload)))
        res = await asyncio.wait_for(fut, timeout)
        if res.get("type") == P.ERROR:
            raise TaskError(res.get("error"))
        return res

    def _cheapest(self) -> List[str]:
        return [k for k, _ in sorted(self.workers.items(), key=lambda kv: kv[1]["price"])]

    async def run_pipeline(self, layers: List[Layer], x: np.ndarray) -> np.ndarray:
        """RUN_PIPELINE: one dense layer per worker (round-robin), activations hop through us."""
        ids = self._cheapest()
        cur = np.asarray(x, dtype=np.float32)
        for i, layer in enumerate(layers):
            res = await self.submit(ids[i % len(ids)], {"kind": P.TASK_LAYER_FORWARD, "layer": serialize_layer(layer),
                                                        "x": cur.tolist()})
            cur = np.asarray(res["output"], dtype=np.float32)
        return cur

    async def run_train_step(self, layers: List[Layer], x: np.ndarray, y: np.ndarray, lr: float = 0.1) -> float:
        """RUN_TRAIN_STEP: split-learning forward (cached) + backward through the same workers,
        MSE loss, SGD update applied to ``layers`` in place. Returns the loss."""
        ids = self._cheapest()
        cur = np.asarray(x, dtype=np.float32)
        caches = []
        for i, layer in enumerate(layers):
            res = await self.submit(ids[i % len(ids)], {"kind": P.TASK_LAYER_FORWARD_TRAIN,
                                                        "layer": serialize_layer(layer), "x": cur.tolist()})
            caches.append((ids[i % len(ids)], res["cache_id"]))
            cur = np.asarray(res["output"], dtype=np.float32)
        diff = cur - np.asarray(y, dtype=np.float32)
        loss = float((diff ** 2).mean())
        grad = 2.0 * diff / diff.size
        for i in range(len(layers) - 1, -1, -1):
            nid, cid = caches[i]
            res = await self.submit(nid, {"kind": P.TASK_LAYER_BACKWARD, "cache_id": cid, "upstream_grad": grad.tolist()})
            layers[i].W -= lr * np.asarray(res["gW"], dtype=np.float32)
            layers[i].b -= lr * np.asarray(res["gb"], dtype=np.float32)
            grad = np.asarray(res["dX"], dtype=np.float32)
        return loss

    async def run_hf_pipeline(self, model_name: str, text: str, n_parts: Optional[int] = None,
                              devices: Optional[List[str]] = None) -> np.ndarray:
        """RUN_HF_PIPELINE: split ``model_name`` into layer ranges over the workers, push ``text``
        through, return the last piece's output (logits of the final position)."""
        from .models.config import resolve_config, split_layers

        ids = self._cheapest()
        cfg = resolve_config(model_name)
        ranges = split_layers(cfg.n_layers, n_parts or len(ids))
        handles = []
        for i, r in enumerate(ranges):
            load = {"kind": P.HF_PART_LOAD, "model_name": model_name, "start": r.start,
                    "end": r.stop if i < len(ranges) - 1 else cfg.n_layers}
            if devices:
                load["device"] = devices[i % len(devices)]
            res = await self.submit(ids[i % len(ids)], load)
            handles.append((ids[i % len(ids)], res["model_id"], res.get("backend") == "b200-native"))
        out, ref = None, None
        for i, (nid, mid, native) in enumerate(handles):
            payload = {"kind": P.HF_PART_FORWARD, "model_id": mid, "binary": True}
            if i == 0:
                payload["text"] = text
            elif ref is not None:
                payload["hidden_ref"] = ref              # ~100-byte frame; the payload moves GPU -> GPU
            else:
                payload["hidden_b64"] = out
            nxt_native = i + 1 < len(handles) and handles[i + 1][2]
            payload["keep_on_device"] = bool(native and nxt_native)
            res = await self.submit(nid, payload)
            ref, out = res.get("hidden_ref"), res.get("hidden_b64")
            self.hop_log.append({"stage": i, "on_device": ref is not None,
                                 "frame_bytes": len(json.dumps(res))})
        from .parallel.cpu_pipeline import decode_tensor

        for nid, mid, _ in handles:
            await self.submit(nid, {"kind": P.HF_UNLOAD, "model_id": mid})
        return decode_tensor(out).float().numpy()[0, -1]
