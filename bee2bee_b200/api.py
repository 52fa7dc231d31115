"""HTTP sidecar (parity: /root/reference/bee2bee/api.py): ``/``, ``/peers``, ``/providers``,
``/connect``, ``/chat`` == ``/generate`` with the reference's JSON shapes, ``X-API-KEY`` auth
iff ``BEE2BEE_API_KEY`` is set, CORS from ``CORS_ORIGINS``.

Re-designed where the reference is unsound: request handlers only *enqueue* into the
engine and ``await`` (the reference calls the blocking ``svc.execute`` inside ``async def``
and stalls every WebSocket ping and HTTP request for the whole generation, api.py:229);
``temperature=0`` stays 0 (reference: ``temperature or 0.7``); ``uptime`` is real.
Extra read-only routes: ``/metrics`` (engine counters), ``/topology`` (mesh / piece table).
"""
from __future__ import annotations

import asyncio
import os
import time
from contextlib import asynccontextmanager
from typing import Any, Dict, List, Optional

from fastapi import Depends, FastAPI, HTTPException, status
from fastapi.middleware.cors import CORSMiddleware
from fastapi.responses import StreamingResponse
from fastapi.security import APIKeyHeader
from pydantic import BaseModel

from .p2p_runtime import P2PNode
from .services import sampling_filters
from .utils import now_ms

try:
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("bee2bee")

#: shared with ``run_p2p_node`` (the launcher seeds it before uvicorn starts in the same loop)
node: Optional[P2PNode] = None
_owned_node = False

API_KEY_NAME = "X-API-KEY"
api_key_header = APIKeyHeader(name=API_KEY_NAME, auto_error=False)


async def get_api_key(header_key: Optional[str] = Depends(api_key_header)):
    expected = os.getenv("BEE2BEE_API_KEY")
    if not expected:
        return None                       # open API when no key is configured
    if header_key == expected:
        return header_key
    raise HTTPException(status_code=status.HTTP_401_UNAUTHORIZED, detail="Invalid or missing API Key")


@asynccontextmanager
async def lifespan(app: FastAPI):
    global node, _owned_node
    if node is None:
        ann_port = os.getenv("BEE2BEE_ANNOUNCE_PORT")
        node = P2PNode(host=os.getenv("BEE2BEE_HOST", "0.0.0.0"), port=int(os.getenv("BEE2BEE_PORT", "4001")),
                       announce_host=os.getenv("BEE2BEE_ANNOUNCE_HOST"),
                       announce_port=int(ann_port) if ann_port else None,
                       transport=os.getenv("BEE2BEE_TRANSPORT", "ws"))
        await node.start()
        _owned_node = True
    bootstrap = os.getenv("BEE2BEE_BOOTSTRAP")
    if bootstrap:
        try:
            await node.connect_bootstrap(bootstrap)
        except Exception as exc:
            logger.warning(f"bootstrap failed: {exc}")
    await node.enable_monitoring(interval_seconds=15)
    logger.info(f"API sidecar attached to node {node.peer_id} at {node.addr} "
                f"(auth {'on' if os.getenv('BEE2BEE_API_KEY') else 'off'})")
    yield
    if node is not None and _owned_node:
        await node.stop()
        node = None
        _owned_node = False


app = FastAPI(title="Bee2Bee Node API", lifespan=lifespan)
app.add_middleware(CORSMiddleware, allow_origins=os.getenv("CORS_ORIGINS", "*").split(","), allow_credentials=True,
                   allow_methods=["*"], allow_headers=["*"])


class PeerInfo(BaseModel):
    peer_id: str
    addr: Optional[str]
    latency_ms: Optional[float]


class ProviderInfo(BaseModel):
    peer_id: str
    addr: Optional[str]
    latency_ms: Optional[float]
    models: List[str]
    price_per_token: Optional[float]
    tag: Optional[str] = None


class ChatRequest(BaseModel):
    provider_id: Optional[str] = "local"
    prompt: str
    model: Optional[str] = None
    max_new_tokens: Optional[int] = None
    temperature: Optional[float] = 0.7
    stream: Optional[bool] = False
    top_k: Optional[int] = None       # keep the k most likely tokens; absent = off
    min_p: Optional[float] = None     # keep tokens with p >= min_p * p_max; absent = off
    presence_penalty: Optional[float] = None    # in [-2, 2], subtracted from every generated token; absent = off
    frequency_penalty: Optional[float] = None   # in [-2, 2], times each generated token's count; absent = off
    logit_bias: Optional[Dict[str, float]] = None   # token id (decimal string) -> bias in [-100, 100]; absent = off


@app.get("/")
def home() -> Dict[str, Any]:
    if node is None:
        return {"status": "starting", "node_id": "not_started"}
    services, models = {}, []
    for name, svc in node.local_services.items():
        meta = svc.get_metadata()
        services[name] = meta
        models.extend(meta.get("models") or [])
    return {"status": "ok", "node_id": node.peer_id, "peer_id": node.peer_id, "region": node.region,
            "models": sorted(set(models)), "services": services,
            "metrics": {"uptime": round(node.uptime(), 1), "pool_size": len(node.peers), "status": "active"}}


@app.get("/peers", dependencies=[Depends(get_api_key)])
def peers() -> List[Dict[str, Any]]:
    if node is None:
        return []
    return [{"peer_id": pid, "addr": info.get("addr"), "latency_ms": info.get("last_pong_ms"),
             "health_status": info.get("health_status", "unknown"), "last_audit": info.get("last_audit"),
             "metrics": info.get("metrics")} for pid, info in list(node.peers.items())]


@app.get("/providers", response_model=List[ProviderInfo], dependencies=[Depends(get_api_key)])
def providers():
    return node.list_providers() if node is not None else []


@app.get("/connect", dependencies=[Depends(get_api_key)])
async def connect_peer(addr: str) -> Dict[str, Any]:
    if node is None:
        return {"status": "error", "message": "node not started"}
    try:
        if "://join?" in addr or addr.startswith("p2pnet"):
            ok = await node.connect_bootstrap(addr)
            if not ok:
                return {"status": "error", "message": "no bootstrap address reachable"}
        else:
            await node._connect_peer(addr)
        return {"status": "connected", "addr": addr}
    except Exception as exc:
        return {"status": "error", "message": str(exc)}


def _engine_metrics() -> Dict[str, Any]:
    out: Dict[str, Any] = {}
    if node is None:
        return out
    for name, svc in node.local_services.items():
        eng = getattr(getattr(svc, "model", None), "engine", None)
        if eng is not None:
            out[name] = eng.metrics()
    return out


def prometheus_text(per_service: Dict[str, Any]) -> str:
    """Engine counters in the Prometheus text exposition format (scalars only; nested dicts are flattened with '_')."""
    lines = []

    def emit(service: str, key: str, val) -> None:
        if isinstance(val, bool):
            val = int(val)
        if isinstance(val, (int, float)):
            name = "bee2bee_" + "".join(c if c.isalnum() else "_" for c in key)
            lines.append(f'{name}{{service="{service}"}} {float(val):.6g}')
        elif isinstance(val, dict):
            for k, v in val.items():
                emit(service, f"{key}_{k}", v)

    for service, m in per_service.items():
        for key, val in m.items():
            if key != "trace":
                emit(service, key, val)
    return "\n".join(lines) + "\n"


@app.get("/metrics", dependencies=[Depends(get_api_key)])
def metrics(format: Optional[str] = None):
    """Engine counters per local service (JSON); ``?format=prometheus`` for the text exposition format."""
    data = _engine_metrics()
    if format == "prometheus":
        from fastapi.responses import PlainTextResponse
        return PlainTextResponse(prometheus_text(data), media_type="text/plain; version=0.0.4")
    return data


@app.get("/topology", dependencies=[Depends(get_api_key)])
def topology() -> Dict[str, Any]:
    return node.mesh_topology() if node is not None else {}


@app.post("/chat", dependencies=[Depends(get_api_key)])
@app.post("/generate", dependencies=[Depends(get_api_key)])
async def chat(req: ChatRequest):
    """Local service when one serves the model (exact or substring match either way), else a mesh
    provider.  Failures come back as HTTP 200 ``{"status": "error"}`` like the reference."""
    if node is None:
        return {"status": "error", "message": "node not started"}
    params = {"prompt": req.prompt, "max_new_tokens": req.max_new_tokens or 2048,
              "temperature": 0.7 if req.temperature is None else req.temperature}
    try:
        filters = sampling_filters({"top_k": req.top_k, "min_p": req.min_p, "presence_penalty": req.presence_penalty,
                                    "frequency_penalty": req.frequency_penalty, "logit_bias": req.logit_bias})
        params.update(filters)
        t0 = time.time()
        want_local = req.provider_id in (None, "local", node.peer_id)
        svc = None
        if want_local:
            for cand in node.local_services.values():
                if cand.serves(req.model):
                    svc = cand
                    break
        if svc is not None:
            if req.stream:
                return StreamingResponse(svc.aexecute_stream(params), media_type="text/plain")
            result = await svc.aexecute(params)
            return {"status": "ok", "text": result.get("text", ""), "rid": f"local-{now_ms()}",
                    "metadata": {"engine": "coithub-local", "node": node.peer_id, "service": svc.name,
                                 "latency_ms": result.get("latency_ms", int((time.time() - t0) * 1000)),
                                 "tokens": result.get("tokens")}}
        pid = req.provider_id if req.provider_id not in (None, "local") else None
        if pid is None and req.model:
            picked = node.pick_provider(req.model)
            pid = picked[0] if picked else None
        if pid is None:
            return {"status": "error", "message": f"no provider for model {req.model!r}"}
        if req.stream:
            q: asyncio.Queue = asyncio.Queue()

            async def relay():
                try:
                    await node.request_generation(pid, req.prompt, params["max_new_tokens"], req.model,
                                                  temperature=params["temperature"], stream=True,
                                                  on_chunk=q.put_nowait, **filters)
                finally:
                    q.put_nowait(None)

            task = asyncio.create_task(relay())

            async def body():
                import json as _json
                while True:
                    item = await q.get()
                    if item is None:
                        break
                    yield _json.dumps({"text": item}) + "\n"
                if task.done() and task.exception():
                    yield _json.dumps({"status": "error", "message": str(task.exception())}) + "\n"
                yield _json.dumps({"done": True}) + "\n"

            return StreamingResponse(body(), media_type="text/plain")
        result = await node.request_generation(pid, req.prompt, params["max_new_tokens"], req.model,
                                               temperature=params["temperature"], **filters)
        return {"status": "ok", "text": result.get("text", ""), "rid": f"p2p-{now_ms()}",
                "metadata": {"engine": "coithub-p2p", "node": pid,
                             "latency_ms": result.get("latency_ms", int((time.time() - t0) * 1000))}}
    except Exception as exc:
        return {"status": "error", "message": str(exc)}


def main() -> None:
    import uvicorn

    uvicorn.run(app, host=os.getenv("BEE2BEE_API_HOST", "0.0.0.0"), port=int(os.getenv("BEE2BEE_API_PORT", "4002")))


if __name__ == "__main__":
    main()
