"""Wire protocol catalogue.

Live mesh protocol (JSON frames with a ``type`` key, parity with the dispatch table at
/root/reference/bee2bee/p2p_runtime.py:460-470) as small typed builders, plus the legacy
coordinator/worker constants of /root/reference/bee2bee/protocol.py:17-53 that ``node.py``
still speaks.  Builders only *construct* dicts -- transports decide how they travel
(WebSocket text frame, in-process queue, ...), and never on the token path.
"""
from __future__ import annotations

import time
from typing import Any, Dict, List, Optional


def msg(type: str, **kwargs) -> Dict[str, Any]:
    out: Dict[str, Any] = {"type": type}
    out.update(kwargs)
    return out


def is_message(obj: Any) -> bool:
    return isinstance(obj, dict) and "type" in obj


# ---- live mesh message types ---------------------------------------------------
HELLO = "hello"
PEER_LIST = "peer_list"
PING = "ping"
PONG = "pong"
SERVICE_ANNOUNCE = "service_announce"
GEN_REQUEST = "gen_request"
GEN_CHUNK = "gen_chunk"
GEN_SUCCESS = "gen_success"
GEN_ERROR = "gen_error"
GEN_RESULT = "gen_result"
PIECE_REQUEST = "piece_request"
PIECE_DATA = "piece_data"
# NVLink-mesh extensions (new in this framework)
PIECE_ANNOUNCE = "piece_announce"     # a peer advertises the layer piece it hosts
HIDDEN_FORWARD = "hidden_forward"     # CPU/loopback fallback for the activation hop
HIDDEN_RESULT = "hidden_result"

LIVE_TYPES = (HELLO, PEER_LIST, PING, PONG, SERVICE_ANNOUNCE, GEN_REQUEST, GEN_CHUNK, GEN_SUCCESS, GEN_ERROR,
              GEN_RESULT, PIECE_REQUEST, PIECE_DATA, PIECE_ANNOUNCE, HIDDEN_FORWARD, HIDDEN_RESULT)
#: terminal replies a requester must resolve on (the reference only resolves ``gen_result``, SURVEY R8)
GEN_TERMINAL = (GEN_SUCCESS, GEN_ERROR, GEN_RESULT)


def hello(peer_id: str, addr: str, region: str, metrics: Dict[str, float], services: Dict[str, Any],
          api_port: Optional[int] = None, api_host: Optional[str] = None, public_ip: Optional[str] = None,
          pieces: Optional[List[Dict[str, Any]]] = None) -> Dict[str, Any]:
    m = msg(HELLO, peer_id=peer_id, addr=addr, region=region, metrics=metrics, services=services,
            api_port=api_port, api_host=api_host, public_ip=public_ip)
    if pieces:
        m["pieces"] = pieces
    return m


def peer_list(addrs: List[str]) -> Dict[str, Any]:
    return msg(PEER_LIST, peers=list(addrs))


def ping(metrics: Optional[Dict[str, float]] = None) -> Dict[str, Any]:
    m = msg(PING, ts=time.time())
    if metrics is not None:
        m["metrics"] = metrics
    return m


def pong(ts: float) -> Dict[str, Any]:
    return msg(PONG, ts=ts)


def service_announce(service: str, meta: Dict[str, Any]) -> Dict[str, Any]:
    return msg(SERVICE_ANNOUNCE, service=service, meta=meta)


def gen_request(rid: str, prompt: str, model: Optional[str] = None, svc: str = "hf", max_new_tokens: int = 2048,
                temperature: float = 0.7, stream: bool = False, top_k: Optional[int] = None,
                min_p: Optional[float] = None, presence_penalty: Optional[float] = None,
                frequency_penalty: Optional[float] = None,
                logit_bias: Optional[Dict[int, float]] = None) -> Dict[str, Any]:
    # both spellings are sent: the reference reads ``max_tokens`` but its requester writes
    # ``max_new_tokens`` (p2p_runtime.py:577 vs 822)
    m = msg(GEN_REQUEST, rid=rid, prompt=prompt, model=model, svc=svc, max_new_tokens=max_new_tokens,
            max_tokens=max_new_tokens, temperature=temperature, stream=stream)
    # optional sampling filters travel only when set, so a request without them is the reference's message
    if top_k is not None:
        m["top_k"] = int(top_k)
    if min_p is not None:
        m["min_p"] = float(min_p)
    if presence_penalty is not None:
        m["presence_penalty"] = float(presence_penalty)
    if frequency_penalty is not None:
        m["frequency_penalty"] = float(frequency_penalty)
    if logit_bias:
        m["logit_bias"] = {str(int(k)): float(v) for k, v in logit_bias.items()}     # JSON keys: decimal strings
    return m


def request_id_of(m: Dict[str, Any]) -> Optional[str]:
    return m.get("rid") or m.get("task_id")


# ---- legacy coordinator protocol (worker side kept in node.py) -----------------
REGISTER = "register"
HEARTBEAT = "heartbeat"
TASK = "task"
RESULT = "result"
ERROR = "error"
INFO = "info"
NODE_LIST = "node_list"
LIST_NODES = "list_nodes"
RUN_PIPELINE = "run_pipeline"
RUN_TRAIN_STEP = "run_train_step"
CREATE_JOB = "create_job"
RUN_JOB_STEPS = "run_job_steps"
GET_JOB = "get_job"
STOP_JOB = "stop_job"
FORWARD_TASK = "forward_task"
RUN_HF_PIPELINE = "run_hf_pipeline"

TASK_LAYER_FORWARD = "layer_forward"
TASK_LAYER_FORWARD_TRAIN = "layer_forward_train"
TASK_LAYER_BACKWARD = "layer_backward"
HF_LOAD = "hf_load"
HF_UNLOAD = "hf_unload"
HF_INFER = "hf_infer"
ONNX_LOAD = "onnx_load"
ONNX_UNLOAD = "onnx_unload"
ONNX_INFER = "onnx_infer"
HF_PART_LOAD = "hf_part_load"
HF_PART_FORWARD = "hf_part_forward"

TASK_KINDS = (TASK_LAYER_FORWARD, TASK_LAYER_FORWARD_TRAIN, TASK_LAYER_BACKWARD, HF_LOAD, HF_UNLOAD, HF_INFER,
              ONNX_LOAD, ONNX_UNLOAD, ONNX_INFER, HF_PART_LOAD, HF_PART_FORWARD)
