"""Layer range [start, end) of a decoder LM resident on ONE H100 for the legacy coordinator / worker protocol
(``hf_part_load`` / ``hf_part_forward``, /root/reference/bee2bee/node.py:236-277), executed by the hand-written
kernels (``NativePiece``) with a paged KV cache per session.

The reference ships the hidden state of every hop as a JSON list of fp32 (D2H -> ``.tolist()`` -> WebSocket ->
``np.array`` -> H2D, node.py:270-277).  Here the payload stays in device memory:

  * ``forward(..., keep_on_device=True)`` leaves the piece output in a ``cudaMalloc`` buffer and returns a *reference*
    ``{"ref": id, "device": k, "shape": [T, H], "ipc": <64-byte CUDA IPC handle, hex>}``;
  * the next stage accepts that reference: same process -> ``cudaMemcpyPeerAsync`` GPU k -> its own GPU (NVLink), other
    process -> ``cudaIpcOpenMemHandle`` + the same peer copy.  The control frame (the JSON task) carries ~100 bytes.

Legacy payloads (JSON lists, base64 frames, text / ids) are still accepted and produced on request.
"""
from __future__ import annotations

import threading
from typing import Dict, List, Optional

import torch

from .. import ops
from ..engine.kv import PAGE
from ..models.config import resolve_config
from ..models.native import BatchMeta, NativePiece
from ..models.weights import load_or_init

_LOCK = threading.Lock()
_BUFFERS: Dict[str, dict] = {}       # process-wide registry of device-resident hop payloads: ref id -> entry
_COUNTER = [0]


def register_buffer(ptr: int, device: int, shape: List[int]) -> dict:
    with _LOCK:
        _COUNTER[0] += 1
        ref = f"hop-{_COUNTER[0]}"
        ent = {"ref": ref, "device": device, "shape": list(shape), "ptr": ptr}
        _BUFFERS[ref] = ent
    return ent


def release_buffer(ref: str) -> None:
    with _LOCK:
        ent = _BUFFERS.pop(ref, None)
    if ent is not None:
        try:
            ops.native().peer_free(ent["ptr"])
        except Exception:
            pass


class GpuPieceHost:
    def __init__(self, model: str, start: int, end: int, device: str = "cuda:0", max_tokens: int = 512,
                 max_sessions: int = 4, max_seq_len: int = 1024, seed: int = 0):
        self.cfg = cfg = resolve_config(model)
        self.device = torch.device(device)
        end = min(end, cfg.n_layers)
        self.first, self.last = start == 0, end >= cfg.n_layers
        self.layers = list(range(start, end))
        self.max_tokens, self.max_seq_len = max_tokens, max_seq_len
        self.pages_per_session = (max_seq_len + PAGE - 1) // PAGE
        torch.cuda.set_device(self.device)
        self.C = ops.native()
        self.C.init_kernels(self.device.index)
        tensors = load_or_init(model, cfg, self.layers, self.first, self.last, device=self.device, dtype=torch.bfloat16,
                               seed=seed)
        self.piece = NativePiece(cfg, self.layers, self.first, self.last, tensors, self.device, max_tokens, 1,
                                 1 + max_sessions * self.pages_per_session)
        del tensors
        self.sessions: Dict[str, dict] = {}
        self.max_sessions = max_sessions
        self.x_in = torch.zeros((max_tokens, cfg.hidden_size), device=self.device, dtype=torch.bfloat16)
        self.stream = torch.cuda.Stream(device=self.device)
        self.launches = 0

    # ------------------------------------------------------------------ sessions (KV residency)
    def _session(self, name: Optional[str]) -> dict:
        key = name or "__anon__"
        s = self.sessions.get(key)
        if s is None:
            if len(self.sessions) >= self.max_sessions:
                self.sessions.pop(next(iter(self.sessions)))          # oldest session gives up its pages
            used = {s2["base"] for s2 in self.sessions.values()}
            base = next(b for b in range(self.max_sessions) if b not in used)
            pages = [1 + base * self.pages_per_session + i for i in range(self.pages_per_session)]
            s = {"base": base, "pages": pages, "len": 0}
            self.sessions[key] = s
        return s

    def drop_session(self, name: Optional[str]) -> None:
        self.sessions.pop(name or "__anon__", None)

    # ------------------------------------------------------------------ inputs
    def load_hidden_ref(self, ref: dict) -> torch.Tensor:
        """hop payload by reference -> this piece's input buffer (device-to-device, never through the host)"""
        T, H = ref["shape"]
        assert H == self.cfg.hidden_size and T <= self.max_tokens
        ent = _BUFFERS.get(ref.get("ref", ""))
        opened = 0
        if ent is not None:
            src, src_dev = ent["ptr"], ent["device"]
        else:
            src = opened = self.C.ipc_import(bytes.fromhex(ref["ipc"]))       # produced by another process
            src_dev = int(ref["device"])
        with torch.cuda.stream(self.stream):
            self.C.memcpy_peer(self.x_in.data_ptr(), self.device.index, src, src_dev, T * H * 2)
        if opened:
            self.stream.synchronize()
            self.C.ipc_close(opened)
        return self.x_in[:T]

    def load_hidden_host(self, t: torch.Tensor) -> torch.Tensor:
        T = t.shape[-2]
        with torch.cuda.stream(self.stream):
            self.x_in[:T].copy_(t.reshape(T, -1).to(torch.bfloat16), non_blocking=False)
        return self.x_in[:T]

    # ------------------------------------------------------------------ forward
    def forward(self, session: Optional[str], ids: Optional[List[int]] = None, hidden: Optional[torch.Tensor] = None,
                pos0: Optional[int] = None, keep_on_device: bool = False):
        """One hop: ``ids`` (first piece) or ``hidden`` [T, H] (device tensor inside this host) in; hidden states
        [T, H] (or fp32 logits [1, V] on the last piece) out -- as a device reference when ``keep_on_device``."""
        c = self.cfg
        s = self._session(session)
        T = len(ids) if ids is not None else hidden.shape[0]
        if pos0 is None:
            pos0 = s["len"]
        assert T <= self.max_tokens and pos0 + T <= self.max_seq_len, "hop exceeds the piece's token / context budget"
        dev, i32 = self.device, torch.int32
        with torch.cuda.stream(self.stream):
            pos = torch.arange(pos0, pos0 + T, device=dev, dtype=i32)
            pages = torch.tensor(s["pages"], device=dev, dtype=i32)
            slots = (pages[(pos // PAGE).long()] * PAGE + pos % PAGE).to(i32)
            meta = BatchMeta(ids=torch.tensor(ids if ids is not None else [0] * T, device=dev, dtype=i32), positions=pos,
                             slots=slots, q_start=torch.zeros(1, device=dev, dtype=i32),
                             q_len=torch.tensor([T], device=dev, dtype=i32),
                             kv_len=torch.tensor([pos0 + T], device=dev, dtype=i32), block_table=pages[None, :].contiguous(),
                             n_tokens=T, n_seqs=1, max_q=T, last_idx=torch.tensor([T - 1], device=dev, dtype=torch.int64))
            out = self.piece.forward(meta, x_in=hidden)
            s["len"] = pos0 + T
            self.launches += 5 * len(self.layers) + 2
            if self.last:
                logits = out[:1, :c.vocab_size].float()
                self.stream.synchronize()
                return {"logits": logits}
            if keep_on_device:
                ptr = self.C.peer_alloc(T * c.hidden_size * 2)
                self.C.memcpy_peer(ptr, dev.index, out.data_ptr(), dev.index, T * c.hidden_size * 2)
                self.stream.synchronize()
                ent = register_buffer(ptr, dev.index, [T, c.hidden_size])
                return {"hidden_ref": {"ref": ent["ref"], "device": dev.index, "shape": [T, c.hidden_size],
                                       "ipc": bytes(self.C.ipc_export(ptr)).hex()}}
            res = out[:T].clone()
        self.stream.synchronize()
        return {"hidden": res}
