"""Layer-piece pipeline over the *control-plane* mesh, for hosts without NVLink (CPU plumbing
configuration of BASELINE.json: distilgpt2 split in two pieces over the loopback
``p2p_runtime``).  This is the generalisation of the reference's orphaned
``hf_part_load`` / ``hf_part_forward`` worker tasks (/root/reference/bee2bee/node.py:236-277)
to decoder LMs with a KV cache:

* ``PieceHost``           one layer range + per-session KV caches on a peer,
* ``encode/decode_tensor`` binary payloads (base64 of raw bytes + shape + dtype) instead of
                           JSON nested lists of floats (10+ bytes per fp32 in the reference),
* ``MeshPipelineService``  an ``hf``-shaped service on the head peer that drives generation
                           through the chain piece0 (local) -> piece1 (remote) -> ... and samples.

On a H100 box this path is not used: pieces hand activations GPU->GPU (``parallel.mesh``).
"""
from __future__ import annotations

import asyncio
import base64
import json
import threading
import time
from typing import Any, Dict, Iterator, List, Mapping, Optional

import torch

from ..engine.core import SamplerControls
from ..engine.tokenizer import STOP_WORDS, cut_at_stop_words, load_tokenizer, parse_transcript
from ..models.config import ModelConfig, resolve_config, split_layers
from ..models.torch_ref import SequenceSampler, TorchPiece
from ..models.weights import load_or_init
from ..services import BaseService, ServiceError, sampling_filters
from ..utils import new_id

_DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16, "int64": torch.int64}


def encode_tensor(t: torch.Tensor) -> Dict[str, Any]:
    t = t.detach().cpu().contiguous()
    name = str(t.dtype).replace("torch.", "")
    raw = t.view(torch.uint8).numpy().tobytes() if t.dtype == torch.bfloat16 else t.numpy().tobytes()
    return {"shape": list(t.shape), "dtype": name, "b64": base64.b64encode(raw).decode("ascii")}


def decode_tensor(p: Dict[str, Any]) -> torch.Tensor:
    raw = base64.b64decode(p["b64"])
    dt = _DT[p["dtype"]]
    if dt == torch.bfloat16:
        return torch.frombuffer(bytearray(raw), dtype=torch.uint8).view(torch.bfloat16).reshape(p["shape"]).clone()
    return torch.frombuffer(bytearray(raw), dtype=dt).reshape(p["shape"]).clone()


def piece_key(model: str, index: int) -> str:
    return f"{model}:{index}"


class PieceHost:
    """One resident layer range; sessions (= requests) keep their own KV cache on this peer."""

    def __init__(self, model: str, index: int, n_pieces: int, device: str = "cpu", seed: int = 0,
                 cfg: Optional[ModelConfig] = None):
        self.cfg = cfg or resolve_config(model)
        ranges = split_layers(self.cfg.n_layers, n_pieces)
        self.index, self.n_pieces = index, len(ranges)
        self.first, self.last = index == 0, index == len(ranges) - 1
        tensors = load_or_init(model, self.cfg, ranges[index], self.first, self.last, device=device,
                               dtype=torch.float32, seed=seed)
        self.piece = TorchPiece(self.cfg, ranges[index], self.first, self.last, tensors)
        self.device = device
        self.sessions: Dict[str, dict] = {}
        self._lock = threading.Lock()

    def forward(self, session: str, x: torch.Tensor, positions: List[int], reset: bool = False,
                release: bool = False) -> Optional[torch.Tensor]:
        with self._lock:
            if release:
                self.sessions.pop(session, None)
                return None
            if reset or session not in self.sessions:
                self.sessions[session] = self.piece.new_cache()
            cache = self.sessions[session]
        pos = torch.tensor([positions], device=self.device)
        with torch.no_grad():
            return self.piece.forward(x.to(self.device), pos, cache, logits_last_only=True)


class MeshPipelineService(BaseService):
    """``hf``-named service whose model is split across mesh peers.

    ``chain`` lists, for pieces 1..N-1, the peer id hosting it (piece 0 is local).  Runs on the
    node's event loop; torch compute goes through the default executor."""

    def __init__(self, node, model: str, n_pieces: int, chain: List[str], price_per_token: float = 0.0,
                 max_new_tokens: int = 2048, seed: int = 0):
        super().__init__("hf")
        self.node, self.model_name, self.n_pieces, self.chain = node, model, n_pieces, chain
        self.price_per_token, self.max_new_tokens = price_per_token, max_new_tokens
        self.cfg = resolve_config(model)
        self.head = PieceHost(model, 0, n_pieces, seed=seed, cfg=self.cfg)
        self.tokenizer = load_tokenizer(model, self.cfg.vocab_size, self.cfg.eos_token_id, self.cfg.bos_token_id)
        self.loop: Optional[asyncio.AbstractEventLoop] = None
        self.hop_bytes = 0
        self.hops = 0

    def bind_loop(self, loop: asyncio.AbstractEventLoop) -> None:
        self.loop = loop

    def get_metadata(self) -> Dict[str, Any]:
        return {"models": [self.model_name], "price_per_token": self.price_per_token,
                "max_new_tokens": self.max_new_tokens, "backend": "mesh-pipeline", "pieces": self.n_pieces}

    async def _through_chain(self, session: str, x: torch.Tensor, positions: List[int], reset: bool) -> torch.Tensor:
        loop = asyncio.get_running_loop()
        y = await loop.run_in_executor(None, self.head.forward, session, x, positions, reset, False)
        for i, pid in enumerate(self.chain, start=1):
            payload = encode_tensor(y)
            self.hop_bytes += len(payload["b64"]) * 3 // 4
            self.hops += 1
            res = await self.node.forward_hidden(pid, piece_key(self.model_name, i), session, payload, positions,
                                                 reset=reset)
            y = decode_tensor(res["tensor"])
        return y                                              # logits [1, 1, V] from the last piece

    async def _release(self, session: str) -> None:
        self.head.forward(session, torch.zeros(1), [], release=True)
        for i, pid in enumerate(self.chain, start=1):
            try:
                await self.node.forward_hidden(pid, piece_key(self.model_name, i), session,
                                               encode_tensor(torch.zeros(1)), [], release=True, timeout=10)
            except Exception:
                pass

    async def agenerate(self, prompt_ids: List[int], max_new: int, temperature: float, top_p: float = 1.0,
                        rep: float = 1.0, on_token=None, seed: int = 0, top_k: int = 0,
                        min_p: float = 0.0, presence_penalty: float = 0.0,
                        frequency_penalty: float = 0.0, logit_bias: Optional[Mapping[int, float]] = None) -> List[int]:
        session = new_id("sess")
        controls = SamplerControls(temperature=temperature, top_p=top_p, repetition_penalty=rep, top_k=top_k,
                                   min_p=min_p, presence_penalty=presence_penalty, frequency_penalty=frequency_penalty,
                                   logit_bias=dict(logit_bias or {}))
        if controls.logit_bias:      # the ids must lie in the vocabulary (the other controls are taken as given)
            SamplerControls(logit_bias=controls.logit_bias).validate(self.cfg.vocab_size)
        sampler = SequenceSampler(controls, self.cfg.vocab_size, prompt_ids, torch.Generator().manual_seed(seed))
        out: List[int] = []
        try:
            x = torch.tensor([prompt_ids])
            pos = list(range(len(prompt_ids)))
            logits = await self._through_chain(session, x, pos, reset=True)
            for step in range(max_new):
                tok = sampler.draw(logits[0, -1])
                out.append(tok)
                if on_token is not None:
                    on_token(tok)
                if tok in self.cfg.eos_ids or step == max_new - 1:
                    break
                p = len(prompt_ids) + step
                logits = await self._through_chain(session, torch.tensor([[tok]]), [p], reset=False)
        finally:
            await self._release(session)
        return out

    # ---- BaseService ---------------------------------------------------------------------
    def _params(self, params: Dict[str, Any]):
        prompt = params.get("prompt")
        if not prompt:
            raise ServiceError("Missing prompt")
        t = params.get("temperature", 0.7)
        return prompt, int(params.get("max_new_tokens") or self.max_new_tokens), float(0.7 if t is None else t)

    async def aexecute(self, params: Dict[str, Any]) -> Dict[str, Any]:
        prompt, max_new, temperature = self._params(params)
        t0 = time.time()
        ids = self.tokenizer.encode(prompt)
        out = await self.agenerate(ids, max_new, temperature, **sampling_filters(params))
        text = prompt + self.tokenizer.decode(out)
        return {"text": text, "tokens": len(out), "latency_ms": int((time.time() - t0) * 1000),
                "price_per_token": self.price_per_token, "cost": self.price_per_token * len(out)}

    async def aexecute_stream(self, params: Dict[str, Any]):
        try:
            prompt, max_new, temperature = self._params(params)
            rendered = self.tokenizer.apply_chat_template(parse_transcript(prompt), add_generation_prompt=True)
            ids = self.tokenizer.encode(rendered)
            q: asyncio.Queue = asyncio.Queue()
            task = asyncio.create_task(self.agenerate(ids, max_new, temperature, 0.95, 1.15, on_token=q.put_nowait,
                                                      **sampling_filters(params)))
            toks: List[int] = []
            sent = ""
            while not (task.done() and q.empty()):
                try:
                    toks.append(await asyncio.wait_for(q.get(), 0.05))
                except asyncio.TimeoutError:
                    continue
                text, hit = cut_at_stop_words(self.tokenizer.decode(toks), STOP_WORDS)
                if len(text) > len(sent) and not text.endswith("�"):
                    yield json.dumps({"text": text[len(sent):]}) + "\n"
                    sent = text
                if hit:
                    task.cancel()
                    break
            if task.done() and not task.cancelled() and task.exception():
                raise task.exception()
            yield json.dumps({"done": True}) + "\n"
        except Exception as exc:
            yield json.dumps({"status": "error", "message": str(exc)}) + "\n"

    def _run(self, coro):
        if self.loop is None or not self.loop.is_running():
            raise ServiceError("MeshPipelineService needs its node's running event loop (bind_loop)")
        try:
            running = asyncio.get_running_loop()
        except RuntimeError:
            running = None
        if running is self.loop:
            raise ServiceError("call aexecute()/aexecute_stream() from the event loop")
        return asyncio.run_coroutine_threadsafe(coro, self.loop).result(600)

    def execute(self, params: Dict[str, Any]) -> Dict[str, Any]:
        return self._run(self.aexecute(params))

    def execute_stream(self, params: Dict[str, Any]) -> Iterator[str]:
        async def collect():
            return [c async for c in self.aexecute_stream(params)]

        yield from self._run(collect())
