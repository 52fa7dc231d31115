"""Service abstraction: what a peer *offers* to the mesh (parity:
/root/reference/bee2bee/services.py:10-308).

    BaseService(name).get_metadata() / execute(params) -> dict / execute_stream(params) -> iterator

Result / metadata keys and stream formats are the reference's (NDJSON ``{"text":..}``
lines + ``{"done": true}`` for HF, raw text chunks for Ollama).  What differs is what is
behind them: ``HFService`` enqueues into this framework's continuous-batching engine
(hand-written sm_90a kernels, pieces across GPUs) instead of calling
``transformers.generate`` inline, and every service exposes ``aexecute`` /
``aexecute_stream`` so asyncio callers never block their loop (SURVEY section 8).
"""
from __future__ import annotations

import asyncio
import json
import os
import threading
import time
from typing import Any, AsyncIterator, Dict, Iterator, List, Optional

from .utils import offline

try:
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("bee2bee")


class ServiceError(Exception):
    pass


class BaseService:
    def __init__(self, name: str):
        self.name = name

    def get_metadata(self) -> Dict[str, Any]:
        raise NotImplementedError

    def load_sync(self) -> None:  # optional for subclasses
        return None

    def execute(self, params: Dict[str, Any]) -> Dict[str, Any]:
        raise NotImplementedError

    def execute_stream(self, params: Dict[str, Any]) -> Iterator[str]:
        raise NotImplementedError

    # ---- asyncio adapters: the blocking work runs on a worker thread ------------------------
    async def aexecute(self, params: Dict[str, Any]) -> Dict[str, Any]:
        return await asyncio.get_running_loop().run_in_executor(None, self.execute, params)

    async def aexecute_stream(self, params: Dict[str, Any]) -> AsyncIterator[str]:
        loop = asyncio.get_running_loop()
        q: asyncio.Queue = asyncio.Queue()
        DONE = object()

        def pump():
            try:
                for chunk in self.execute_stream(params):
                    loop.call_soon_threadsafe(q.put_nowait, chunk)
            except Exception as exc:  # surfaced to the consumer as a final error line
                loop.call_soon_threadsafe(q.put_nowait, json.dumps({"status": "error", "message": str(exc)}) + "\n")
            finally:
                loop.call_soon_threadsafe(q.put_nowait, DONE)

        threading.Thread(target=pump, daemon=True).start()
        while True:
            item = await q.get()
            if item is DONE:
                return
            yield item

    def serves(self, model: Optional[str]) -> bool:
        """Exact match or substring either way (the reference's /chat rule, api.py:205-212)."""
        if not model:
            return True
        for m in self.get_metadata().get("models", []):
            if model == m or model in m or m in model:
                return True
        return False


# =============================================================================== HF (native engine)
class HFService(BaseService):
    def __init__(self, model_name: str, price_per_token: float = 0.0, max_new_tokens: int = 2048, pieces: int = 1,
                 device: Optional[str] = None, **engine_kw):
        super().__init__("hf")
        self.model_name, self.price_per_token, self.max_new_tokens = model_name, price_per_token, max_new_tokens
        self.pieces, self.device_pref, self.engine_kw = pieces, device, engine_kw
        self.model = None
        self.tokenizer = None
        self.device = None

    def load_sync(self) -> None:
        try:
            from .hf import load_model_and_tokenizer

            self.model, self.tokenizer, self.device = load_model_and_tokenizer(
                self.model_name, self.device_pref, pieces=self.pieces, **self.engine_kw)
            from .utils import set_throughput_source

            eng = self.model.engine
            set_throughput_source(lambda: eng.metrics()["tokens_per_s"])
            logger.info(f"model '{self.model_name}' resident on {self.device} ({self.pieces} piece(s))")
        except KeyError as exc:
            raise ServiceError(f"Failed to load model: {exc}")
        except Exception as exc:
            raise ServiceError(f"Failed to load model: {exc}")

    def get_metadata(self) -> Dict[str, Any]:
        from .models.weights import WEIGHT_SOURCE

        return {"models": [self.model_name], "price_per_token": self.price_per_token,
                "max_new_tokens": self.max_new_tokens, "backend": "b200-native", "pieces": self.pieces,
                "weights": WEIGHT_SOURCE.get(self.model_name, "unloaded"), "healthy": self.healthy()}

    def healthy(self) -> bool:
        """False once the engine's GPU mesh aborted (a peer piece stalled or died): the provider must stop attracting
        requests -- the reference's semantics for a lost peer (p2p_runtime.py:396-410: dropped, next pick skips it)."""
        eng = getattr(self.model, "engine", None)
        return not (eng is not None and getattr(eng, "broken", None))

    def _args(self, params: Dict[str, Any]):
        prompt = params.get("prompt")
        if not prompt:
            raise ServiceError("Missing prompt")
        if self.model is None:
            raise ServiceError("Model not loaded")
        max_new = int(params.get("max_new_tokens") or params.get("max_tokens") or self.max_new_tokens)
        t = params.get("temperature", 0.7)
        return prompt, max_new, float(0.7 if t is None else t)

    def execute(self, params: Dict[str, Any]) -> Dict[str, Any]:
        prompt, max_new, temperature = self._args(params)
        try:
            t0 = time.time()
            from .hf import generate_text

            text, ids = generate_text(self.model, self.tokenizer, self.device, prompt, max_new, temperature=temperature,
                                      return_ids=True)
            n = len(ids)                       # exact count (the reference re-encodes text to estimate it)
            return {"text": text, "tokens": n, "latency_ms": int((time.time() - t0) * 1000.0),
                    "price_per_token": self.price_per_token, "cost": self.price_per_token * n}
        except ServiceError:
            raise
        except Exception as exc:
            raise ServiceError(str(exc))

    def execute_stream(self, params: Dict[str, Any]) -> Iterator[str]:
        try:
            prompt, max_new, temperature = self._args(params)
            from .hf import generate_text_stream

            for delta in generate_text_stream(self.model, self.tokenizer, self.device, prompt, max_new, temperature):
                yield json.dumps({"text": delta}) + "\n"
            yield json.dumps({"done": True}) + "\n"
        except Exception as exc:
            yield json.dumps({"status": "error", "message": str(exc)}) + "\n"


# ========================================================================================== Ollama
class EmbeddedOllama:
    """In-process stand-in for an Ollama daemon with the same JSON shapes (``/api/tags``,
    ``/api/generate``).  There is no ``ollama`` binary on the H100 box (and no network to pull
    models), so ``serve-ollama`` serves the requested model through the native engine while
    keeping the Ollama request/response contract."""

    def __init__(self, model_name: str, pieces: int = 1, device: Optional[str] = None, **engine_kw):
        self.model_name, self.pieces, self.device, self.engine_kw = model_name, pieces, device, engine_kw
        self._lm = None

    def _ensure(self):
        if self._lm is None:
            from .hf import load_model_and_tokenizer

            self._lm, self._tok, self._dev = load_model_and_tokenizer(self.model_name, self.device, pieces=self.pieces,
                                                                      **self.engine_kw)
        return self._lm

    def tags(self) -> Dict[str, Any]:
        tag = self.model_name if ":" in self.model_name else self.model_name + ":latest"
        return {"models": [{"name": tag, "model": tag, "details": {"family": "b200-native"}}]}

    def generate(self, payload: Dict[str, Any]) -> Iterator[Dict[str, Any]]:
        from .engine.core import SamplingParams

        lm = self._ensure()
        opts = payload.get("options") or {}
        sp = SamplingParams(max_new_tokens=int(opts.get("num_predict", 128)),
                            temperature=float(opts.get("temperature", 0.8)), top_p=float(opts.get("top_p", 0.9)),
                            repetition_penalty=float(opts.get("repeat_penalty", 1.1)))
        ids = self._tok.encode(payload.get("prompt", ""))
        t0 = time.time()
        import queue as _q

        q: "_q.Queue[int]" = _q.Queue()
        req = lm.engine.submit(ids, sp, on_token=q.put)
        toks: List[int] = []
        sent = ""
        stream = bool(payload.get("stream", True))
        try:
            while not (req.done.is_set() and q.empty()):
                try:
                    toks.append(q.get(timeout=0.05))
                except _q.Empty:
                    continue
                if stream:
                    text = self._tok.decode(toks)
                    if len(text) > len(sent) and not text.endswith("�"):
                        yield {"model": payload.get("model"), "response": text[len(sent):], "done": False}
                        sent = text
        finally:
            if not req.done.is_set():          # consumer went away mid-stream
                lm.engine.cancel(req, "client_disconnect")
        text = self._tok.decode(toks)
        final = {"model": payload.get("model"), "response": "" if stream else text, "done": True,
                 "eval_count": len(toks), "prompt_eval_count": len(ids), "total_duration": int((time.time() - t0) * 1e9)}
        if stream and len(text) > len(sent):
            yield {"model": payload.get("model"), "response": text[len(sent):], "done": False}
        yield final


class OllamaService(BaseService):
    def __init__(self, model_name: str, host: Optional[str] = None, pieces: int = 1, device: Optional[str] = None,
                 **engine_kw):
        super().__init__("ollama")
        self.model_name = model_name
        # OLLAMA_HOST is honoured (the reference sets it but never reads it, SURVEY section 8)
        self.host = host or os.environ.get("OLLAMA_HOST") or "http://localhost:11434"
        if not self.host.startswith("http") and self.host != "embedded":
            self.host = "http://" + self.host
        self.price_per_token = 0.0
        self.actual_model = model_name
        self.embedded: Optional[EmbeddedOllama] = None
        self._embedded_args = dict(pieces=pieces, device=device, **engine_kw)

    # ---- transport: real daemon over HTTP, or the embedded engine -----------------------------
    def _http_tags(self) -> Optional[Dict[str, Any]]:
        if self.host == "embedded" or offline():
            return None
        try:
            import requests

            res = requests.get(f"{self.host}/api/tags", timeout=5)
            return res.json() if res.status_code == 200 else None
        except Exception:
            return None

    def load_sync(self) -> None:
        tags = self._http_tags()
        if tags is None:
            self.embedded = EmbeddedOllama(self.model_name, **self._embedded_args)
            try:
                self.embedded._ensure()
            except Exception as exc:
                raise ServiceError(f"Ollama connection failed and embedded backend unavailable: {exc}")
            tags = self.embedded.tags()
            logger.info(f"no Ollama daemon at {self.host}: serving '{self.model_name}' from the embedded engine")
        names = [m.get("name", "") for m in tags.get("models", [])]
        for n in names:       # fuzzy tag match: 'llama3' ~ 'llama3:latest'
            if self.model_name == n or self.model_name in n or (n and n in self.model_name):
                self.actual_model = n
                break
        else:
            logger.warning(f"model '{self.model_name}' not listed by Ollama at {self.host}; available: {names}")

    def get_metadata(self) -> Dict[str, Any]:
        return {"models": [self.model_name, self.actual_model], "price_per_token": self.price_per_token,
                "backend": "ollama"}

    def _payload(self, params: Dict[str, Any], stream: bool) -> Dict[str, Any]:
        prompt = params.get("prompt")
        if not prompt:
            raise ServiceError("Missing prompt")
        return {"model": self.actual_model, "prompt": prompt, "stream": stream,
                "options": {"num_predict": int(params.get("max_new_tokens") or params.get("max_tokens") or 2048),
                            "temperature": float(params.get("temperature", 0.7) or 0.7)}}

    def execute(self, params: Dict[str, Any]) -> Dict[str, Any]:
        payload = self._payload(params, stream=False)
        t0 = time.time()
        try:
            if self.embedded is not None:
                data = list(self.embedded.generate(payload))[-1]
            else:
                import requests

                res = requests.post(f"{self.host}/api/generate", json=payload, timeout=300)
                if res.status_code != 200:
                    raise ServiceError(f"Ollama Error: {res.text}")
                data = res.json()
        except ServiceError:
            raise
        except Exception as exc:
            raise ServiceError(f"Ollama Exec Error: {exc}")
        dur = data.get("total_duration", 0)
        return {"text": data.get("response", ""), "tokens": data.get("eval_count", 0),
                "latency_ms": dur / 1e6 if dur else (time.time() - t0) * 1000.0,
                "price_per_token": self.price_per_token, "cost": 0.0}

    def execute_stream(self, params: Dict[str, Any]) -> Iterator[str]:
        """Raw text chunks (not NDJSON) -- the web client's fallback parser relies on this."""
        try:
            payload = self._payload(params, stream=True)
            if self.embedded is not None:
                for part in self.embedded.generate(payload):
                    if part.get("response"):
                        yield part["response"]
                return
            import requests

            res = requests.post(f"{self.host}/api/generate", json=payload, stream=True, timeout=300)
            if res.status_code != 200:
                yield json.dumps({"error": f"Ollama Error: {res.text}"})
                return
            for line in res.iter_lines():
                if not line:
                    continue
                try:
                    data = json.loads(line.decode("utf-8"))
                except ValueError:
                    continue
                if data.get("response"):
                    yield data["response"]
                if data.get("done"):
                    break
        except Exception as exc:
            yield json.dumps({"error": str(exc)})


# ======================================================================================= HF remote
class HFRemoteService(BaseService):
    def __init__(self, model_name: str, token: Optional[str] = None, price_per_token: float = 0.005,
                 client_factory=None):
        super().__init__("hf_remote")
        self.model_name = model_name
        self.token = token or os.getenv("HUGGING_FACE_HUB_TOKEN")
        self.price_per_token = price_per_token
        self.client = None
        self._factory = client_factory

    def load_sync(self) -> None:
        try:
            if self._factory is not None:
                self.client = self._factory(self.model_name, self.token)
            else:
                from huggingface_hub import InferenceClient

                self.client = InferenceClient(model=self.model_name, token=self.token)
        except ImportError:
            raise ServiceError("huggingface_hub not installed. Run 'pip install huggingface-hub'")
        except Exception as exc:
            raise ServiceError(f"Failed to init HF Remote Client: {exc}")

    def get_metadata(self) -> Dict[str, Any]:
        return {"models": [self.model_name], "price_per_token": self.price_per_token, "tag": "remote",
                "backend": "hf_remote"}

    def execute(self, params: Dict[str, Any]) -> Dict[str, Any]:
        if self.client is None:
            raise ServiceError("Remote client not initialized")
        prompt = params.get("prompt")
        if not prompt:
            raise ServiceError("Missing prompt")
        try:
            t0 = time.time()
            text = self.client.text_generation(prompt, max_new_tokens=int(params.get("max_new_tokens", 32)),
                                               temperature=params.get("temperature", 0.7),
                                               do_sample=params.get("do_sample", True))
            tokens = len(text) // 4          # the hosted API does not report usage; same estimate as the reference
            return {"text": text, "tokens": tokens, "latency_ms": int((time.time() - t0) * 1000.0),
                    "price_per_token": self.price_per_token, "cost": self.price_per_token * tokens,
                    "backend": "hf_remote"}
        except Exception as exc:
            raise ServiceError(f"HF Remote Execution Error: {exc}")

    def execute_stream(self, params: Dict[str, Any]) -> Iterator[str]:
        """NDJSON like HFService (the reference leaves this unimplemented for hf_remote)."""
        try:
            if self.client is None:
                raise ServiceError("Remote client not initialized")
            try:
                it = self.client.text_generation(params.get("prompt"), max_new_tokens=int(params.get("max_new_tokens", 32)),
                                                 temperature=params.get("temperature", 0.7), stream=True)
                for piece in it:
                    yield json.dumps({"text": str(piece)}) + "\n"
            except TypeError:
                yield json.dumps({"text": self.execute(params)["text"]}) + "\n"
            yield json.dumps({"done": True}) + "\n"
        except Exception as exc:
            yield json.dumps({"status": "error", "message": str(exc)}) + "\n"


def build_service(backend: str, model: str, **kw) -> BaseService:
    """Factory used by the launcher (backend in {"hf", "ollama", "hf_remote"})."""
    if backend == "hf":
        return HFService(model, price_per_token=kw.pop("price_per_token", 0.0), **kw)
    if backend == "ollama":
        return OllamaService(model, **kw)
    if backend == "hf_remote":
        return HFRemoteService(model, token=kw.get("token"))
    raise ServiceError(f"unknown backend '{backend}'")
