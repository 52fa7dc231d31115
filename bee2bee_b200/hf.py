"""Model-backend helpers with the reference's L2 surface
(/root/reference/bee2bee/hf.py:7-205) on top of this framework's engine instead of
``transformers.generate``:

    load_model_and_tokenizer -> (LoadedModel, tokenizer, device)
    generate_text / generate_text_stream      (same defaults: rep. penalty 1.15, top_p 0.95,
                                               greedy when temperature <= 0, stop-word cut;
                                               optional top_k / min_p, off by default: transformers'
                                               implicit top_k=50 is not applied; optional presence /
                                               frequency penalties and logit_bias, off by default)
    export_torchscript / export_onnx          (over the plain-torch module of the model)
    load_dataset / preprocess_examples
    build_layer_partial (== build_distilbert_partial generalised to decoder LMs: only the
                         requested layer range is materialised on the device)
"""
from __future__ import annotations

import queue
import threading
from typing import Any, Dict, Iterator, Optional, Tuple

from .engine.core import Engine, SamplingParams
from .engine.tokenizer import STOP_WORDS, cut_at_stop_words, load_tokenizer, parse_transcript
from .models.config import ModelConfig, resolve_config


def has_transformers() -> bool:
    try:
        import transformers  # noqa: F401
        return True
    except Exception:
        return False


def has_datasets() -> bool:
    try:
        import datasets  # noqa: F401
        return True
    except Exception:
        return False


class LoadedModel:
    """What ``load_model_and_tokenizer`` hands back in place of an HF ``PreTrainedModel``."""

    def __init__(self, name: str, engine: Engine, tokenizer):
        self.name, self.engine, self.tokenizer = name, engine, tokenizer
        self.config: ModelConfig = engine.cfg

    def eval(self):
        return self

    def to(self, *_a, **_k):
        return self

    def close(self):
        self.engine.close()


_MODELS: Dict[Tuple[str, str, int, bool], LoadedModel] = {}
_LOCK = threading.Lock()


def load_model_and_tokenizer(model_name: str, device: Optional[str] = None, pieces: int = 1, **engine_kw):
    """Resolve ``model_name`` (preset, alias or local HF directory), build the engine on
    ``device`` (``cuda`` when available) and start its scheduler thread.  Cached per
    (name, device, pieces) so several services share one resident copy of the weights."""
    import torch

    if device is None:
        device = "cuda" if torch.cuda.is_available() else "cpu"
    import os

    supervised = os.environ.get("B2B_SUPERVISED", "0") == "1"
    key = (model_name, str(device), int(pieces), supervised)
    with _LOCK:
        lm = _MODELS.get(key)
        if lm is None:
            cfg = resolve_config(model_name)
            if supervised:
                # the engine (one worker process per GPU piece, or one CPU worker) runs as a restartable child group;
                # this process never owns a CUDA context, so a dead rank cannot take the serving front down
                from .parallel.supervisor import SupervisedEngine

                gpu_mesh = pieces > 1 and str(device).startswith("cuda")
                kw = dict(engine_kw) if gpu_mesh else dict(engine_kw, pieces=pieces)
                eng = SupervisedEngine(model_name, device=str(device), world=pieces if gpu_mesh else 1, engine_kw=kw)
            elif pieces > 1 and str(device).startswith("cuda"):
                # one process per GPU: this process becomes rank 0, followers are spawned
                from .parallel.launch import build_engine, spawn_followers

                lm_procs = spawn_followers(model_name, pieces, dict(engine_kw))
                eng = build_engine(model_name, 0, pieces, **engine_kw)
                eng._followers = lm_procs
            else:
                eng = Engine(model_name, cfg=cfg, device=str(device), pieces=pieces, **engine_kw)
            eng.start()
            tok = load_tokenizer(model_name, cfg.vocab_size, cfg.eos_token_id, cfg.bos_token_id)
            lm = LoadedModel(model_name, eng, tok)
            _MODELS[key] = lm
        lm.engine.start()             # no-op when the scheduler thread is alive; revives a stopped engine
    return lm, lm.tokenizer, str(device)


def unload_model(model_name: str) -> int:
    with _LOCK:
        keys = [k for k in _MODELS if k[0] == model_name]
        for k in keys:
            _MODELS.pop(k).close()
    return len(keys)


def generate_text(model: LoadedModel, tokenizer, device: str, prompt: str, max_new_tokens: int = 32,
                  temperature: float = 0.7, return_full_text: bool = True, return_ids: bool = False, top_k: int = 0,
                  min_p: float = 0.0, presence_penalty: float = 0.0, frequency_penalty: float = 0.0,
                  logit_bias: Optional[Dict[int, float]] = None):
    """Non-streaming path: temperature + do_sample only (no top-p / repetition penalty), returns
    prompt + completion like the reference (hf.py:35-44).  ``top_k`` / ``min_p``, the presence / frequency
    penalties and ``logit_bias`` (token id -> bias) are off unless given."""
    ids = tokenizer.encode(prompt)
    sp = SamplingParams(max_new_tokens=max_new_tokens, temperature=temperature, top_p=1.0, repetition_penalty=1.0,
                        top_k=top_k, min_p=min_p, presence_penalty=presence_penalty,
                        frequency_penalty=frequency_penalty, logit_bias=dict(logit_bias or {}))
    req = model.engine.submit(ids, sp)
    try:
        req.wait(timeout=600)
    except TimeoutError:
        model.engine.cancel(req, "timeout")      # do not leave a zombie decoding to max_new_tokens
        raise
    text = tokenizer.decode(req.out_ids)
    full = (prompt + text) if return_full_text else text
    return (full, req.out_ids) if return_ids else full


def generate_text_stream(model: LoadedModel, tokenizer, device: str, prompt: str, max_new_tokens: int = 512,
                         temperature: float = 0.7, top_k: int = 0, min_p: float = 0.0, presence_penalty: float = 0.0,
                         frequency_penalty: float = 0.0,
                         logit_bias: Optional[Dict[int, float]] = None) -> Iterator[str]:
    """Streaming path (hf.py:46-136): transcript -> chat template, rep. penalty 1.15, top_p 0.95
    (greedy when temperature <= 0), yields text deltas, stops at the first stop word.  ``top_k`` / ``min_p``, the
    presence / frequency penalties and ``logit_bias`` are off unless given."""
    messages = parse_transcript(prompt)
    try:
        rendered = tokenizer.apply_chat_template(messages, add_generation_prompt=True)
    except Exception:
        rendered = prompt
    ids = tokenizer.encode(rendered)
    q: "queue.Queue[Optional[int]]" = queue.Queue()
    sp = SamplingParams(max_new_tokens=max_new_tokens, temperature=temperature, top_p=0.95, repetition_penalty=1.15,
                        top_k=top_k, min_p=min_p, presence_penalty=presence_penalty,
                        frequency_penalty=frequency_penalty, logit_bias=dict(logit_bias or {}))
    req = model.engine.submit(ids, sp, on_token=q.put)
    emitted, toks = "", []
    try:
        while True:
            try:
                tok = q.get(timeout=0.05)
            except queue.Empty:
                if req.done.is_set() and q.empty():
                    break
                continue
            toks.append(tok)
            text = tokenizer.decode(toks)
            if text.endswith("�"):
                continue                      # incomplete multi-byte sequence: wait for more ids
            visible, hit = cut_at_stop_words(text, STOP_WORDS)
            if len(visible) > len(emitted):
                yield visible[len(emitted):]
                emitted = visible
            if hit:
                break
    finally:
        # stop word hit, or the consumer closed the generator (client disconnect): free the batch slot and the
        # KV pages at the next burst boundary instead of decoding up to max_new_tokens (2048 from /chat)
        if not req.done.is_set():
            model.engine.cancel(req, "stop")
    if req.error:
        raise RuntimeError(req.error)


# ------------------------------------------------------------------- exporters
def as_torch_module(model_name: str, device: str = "cpu"):
    """The whole model as a plain ``torch.nn.Module`` (ids, positions -> logits), for export."""
    import torch

    from .models.torch_ref import TorchPiece
    from .models.weights import load_or_init

    cfg = resolve_config(model_name)
    tensors = load_or_init(model_name, cfg, range(cfg.n_layers), True, True, device=device, dtype=torch.float32)

    class Module(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.params = torch.nn.ParameterDict(
                {k.replace(".", "__"): torch.nn.Parameter(v, requires_grad=False) for k, v in tensors.items()})
            self.piece = TorchPiece(cfg, range(cfg.n_layers), True, True,
                                    {k: self.params[k.replace(".", "__")] for k in tensors})

        def forward(self, input_ids, attention_mask=None):
            pos = torch.arange(input_ids.shape[1], device=input_ids.device)[None].expand_as(input_ids)
            return self.piece.forward(input_ids, pos, None)

    return Module().eval()


def export_torchscript(model, example_inputs) -> Any:
    import torch

    model = model.eval()
    with torch.no_grad():
        return torch.jit.trace(model, example_inputs, check_trace=False)


def export_onnx(model, example_inputs, output_path: str) -> str:
    import torch

    torch.onnx.export(model, example_inputs, output_path, input_names=["input_ids", "attention_mask"],
                      output_names=["logits"], opset_version=14,
                      dynamic_axes={"input_ids": {0: "batch", 1: "seq"}, "attention_mask": {0: "batch", 1: "seq"},
                                    "logits": {0: "batch", 1: "seq"}})
    return output_path


# --------------------------------------------------------------------- datasets
def load_dataset(name: str, split: str = "train", streaming: bool = False, **kwargs):
    """``datasets.load_dataset``; ``synthetic:<n>`` yields n deterministic text rows offline."""
    if name.startswith("synthetic"):
        n = int(name.split(":")[1]) if ":" in name else 64
        rows = {"text": [f"sample {i}: the quick brown fox jumps over the lazy dog {i * 7919 % 101}" for i in range(n)]}
        if has_datasets():
            from datasets import Dataset
            return Dataset.from_dict(rows)
        return rows
    from datasets import load_dataset as _ld

    return _ld(name, split=split, streaming=streaming, **kwargs)


def preprocess_examples(dataset, tokenizer_name: str, text_field: str = "text", max_length: int = 128,
                        lower_case: bool = False):
    """Tokenise to fixed length (padding + truncation), batched ``map`` like the reference."""
    cfg = None
    try:
        cfg = resolve_config(tokenizer_name)
    except KeyError:
        pass
    tok = load_tokenizer(tokenizer_name, cfg.vocab_size if cfg else 260)

    def encode_batch(batch):
        texts = [t.lower() if lower_case else t for t in batch[text_field]]
        ids, mask = [], []
        for t in texts:
            e = tok.encode(t)[:max_length]
            mask.append([1] * len(e) + [0] * (max_length - len(e)))
            ids.append(e + [0] * (max_length - len(e)))
        return {"input_ids": ids, "attention_mask": mask}

    if hasattr(dataset, "map"):
        return dataset.map(encode_batch, batched=True)
    return {**dataset, **encode_batch(dataset)}


# --------------------------------------------------------------- layer partials
def build_layer_partial(model_name: str, start: int, end: int, device: Optional[str] = None, seed: int = 0):
    """Layers [start, end) of a decoder LM as a callable piece (text/ids in on the first piece,
    hidden states in otherwise; hidden states or logits out).  Only that range is loaded."""
    import torch

    from .models.torch_ref import TorchPiece
    from .models.weights import load_or_init

    cfg = resolve_config(model_name)
    if device is None:
        device = "cuda" if torch.cuda.is_available() else "cpu"
    first, last = start == 0, end >= cfg.n_layers
    dtype = torch.bfloat16 if str(device).startswith("cuda") else torch.float32
    tensors = load_or_init(model_name, cfg, range(start, min(end, cfg.n_layers)), first, last, device=device,
                           dtype=dtype, seed=seed)
    piece = TorchPiece(cfg, range(start, min(end, cfg.n_layers)), first, last, tensors)
    tok = load_tokenizer(model_name, cfg.vocab_size, cfg.eos_token_id, cfg.bos_token_id)
    return piece, tok, device


build_distilbert_partial = build_layer_partial   # reference name (hf.py:180)
