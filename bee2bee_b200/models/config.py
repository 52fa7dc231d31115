"""Model architecture descriptions for the decoder families the mesh serves.

The reference ships no model configs (it defers to ``transformers``,
/root/reference/bee2bee/hf.py:23-32); these presets are the public architectures named in
BASELINE.json (distilgpt2, Llama-3-8B, Zephyr-7B-beta = Mistral-7B, gemma-2-2b) plus tiny
variants of each family for tests.  A config can also be read from a Hugging Face
``config.json`` (``ModelConfig.from_hf_dict``) so ``serve-hf --model <local dir>`` works.
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import asdict, dataclass
from typing import Dict, List, Optional


@dataclass
class ModelConfig:
    name: str = "tiny-llama"
    family: str = "llama"            # gpt2 | llama | mistral | gemma2
    vocab_size: int = 512
    hidden_size: int = 256
    n_layers: int = 2
    n_heads: int = 2
    n_kv_heads: int = 1
    head_dim: int = 128
    ffn_size: int = 512
    max_position: int = 8192
    norm: str = "rms"                # rms | ln
    norm_eps: float = 1e-5
    act: str = "silu"                # silu | gelu_tanh
    glu: bool = True
    rope_theta: float = 10000.0      # <= 0: learned absolute positions (GPT-2)
    tie_embeddings: bool = False
    bias: bool = False               # GPT-2 style biases on every linear
    sliding_window: int = 0          # 0 = full attention
    window_pattern: str = "all"      # all | alternate (Gemma-2: even layers are local)
    attn_softcap: float = 0.0
    final_softcap: float = 0.0
    query_scale: float = 0.0         # 0 -> 1/sqrt(head_dim); Gemma-2: query_pre_attn_scalar ** -0.5
    post_norms: bool = False         # Gemma-2 post-attention / post-FFN norms
    gemma_norm: bool = False         # RMSNorm weight stored as (w - 1)
    embed_scale: float = 1.0         # Gemma: sqrt(hidden)
    eos_token_id: int = -1
    bos_token_id: int = -1

    # ------------------------------------------------------------------ derived
    @property
    def q_dim(self) -> int:
        return self.n_heads * self.head_dim

    @property
    def kv_dim(self) -> int:
        return self.n_kv_heads * self.head_dim

    @property
    def softmax_scale(self) -> float:
        return self.query_scale if self.query_scale > 0 else 1.0 / math.sqrt(self.head_dim)

    def layer_window(self, layer: int) -> int:
        if self.sliding_window <= 0:
            return 0
        if self.window_pattern == "alternate":
            return self.sliding_window if layer % 2 == 0 else 0
        return self.sliding_window

    def param_count(self) -> int:
        h, f = self.hidden_size, self.ffn_size
        per = h * (self.q_dim + 2 * self.kv_dim) + self.q_dim * h + (3 if self.glu else 2) * h * f
        emb = self.vocab_size * h * (1 if self.tie_embeddings else 2)
        return self.n_layers * per + emb

    def to_dict(self) -> Dict:
        return asdict(self)

    # --------------------------------------------------------------- HF interop
    @staticmethod
    def from_hf_dict(d: Dict, name: str = "") -> "ModelConfig":
        mt = d.get("model_type", "llama")
        if mt == "gpt2":
            h = d.get("n_embd", 768)
            nh = d.get("n_head", 12)
            return ModelConfig(
                name=name or "gpt2", family="gpt2", vocab_size=d.get("vocab_size", 50257), hidden_size=h,
                n_layers=d.get("n_layer", 12), n_heads=nh, n_kv_heads=nh, head_dim=h // nh,
                ffn_size=d.get("n_inner") or 4 * h, max_position=d.get("n_positions", 1024), norm="ln",
                norm_eps=d.get("layer_norm_epsilon", 1e-5), act="gelu_tanh", glu=False, rope_theta=0.0,
                tie_embeddings=True, bias=True, eos_token_id=d.get("eos_token_id", 50256),
                bos_token_id=d.get("bos_token_id", 50256))
        # checkpoints the loader would map wrongly are rejected instead of loading "successfully" (ADVICE r1)
        if d.get("attention_bias") or d.get("mlp_bias"):
            raise ValueError(f"{name or mt}: attention_bias / mlp_bias checkpoints (Qwen-style) are not supported: "
                             "the weight map carries no bias tensors for this family")
        rs = d.get("rope_scaling")
        if rs and (rs.get("rope_type") or rs.get("type") or "default") not in ("default",):
            raise ValueError(f"{name or mt}: rope_scaling {rs!r} is not implemented (plain RoPE only)")
        h = d["hidden_size"]
        nh = d["num_attention_heads"]
        hd = d.get("head_dim") or h // nh
        common = dict(
            name=name or mt, vocab_size=d["vocab_size"], hidden_size=h, n_layers=d["num_hidden_layers"], n_heads=nh,
            n_kv_heads=d.get("num_key_value_heads", nh), head_dim=hd, ffn_size=d["intermediate_size"],
            max_position=d.get("max_position_embeddings", 8192), norm="rms", norm_eps=d.get("rms_norm_eps", 1e-5),
            rope_theta=float(d.get("rope_theta", 10000.0)), tie_embeddings=bool(d.get("tie_word_embeddings", False)),
            eos_token_id=_first_int(d.get("eos_token_id", -1)), bos_token_id=_first_int(d.get("bos_token_id", -1)))
        if mt == "gemma2":
            return ModelConfig(
                family="gemma2", act="gelu_tanh", glu=True, sliding_window=d.get("sliding_window", 4096),
                window_pattern="alternate", attn_softcap=float(d.get("attn_logit_softcapping") or 0.0),
                final_softcap=float(d.get("final_logit_softcapping") or 0.0),
                query_scale=float(d.get("query_pre_attn_scalar", hd)) ** -0.5, post_norms=True, gemma_norm=True,
                embed_scale=math.sqrt(h), **{**common, "tie_embeddings": True})
        if mt == "mistral":
            return ModelConfig(family="mistral", act="silu", glu=True, sliding_window=d.get("sliding_window") or 0,
                               **common)
        return ModelConfig(family="llama", act="silu", glu=True, **common)

    def to_hf_dict(self) -> Dict:
        """A ``config.json`` that ``transformers`` accepts for this architecture."""
        if self.family == "gpt2":
            return {"model_type": "gpt2", "architectures": ["GPT2LMHeadModel"], "vocab_size": self.vocab_size,
                    "n_embd": self.hidden_size, "n_layer": self.n_layers, "n_head": self.n_heads,
                    "n_positions": self.max_position, "n_ctx": self.max_position, "n_inner": self.ffn_size,
                    "activation_function": "gelu_new", "layer_norm_epsilon": self.norm_eps,
                    "bos_token_id": self.bos_token_id, "eos_token_id": self.eos_token_id,
                    "resid_pdrop": 0.0, "embd_pdrop": 0.0, "attn_pdrop": 0.0}
        base = {"vocab_size": self.vocab_size, "hidden_size": self.hidden_size,
                "num_hidden_layers": self.n_layers, "num_attention_heads": self.n_heads,
                "num_key_value_heads": self.n_kv_heads, "head_dim": self.head_dim,
                "intermediate_size": self.ffn_size, "max_position_embeddings": self.max_position,
                "rms_norm_eps": self.norm_eps, "rope_theta": self.rope_theta,
                "tie_word_embeddings": self.tie_embeddings, "bos_token_id": self.bos_token_id,
                "eos_token_id": self.eos_token_id, "attention_bias": False, "mlp_bias": False,
                "attention_dropout": 0.0}
        if self.family == "gemma2":
            base.update({"model_type": "gemma2", "architectures": ["Gemma2ForCausalLM"],
                         "hidden_activation": "gelu_pytorch_tanh", "sliding_window": self.sliding_window,
                         "attn_logit_softcapping": self.attn_softcap or None,
                         "final_logit_softcapping": self.final_softcap or None,
                         "query_pre_attn_scalar": round(self.softmax_scale ** -2)})
        elif self.family == "mistral":
            base.update({"model_type": "mistral", "architectures": ["MistralForCausalLM"], "hidden_act": "silu",
                         "sliding_window": self.sliding_window or None})
        else:
            base.update({"model_type": "llama", "architectures": ["LlamaForCausalLM"], "hidden_act": "silu"})
        return base


def _first_int(v) -> int:
    if isinstance(v, (list, tuple)):
        return int(v[0]) if v else -1
    return -1 if v is None else int(v)


def _gpt2(name, layers, hidden, heads):
    return ModelConfig(name=name, family="gpt2", vocab_size=50257, hidden_size=hidden, n_layers=layers, n_heads=heads,
                       n_kv_heads=heads, head_dim=hidden // heads, ffn_size=4 * hidden, max_position=1024, norm="ln",
                       norm_eps=1e-5, act="gelu_tanh", glu=False, rope_theta=0.0, tie_embeddings=True, bias=True,
                       eos_token_id=50256, bos_token_id=50256)


PRESETS: Dict[str, ModelConfig] = {
    "distilgpt2": _gpt2("distilgpt2", 6, 768, 12),
    "gpt2": _gpt2("gpt2", 12, 768, 12),
    "llama-3-8b": ModelConfig(name="llama-3-8b", family="llama", vocab_size=128256, hidden_size=4096, n_layers=32,
                              n_heads=32, n_kv_heads=8, head_dim=128, ffn_size=14336, max_position=8192,
                              norm_eps=1e-5, rope_theta=500000.0, eos_token_id=128001, bos_token_id=128000),
    "zephyr-7b-beta": ModelConfig(name="zephyr-7b-beta", family="mistral", vocab_size=32000, hidden_size=4096,
                                  n_layers=32, n_heads=32, n_kv_heads=8, head_dim=128, ffn_size=14336,
                                  max_position=32768, norm_eps=1e-5, rope_theta=10000.0, sliding_window=4096,
                                  eos_token_id=2, bos_token_id=1),
    "gemma-2-2b": ModelConfig(name="gemma-2-2b", family="gemma2", vocab_size=256000, hidden_size=2304, n_layers=26,
                              n_heads=8, n_kv_heads=4, head_dim=256, ffn_size=9216, max_position=8192,
                              norm_eps=1e-6, act="gelu_tanh", rope_theta=10000.0, tie_embeddings=True,
                              sliding_window=4096, window_pattern="alternate", attn_softcap=50.0, final_softcap=30.0,
                              query_scale=256 ** -0.5, post_norms=True, gemma_norm=True,
                              embed_scale=math.sqrt(2304), eos_token_id=1, bos_token_id=2),
    # tiny variants (tests / smoke): same code paths, kernel-friendly shapes
    "tiny-llama": ModelConfig(name="tiny-llama", family="llama", vocab_size=512, hidden_size=256, n_layers=4,
                              n_heads=4, n_kv_heads=2, head_dim=128, ffn_size=512, rope_theta=500000.0,
                              eos_token_id=1, bos_token_id=0),
    "tiny-mistral": ModelConfig(name="tiny-mistral", family="mistral", vocab_size=512, hidden_size=256, n_layers=4,
                                n_heads=4, n_kv_heads=2, head_dim=128, ffn_size=512, sliding_window=96,
                                eos_token_id=1, bos_token_id=0),
    "tiny-gemma2": ModelConfig(name="tiny-gemma2", family="gemma2", vocab_size=512, hidden_size=256, n_layers=4,
                               n_heads=2, n_kv_heads=1, head_dim=256, ffn_size=512, norm_eps=1e-6, act="gelu_tanh",
                               tie_embeddings=True, sliding_window=96, window_pattern="alternate", attn_softcap=50.0,
                               final_softcap=30.0, query_scale=256 ** -0.5, post_norms=True, gemma_norm=True,
                               embed_scale=16.0, eos_token_id=1, bos_token_id=0),
    "tiny-gpt2": _gpt2("tiny-gpt2", 4, 128, 2),
    # Llama-3-8B layer shapes (hidden 4096, GQA 32:8, FFN 14336), 8 layers, small vocabulary: multi-GPU correctness
    # tests at the real GEMM / handoff tile shapes without 16 GB of weights
    "mini-llama-4096": ModelConfig(name="mini-llama-4096", family="llama", vocab_size=32000, hidden_size=4096,
                                   n_layers=8, n_heads=32, n_kv_heads=8, head_dim=128, ffn_size=14336,
                                   rope_theta=500000.0, eos_token_id=1, bos_token_id=0),
}
PRESETS["tiny-gpt2"].vocab_size = 384
PRESETS["tiny-gpt2"].eos_token_id = 1
PRESETS["tiny-gpt2"].bos_token_id = 0

ALIASES = {
    "meta-llama/meta-llama-3-8b": "llama-3-8b", "meta-llama/llama-3-8b": "llama-3-8b", "llama3": "llama-3-8b",
    "llama-3-8b-instruct": "llama-3-8b", "huggingfaceh4/zephyr-7b-beta": "zephyr-7b-beta",
    "zephyr": "zephyr-7b-beta", "mistral-7b": "zephyr-7b-beta", "google/gemma-2-2b": "gemma-2-2b",
    "gemma2:2b": "gemma-2-2b", "gemma2": "gemma-2-2b", "distilbert/distilgpt2": "distilgpt2",
    "openai-community/gpt2": "gpt2",
}


def resolve_config(model: str) -> ModelConfig:
    """Preset name, alias, or a local directory containing ``config.json``."""
    if os.path.isdir(model) and os.path.exists(os.path.join(model, "config.json")):
        with open(os.path.join(model, "config.json")) as f:
            return ModelConfig.from_hf_dict(json.load(f), name=os.path.basename(os.path.normpath(model)))
    key = model.lower()
    key = ALIASES.get(key, key)
    if key in PRESETS:
        return PRESETS[key]
    tail = key.split("/")[-1]
    tail = ALIASES.get(tail, tail)
    if tail in PRESETS:
        return PRESETS[tail]
    raise KeyError(f"unknown model '{model}' (presets: {sorted(PRESETS)})")


def split_layers(n_layers: int, pieces: int) -> List[range]:
    """Contiguous layer ranges, earlier pieces take the remainder (26 over 4 -> 7/7/6/6)."""
    pieces = max(1, min(pieces, n_layers))
    base, rem = divmod(n_layers, pieces)
    out, start = [], 0
    for i in range(pieces):
        n = base + (1 if i < rem else 0)
        out.append(range(start, start + n))
        start += n
    return out


def balanced_split(cfg: "ModelConfig", pieces: int) -> List[range]:
    """Contiguous layer ranges that minimise the heaviest piece when the last piece also streams the
    lm_head (Llama-3-8B: the 1.05 GB head weighs 2.4 decoder layers) -- the wavefront runs at the pace
    of its slowest stage.  Falls back to ``split_layers`` when the head is negligible."""
    pieces = max(1, min(pieces, cfg.n_layers))
    h, f = cfg.hidden_size, cfg.ffn_size
    layer = h * (cfg.q_dim + 2 * cfg.kv_dim) + cfg.q_dim * h + (3 if cfg.glu else 2) * h * f
    head = cfg.vocab_size * h
    if pieces == 1 or head < 0.5 * layer:
        return split_layers(cfg.n_layers, pieces)
    best, best_cost = None, None
    for last_n in range(1, cfg.n_layers - pieces + 2):
        rest = split_layers(cfg.n_layers - last_n, pieces - 1)
        cost = max(max(len(r) for r in rest) * layer, last_n * layer + head)
        if best_cost is None or cost <= best_cost:     # ties -> the more even split (larger last piece)
            best, best_cost = rest + [range(cfg.n_layers - last_n, cfg.n_layers)], cost
    return best


def supports_half_layer_pieces(cfg: "ModelConfig") -> bool:
    """A piece boundary may fall between the attention and the MLP block of a layer when both boundary GEMMs
    are the fused kinds the handoff needs: O-proj with residual epilogue (tail) and gate/up with the RMSNorm
    folded in (head) -- the Llama / Mistral graphs."""
    return cfg.norm == "rms" and not cfg.post_norms and cfg.glu and not cfg.bias


UNITS_PER_LAYER = 3       # attention block (QKV GEMM, attention, O-proj) | gate/up GEMM | down GEMM


def piece_units(cfg: "ModelConfig", pieces: int, bounds: Optional[List[int]] = None) -> List[tuple]:
    """Piece boundaries in THIRD-OF-A-LAYER units: unit 3l is the attention block of layer l (QKV GEMM, attention,
    O-proj), 3l+1 its gate/up GEMM, 3l+2 its down GEMM -- any GEMM can be the fused tail GEMM of a piece and any GEMM
    its head.  Returns ``pieces`` contiguous ``(u0, u1)`` ranges that minimise the heaviest stage of the wavefront under
    a bytes-plus-launch-latency cost model (a decode step is weight-bandwidth bound with a few us of fixed cost per
    kernel); the last piece also carries the lm_head and the sampler.  Llama-3-8B over 8 GPUs: whole layers give
    5/4/4/4/4/4/4/3 (+head) = 0.81 of the ideal stage time, half layers (round 1) 0.92, thirds 0.97.  ``bounds``
    overrides the search (tests).  Graphs without the fused RMSNorm / GLU epilogues are cut at whole layers."""
    UPL = UNITS_PER_LAYER
    U = UPL * cfg.n_layers
    if bounds is not None:
        assert bounds[0] == 0 and bounds[-1] == U and all(a < b for a, b in zip(bounds, bounds[1:])), bounds
        return list(zip(bounds[:-1], bounds[1:]))
    pieces = max(1, min(pieces, cfg.n_layers))
    if pieces == 1 or not supports_half_layer_pieces(cfg):
        return [(UPL * r.start, UPL * r.stop) for r in balanced_split(cfg, pieces)]
    # stage time model of a decode step: weight bytes at an effective 6.4 TB/s plus a fixed cost per kernel; the last
    # piece adds the lm_head GEMM and the sampler.  These constants are not measured on H100 (data-sheet HBM3: 3.35
    # TB/s).  The boundaries depend on them: the streaming rate sets how much a weight byte costs against the fixed
    # per-kernel cost, so a different rate can move a cut.
    h, f = cfg.hidden_size, cfg.ffn_size
    us_per_elem = 2.0 / 6.4e6                            # bf16 element -> microseconds of weight streaming
    launch = 7.0
    attn = (h * (cfg.q_dim + 2 * cfg.kv_dim) + cfg.q_dim * h) * us_per_elem + 3 * launch
    gu = 2 * h * f * us_per_elem + 4.0
    down = h * f * us_per_elem + launch
    head = cfg.vocab_size * h * us_per_elem + launch + 30.0
    cost = [(attn, gu, down)[u % UPL] for u in range(U)]
    pre = [0.0]
    for c in cost:
        pre.append(pre[-1] + c)
    INF = float("inf")
    # best[k][u]: minimal max-stage cost of covering units [0, u) with k pieces
    best = [[INF] * (U + 1) for _ in range(pieces + 1)]
    arg = [[0] * (U + 1) for _ in range(pieces + 1)]
    best[0][0] = 0.0
    for k in range(1, pieces + 1):
        for u in range(k, U + 1):
            for v in range(k - 1, u - 1):          # every piece spans >= 2 units (no lone GEMM)
                if best[k - 1][v] == INF:
                    continue
                stage = pre[u] - pre[v] + (head if (k == pieces and u == U) else 0.0)
                c = max(best[k - 1][v], stage)
                if c < best[k][u]:
                    best[k][u], arg[k][u] = c, v
    out, u = [], U
    for k in range(pieces, 0, -1):
        v = arg[k][u]
        out.append((v, u))
        u = v
    return out[::-1]


def unit_layers(units: tuple) -> range:
    """layers touched by a ``(u0, u1)`` unit range"""
    return range(units[0] // UNITS_PER_LAYER, (units[1] - 1) // UNITS_PER_LAYER + 1)
