"""Plain-PyTorch implementation of every supported decoder family.

Two jobs: (1) the numerical oracle every CUDA kernel / fused path is tested against, and
(2) the execution backend on machines without a H100 (CPU plumbing config of
BASELINE.json: distilgpt2 split in two pieces over the loopback mesh).  Semantics follow
the Hugging Face modelling code the reference delegates to
(/root/reference/bee2bee/hf.py:23-44).
"""
from __future__ import annotations

from typing import Dict, Iterable, Optional, Tuple

import torch
import torch.nn.functional as F

from .config import ModelConfig, rope_inv_freq
from .weights import Tensors

KV = Dict[int, Tuple[torch.Tensor, torch.Tensor]]


def rms_norm(x: torch.Tensor, w: torch.Tensor, eps: float, plus_one: bool) -> torch.Tensor:
    xf = x.float()
    y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    g = w.float() + 1.0 if plus_one else w.float()
    return (y * g).to(x.dtype)


def layer_norm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float) -> torch.Tensor:
    return F.layer_norm(x.float(), (x.shape[-1],), w.float(), b.float(), eps).to(x.dtype)


def gelu_tanh(x: torch.Tensor) -> torch.Tensor:
    return F.gelu(x, approximate="tanh")


def rope(x: torch.Tensor, positions: torch.Tensor, theta: float, inv_freq: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [B, T, H, D]; rotate-half convention (pairs (i, i + D/2)), fp32 angles.  ``inv_freq``: the [D/2] frequency
    table of a scaled config (``config.rope_inv_freq``); None = theta^(-2i/D)."""
    d = x.shape[-1]
    if inv_freq is None:
        inv = theta ** (-torch.arange(0, d, 2, device=x.device, dtype=torch.float32) / d)
    else:
        inv = inv_freq.to(x.device)
    ang = positions.float()[..., None] * inv                      # [B, T, D/2]
    cos, sin = ang.cos()[:, :, None, :], ang.sin()[:, :, None, :]
    x1, x2 = x.float()[..., : d // 2], x.float()[..., d // 2:]
    return torch.cat([x1 * cos - x2 * sin, x2 * cos + x1 * sin], -1).to(x.dtype)


class TorchPiece:
    """Layers ``layers`` of a model (+ embeddings if ``first``, + final norm / lm_head if ``last``)."""

    def __init__(self, cfg: ModelConfig, layers: Iterable[int], first: bool, last: bool, tensors: Tensors):
        self.cfg, self.layers, self.first, self.last, self.t = cfg, list(layers), first, last, tensors
        self.inv_freq = rope_inv_freq(cfg)

    # -- helpers -----------------------------------------------------------------
    def _norm(self, x, name: str):
        c = self.cfg
        if c.norm == "ln":
            return layer_norm(x, self.t[name + "_w"], self.t[name + "_b"], c.norm_eps)
        return rms_norm(x, self.t[name + "_w"], c.norm_eps, c.gemma_norm)

    def _lin(self, x, w: str, b: Optional[str] = None):
        y = x @ self.t[w].to(x.dtype).t()
        if b is not None and b in self.t:
            y = y + self.t[b].to(x.dtype)
        return y

    def new_cache(self) -> KV:
        return {}

    # -- forward ------------------------------------------------------------------
    def forward(self, inp: torch.Tensor, positions: torch.Tensor, cache: Optional[KV] = None,
                logits_last_only: bool = False) -> torch.Tensor:
        """inp: ids [B, T] (first piece) or hidden [B, T, H]; positions [B, T] absolute."""
        c = self.cfg
        if self.first:
            x = self.t["embed"][inp]
            if c.embed_scale != 1.0:
                x = x * torch.tensor(c.embed_scale, dtype=x.dtype)
            if c.rope_theta <= 0:
                x = x + self.t["pos_embed"][positions]
        else:
            x = inp
        B, T, _ = x.shape
        for l in self.layers:
            p = f"l{l}."
            h = self._norm(x, p + "ln1")
            q = self._lin(h, p + "wq", p + "bq").view(B, T, c.n_heads, c.head_dim)
            k = self._lin(h, p + "wk", p + "bk").view(B, T, c.n_kv_heads, c.head_dim)
            v = self._lin(h, p + "wv", p + "bv").view(B, T, c.n_kv_heads, c.head_dim)
            if c.rope_theta > 0:
                q, k = rope(q, positions, c.rope_theta, self.inv_freq), rope(k, positions, c.rope_theta, self.inv_freq)
            k, v = k.transpose(1, 2), v.transpose(1, 2)                     # [B, n_kv, T, D]
            if cache is not None:
                if l in cache:
                    k = torch.cat([cache[l][0], k], 2)
                    v = torch.cat([cache[l][1], v], 2)
                cache[l] = (k, v)
            S = k.shape[2]
            g = c.n_heads // c.n_kv_heads
            qh = q.transpose(1, 2).reshape(B, c.n_kv_heads, g, T, c.head_dim)
            s = torch.einsum("bkgtd,bksd->bkgts", qh.float(), k.float()) * c.softmax_scale
            if c.attn_softcap > 0:
                s = torch.tanh(s / c.attn_softcap) * c.attn_softcap
            kpos = torch.arange(S, device=x.device)[None, None, :]           # keys sit at positions 0..S-1
            qpos = positions[:, :, None]
            ok = kpos <= qpos
            w = c.layer_window(l)
            if w > 0:
                ok = ok & (kpos > qpos - w)
            s = s.masked_fill(~ok[:, None, None, :, :], float("-inf"))
            a = torch.einsum("bkgts,bksd->bkgtd", torch.softmax(s, -1), v.float()).to(x.dtype)
            a = a.reshape(B, c.n_heads, T, c.head_dim).transpose(1, 2).reshape(B, T, c.q_dim)
            o = self._lin(a, p + "wo", p + "bo")
            if c.post_norms:
                o = rms_norm(o, self.t[p + "post_attn_w"], c.norm_eps, c.gemma_norm)
            x = x + o
            h = self._norm(x, p + "ln2")
            if c.glu:
                gate = self._lin(h, p + "w_gate")
                gate = gelu_tanh(gate) if c.act == "gelu_tanh" else F.silu(gate)
                m = self._lin(gate * self._lin(h, p + "w_up"), p + "w_down")
            else:
                m = self._lin(gelu_tanh(self._lin(h, p + "w_up", p + "b_up")), p + "w_down", p + "b_down")
            if c.post_norms:
                m = rms_norm(m, self.t[p + "post_ffn_w"], c.norm_eps, c.gemma_norm)
            x = x + m
        if not self.last:
            return x
        if logits_last_only:
            x = x[:, -1:, :]
        x = self._norm(x, "final_norm")
        head = self.t["embed"] if c.tie_embeddings else self.t["lm_head"]
        logits = x.float() @ head.float().t()
        if c.final_softcap > 0:
            logits = torch.tanh(logits / c.final_softcap) * c.final_softcap
        return logits


COUNT_MAX = 32767       # generated-token counts saturate here (the sampler's int16 count table)


def sample_reference(logits: torch.Tensor, seen: Optional[torch.Tensor], temperature: float, top_p: float,
                     rep_penalty: float, generator: Optional[torch.Generator] = None, top_k: int = 0,
                     min_p: float = 0.0, counts: Optional[torch.Tensor] = None, presence: float = 0.0,
                     frequency: float = 0.0, bias: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> torch.Tensor:
    """HF-processor semantics (logit bias -> repetition penalty -> presence / frequency penalty -> temperature -> top-k
    -> top-p -> min-p -> multinomial / greedy when temperature <= 0), cf. /root/reference/bee2bee/hf.py:91-105.
    ``bias`` = (ids int64 [n], values fp32 [n]): every row's logit of ids[j] gains values[j] in fp32 (vLLM's and
    OpenAI's ``logit_bias``; ids unique); the other ids are untouched.  The logits arrive soft-capped, so the bias
    follows soft-cap and the repetition penalty sees the biased logit.
    logits [B, V] fp32; seen [B, V] bool of ids already in the context.  ``top_k`` keeps the tokens at least as likely
    as the k-th (ties kept; <= 0 or >= V = off); top-p then sees the top-k survivors renormalised; ``min_p`` keeps
    p >= min_p * p_max (<= 0 = off).  ``counts`` [B, V] holds how often each id was generated (prompt excluded); where
    it is positive, l = (l - frequency * c) - presence in fp32, as vLLM / OpenAI define the two penalties (0 = off);
    greedy rows are penalised too."""
    l = logits.float().clone()
    if bias is not None and bias[0].numel() > 0:
        ids, vals = bias
        l[:, ids] = l[:, ids] + vals.to(torch.float32)
    if seen is not None and rep_penalty != 1.0:
        pen = torch.where(l > 0, l / rep_penalty, l * rep_penalty)
        l = torch.where(seen, pen, l)
    if counts is not None and (presence != 0.0 or frequency != 0.0):
        c = counts.to(torch.float32)
        pf = (l - torch.tensor(frequency, dtype=torch.float32) * c) - torch.tensor(presence, dtype=torch.float32)
        l = torch.where(counts > 0, pf, l)
    if not temperature > 0:
        return l.argmax(-1)
    l = l / temperature
    if 0 < top_k < l.shape[-1]:
        kth = torch.topk(l, top_k, dim=-1).values[..., -1:]
        l = l.masked_fill(l < kth, float("-inf"))
    if top_p < 1.0:
        sl, si = torch.sort(l, descending=False)
        cum = sl.softmax(-1).cumsum(-1)
        remove = cum <= (1 - top_p)
        remove[..., -1:] = False
        l = l.masked_fill(remove.scatter(1, si, remove), float("-inf"))
    if min_p > 0.0:
        p = l.softmax(-1)
        l = l.masked_fill(p < min(min_p, 1.0) * p.amax(-1, keepdim=True), float("-inf"))
    return torch.multinomial(l.softmax(-1), 1, generator=generator).squeeze(-1)


class SequenceSampler:
    """One sequence's sampling on the CPU: its controls (any ``engine.core.SamplerControls``), its generator, the ids
    in its context (repetition penalty), how often each id was generated (presence / frequency penalties) and its
    logit bias."""

    def __init__(self, controls, vocab: int, prompt: Iterable[int], generator: torch.Generator):
        self.controls, self.generator = controls, generator
        self.seen = torch.zeros(1, vocab, dtype=torch.bool)
        self.seen[0, torch.tensor(sorted({int(t) for t in prompt}), dtype=torch.long)] = True
        self.counts = torch.zeros(1, vocab, dtype=torch.int32)       # generated tokens only, saturating at COUNT_MAX
        lb = controls.logit_bias
        self.bias = ((torch.tensor([int(t) for t in lb], dtype=torch.long),
                      torch.tensor([float(v) for v in lb.values()], dtype=torch.float32)) if lb else None)

    def draw(self, logits: torch.Tensor) -> int:
        """The next id from ``logits`` [>= vocab] of the sequence's last position; it is then seen and counted."""
        c = self.controls
        penalised = c.presence_penalty != 0.0 or c.frequency_penalty != 0.0
        tok = int(sample_reference(logits[None, :self.seen.shape[1]].cpu(), self.seen, c.temperature, c.top_p,
                                   c.repetition_penalty, self.generator, top_k=c.top_k, min_p=c.min_p,
                                   counts=self.counts if penalised else None, presence=c.presence_penalty,
                                   frequency=c.frequency_penalty, bias=self.bias))
        self.seen[0, tok] = True
        self.counts[0, tok] = min(int(self.counts[0, tok]) + 1, COUNT_MAX)
        return tok


def top_p_keep_mask(logits: torch.Tensor, temperature: float, top_p: float) -> torch.Tensor:
    """[B, V] bool: the nucleus the sampler is allowed to draw from (oracle for the CUDA sampler)."""
    l = logits.float() / temperature
    sl, si = torch.sort(l, descending=False)
    cum = sl.softmax(-1).cumsum(-1)
    remove = cum <= (1 - top_p)
    remove[..., -1:] = False
    return ~remove.scatter(1, si, remove)
