"""Comparator B of BASELINE.md: OUR CONSTRUCTED NCCL(+cuBLAS) pipeline.  **Not the reference's build** -- the reference
has no multi-GPU path at all (SURVEY.md R2/R3); this is the "path that only calls NCCL for the named ops" that
BASELINE.json tells the product to beat, built by us with library calls only:

  * the same piece split (``models.config.piece_units`` rounded to whole layers) and the same
    micro-batch groups / wavefront order as the product,
  * every op is a PyTorch library call: cuBLAS GEMMs (``torch.matmul``), ``F.scaled_dot_product_attention`` (flash /
    mem-efficient kernels) over a contiguous static KV cache, ATen RMSNorm / RoPE / SiLU, ATen sort + multinomial
    sampling with the reference's generation defaults,
  * the hidden-state hop between consecutive pieces is ``torch.distributed`` NCCL send / recv; sampled tokens return
    to piece 0 over a second NCCL communicator,
  * per (rank, group) the compute between recv and send is captured in a CUDA graph (what a production NCCL pipeline
    does), the NCCL calls stay outside.

None of this repo's kernels, engine or mesh code is on this path (only the model presets and the random-init weight
generator, so both arms hold bit-identical bf16 weights).  Llama / Mistral family with equal-length prompts (the
bench shapes); Gemma-2 runs with a manual soft-capped attention.
"""
from __future__ import annotations

import math
import os
from typing import List, Optional

import torch
import torch.distributed as dist
import torch.nn.functional as F


def _rope(x: torch.Tensor, pos: torch.Tensor, theta: float) -> torch.Tensor:
    """x [B, T, H, D], pos [B, T]; rotate-half convention, fp32 angles."""
    d = x.shape[-1]
    inv = theta ** (-torch.arange(0, d, 2, device=x.device, dtype=torch.float32) / d)
    ang = pos.float()[..., None] * inv
    cos, sin = ang.cos()[:, :, None, :], ang.sin()[:, :, None, :]
    x1, x2 = x.float()[..., : d // 2], x.float()[..., d // 2:]
    return torch.cat([x1 * cos - x2 * sin, x2 * cos + x1 * sin], -1).to(x.dtype)


def _rms(x: torch.Tensor, w: torch.Tensor, eps: float, plus_one: bool) -> torch.Tensor:
    xf = x.float()
    y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return (y * (w.float() + 1.0 if plus_one else w.float())).to(x.dtype)


class NcclPipeline:
    def __init__(self, model: str, rank: int, world: int, device: torch.device, groups: int, group_batch: int,
                 max_len: int, seed: int = 0, use_graphs: bool = True):
        from bee2bee_b200.models.config import piece_units, resolve_config
        from bee2bee_b200.models.weights import load_or_init

        self.cfg = c = resolve_config(model)
        assert c.norm == "rms" and c.glu, "comparator B covers the RMSNorm + GLU families (Llama / Mistral / Gemma-2)"
        if c.rope_scaling:
            raise ValueError(f"{c.name}: comparator B implements plain RoPE only, not rope_scaling {c.rope_scaling}")
        self.rank, self.world, self.dev = rank, world, device
        self.groups, self.gb, self.max_len = groups, group_batch, max_len
        self.first, self.last = rank == 0, rank == world - 1
        units = piece_units(c, world)
        # whole layers (nearest boundary): a cut inside a layer would need extra payloads per hop
        cuts = [0] + [min(c.n_layers, (u1 + 1) // 3) for _, u1 in units]
        cuts[-1] = c.n_layers
        for i in range(1, len(cuts)):
            cuts[i] = max(cuts[i], cuts[i - 1] + 1) if i < len(cuts) - 1 else cuts[i]
        self.layers = list(range(cuts[rank], cuts[rank + 1]))
        self.t = load_or_init(model, c, self.layers, self.first, self.last, device=device, dtype=torch.bfloat16, seed=seed)
        bf = torch.bfloat16
        self.wqkv = {l: torch.cat([self.t[f"l{l}.wq"], self.t[f"l{l}.wk"], self.t[f"l{l}.wv"]], 0) for l in self.layers}
        self.wgu = {l: torch.cat([self.t[f"l{l}.w_gate"], self.t[f"l{l}.w_up"]], 0) for l in self.layers}
        gb, G = group_batch, groups
        self.fa = self._probe_flash_attn()
        shape = (G, gb, max_len, c.n_kv_heads, c.head_dim) if self.fa else (G, gb, c.n_kv_heads, max_len, c.head_dim)
        self.k = {l: torch.zeros(shape, device=device, dtype=bf) for l in self.layers}
        self.v = {l: torch.zeros(shape, device=device, dtype=bf) for l in self.layers}
        self.h_in = torch.zeros((G, gb, c.hidden_size), device=device, dtype=bf)
        self.h_out = torch.zeros((G, gb, c.hidden_size), device=device, dtype=bf)
        self.tok = torch.zeros((G, gb), device=device, dtype=torch.int64)
        self.pos = torch.zeros((G, gb), device=device, dtype=torch.int64)       # position of the token being decoded
        self.seen = torch.zeros((G, gb, c.vocab_size), device=device, dtype=torch.bool) if self.last else None
        self.temperature, self.top_p, self.rep = 0.7, 0.95, 1.15
        self.stream = torch.cuda.Stream(device=device)
        self.side = torch.cuda.Stream(device=device)
        self.tok_group = dist.new_group(backend="nccl") if world > 1 else None
        self.graphs = {}
        self._tok_ev = {}
        self.use_graphs = use_graphs
        self.nccl_calls = 0
        self.kernel_graphs = 0
        self.arange = torch.arange(max_len, device=device)

    def _probe_flash_attn(self):
        """flash-attn's KV-cache kernel (library) when it runs on this GPU; otherwise SDPA over the masked static cache"""
        if os.environ.get("B2B_NCCL_ARM_FLASH", "1") != "1":
            return None
        try:
            import flash_attn
            q = torch.zeros((1, 1, self.cfg.n_heads, self.cfg.head_dim), device=self.dev, dtype=torch.bfloat16)
            kc = torch.zeros((1, 64, self.cfg.n_kv_heads, self.cfg.head_dim), device=self.dev, dtype=torch.bfloat16)
            flash_attn.flash_attn_with_kvcache(q, kc, kc.clone(), k=kc[:, :1], v=kc[:, :1],
                                               cache_seqlens=torch.zeros(1, device=self.dev, dtype=torch.int32), causal=True)
            torch.cuda.synchronize(self.dev)
            return flash_attn
        except Exception:
            return None

    # ------------------------------------------------------------------ model math (library calls only)
    def _attn(self, q, k, v, mask, l):
        c = self.cfg
        if c.attn_softcap > 0:
            g = c.n_heads // c.n_kv_heads
            B, H, T, D = q.shape
            qh = q.view(B, c.n_kv_heads, g, T, D)
            s = torch.einsum("bkgtd,bksd->bkgts", qh, k).float() * c.softmax_scale
            s = torch.tanh(s / c.attn_softcap) * c.attn_softcap
            s = s.masked_fill(~mask[:, None], float("-inf"))
            return torch.einsum("bkgts,bksd->bkgtd", torch.softmax(s, -1).to(v.dtype), v).reshape(B, H, T, D)
        return F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=c.softmax_scale, enable_gqa=True)

    def _layers(self, x, pos, g, T):
        """x [gb, T, H]; pos [gb, T] absolute positions; appends K/V at ``pos`` into the static cache of group g."""
        c = self.cfg
        B = x.shape[0]
        kpos = self.arange[None, None, :]                                      # [1, 1, L]
        for l in self.layers:
            p = f"l{l}."
            h = _rms(x, self.t[p + "ln1_w"], c.norm_eps, c.gemma_norm)
            qkv = h @ self.wqkv[l].t()
            q, k, v = qkv.split([c.q_dim, c.kv_dim, c.kv_dim], -1)
            q = _rope(q.view(B, T, c.n_heads, c.head_dim), pos, c.rope_theta).transpose(1, 2)
            k = _rope(k.view(B, T, c.n_kv_heads, c.head_dim), pos, c.rope_theta).transpose(1, 2)
            v = v.view(B, T, c.n_kv_heads, c.head_dim).transpose(1, 2)
            w = c.layer_window(l)
            if self.fa is not None:
                qf, kf, vf = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)          # [B, T, heads, D]
                kw = dict(softmax_scale=c.softmax_scale, causal=True, window_size=((w - 1, 0) if w > 0 else (-1, -1)),
                          softcap=float(c.attn_softcap))
                if T == 1:
                    # appends k/v at cache_seqlens and attends over [0, seqlen]: one library kernel, graph-capturable
                    a = self.fa.flash_attn_with_kvcache(qf, self.k[l][g], self.v[l][g], k=kf, v=vf,
                                                        cache_seqlens=pos[:, 0].to(torch.int32), **kw)
                else:
                    self.k[l][g][:, :T].copy_(kf)
                    self.v[l][g][:, :T].copy_(vf)
                    a = self.fa.flash_attn_func(qf, kf, vf, **kw)
                a = a.reshape(B, T, c.q_dim)
            else:
                idx = pos[:, None, :, None].expand(B, c.n_kv_heads, T, c.head_dim)
                self.k[l][g].scatter_(2, idx, k)
                self.v[l][g].scatter_(2, idx, v)
                ok = kpos <= pos[:, :, None]                                   # [B, T, L] causal over the static cache
                if w > 0:
                    ok = ok & (kpos > pos[:, :, None] - w)
                a = self._attn(q, self.k[l][g], self.v[l][g], ok[:, None], l)
                a = a.transpose(1, 2).reshape(B, T, c.q_dim)
            o = a @ self.t[p + "wo"].t()
            if c.post_norms:
                o = _rms(o, self.t[p + "post_attn_w"], c.norm_eps, c.gemma_norm)
            x = x + o
            h = _rms(x, self.t[p + "ln2_w"], c.norm_eps, c.gemma_norm)
            gu = h @ self.wgu[l].t()
            gate, up = gu.split(c.ffn_size, -1)
            gate = F.gelu(gate, approximate="tanh") if c.act == "gelu_tanh" else F.silu(gate)
            m = (gate * up) @ self.t[p + "w_down"].t()
            if c.post_norms:
                m = _rms(m, self.t[p + "post_ffn_w"], c.norm_eps, c.gemma_norm)
            x = x + m
        return x

    def _embed(self, ids):
        x = self.t["embed"][ids]
        if self.cfg.embed_scale != 1.0:
            x = x * torch.tensor(self.cfg.embed_scale, dtype=x.dtype)
        return x

    def _sample(self, x_last, g):
        """x_last [gb, H] -> token ids [gb]; reference generation defaults (rep. penalty, temperature, top-p)."""
        c = self.cfg
        x = _rms(x_last, self.t["final_norm_w"], c.norm_eps, c.gemma_norm)
        head = self.t["embed"] if c.tie_embeddings else self.t["lm_head"]
        l = (x @ head.t()).float()
        if c.final_softcap > 0:
            l = torch.tanh(l / c.final_softcap) * c.final_softcap
        pen = torch.where(l > 0, l / self.rep, l * self.rep)
        l = torch.where(self.seen[g], pen, l) / self.temperature
        sl, si = torch.sort(l, descending=False)
        cum = sl.softmax(-1).cumsum(-1)
        remove = cum <= (1 - self.top_p)
        remove[..., -1:] = False
        l = l.masked_fill(remove.scatter(1, si, remove), float("-inf"))
        tok = torch.multinomial(l.softmax(-1), 1).squeeze(-1)
        self.seen[g].scatter_(1, tok[:, None], True)
        return tok

    # ------------------------------------------------------------------ one stage of one group
    def _stage_decode(self, g):
        x = self._embed(self.tok[g])[:, None, :] if self.first else self.h_in[g][:, None, :]
        y = self._layers(x, self.pos[g][:, None], g, 1)
        if self.last:
            self.tok[g].copy_(self._sample(y[:, 0], g))
        else:
            self.h_out[g].copy_(y[:, 0])
        self.pos[g].add_(1)

    def _graph(self, g):
        if not self.use_graphs:
            return None
        gr = self.graphs.get(g)
        if gr is None:
            saved = (self.pos[g].clone(), self.tok[g].clone(), None if self.seen is None else self.seen[g].clone())
            with torch.cuda.stream(self.stream):
                self._stage_decode(g)                 # warm-up (cuBLAS workspaces, SDPA heuristics)
                self.stream.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr, stream=self.stream):
                    self._stage_decode(g)
            self.stream.synchronize()
            self.pos[g].copy_(saved[0]); self.tok[g].copy_(saved[1])
            if self.seen is not None:
                self.seen[g].copy_(saved[2])
            torch.cuda.synchronize(self.dev)
            self.graphs[g] = gr
        return gr

    def capture(self):
        for g in range(self.groups):
            self._graph(g)

    # ------------------------------------------------------------------ prefill / decode drivers
    def prefill(self, prompts: torch.Tensor):
        """prompts [groups * gb, P] int64 on the device (equal lengths).  Pipeline: group by group through the ranks."""
        P = prompts.shape[1]
        c = self.cfg
        with torch.cuda.stream(self.stream):
            pos = torch.arange(P, device=self.dev)[None, :].expand(self.gb, P)
            for g in range(self.groups):
                ids = prompts[g * self.gb:(g + 1) * self.gb]
                if self.first:
                    x = self._embed(ids)
                else:
                    x = torch.empty((self.gb, P, c.hidden_size), device=self.dev, dtype=torch.bfloat16)
                    dist.recv(x, src=self.rank - 1); self.nccl_calls += 1
                y = self._layers(x, pos, g, P)
                if self.last:
                    self.seen[g].zero_()
                    self.seen[g].scatter_(1, ids, True)
                    self.tok[g].copy_(self._sample(y[:, -1], g))
                else:
                    dist.send(y.contiguous(), dst=self.rank + 1); self.nccl_calls += 1
                self.pos[g].fill_(P)
                self._return_tokens([g])

    def _return_tokens(self, gs):
        """sampled tokens of the listed groups: last piece -> piece 0 over the second communicator on a side stream.
        Piece 0 only POSTS the receive here; it waits for a group's tokens right before it embeds them
        (``_await_tokens``), so the wavefront is not serialised on the return path."""
        if self.world == 1:
            return
        ev = torch.cuda.Event(); ev.record(self.stream)
        if self.last:
            with torch.cuda.stream(self.side):
                self.side.wait_event(ev)
                for g in gs:
                    dist.send(self.tok[g], dst=0, group=self.tok_group); self.nccl_calls += 1
        elif self.first:
            with torch.cuda.stream(self.side):
                self.side.wait_event(ev)              # the stage that read tok[g] has been enqueued before this
                for g in gs:
                    dist.recv(self.tok[g], src=self.world - 1, group=self.tok_group); self.nccl_calls += 1
                    e = torch.cuda.Event(); e.record(self.side)
                    self._tok_ev[g] = e

    def _await_tokens(self, g):
        e = self._tok_ev.pop(g, None)
        if e is not None:
            self.stream.wait_event(e)

    def decode(self, n_steps: int):
        with torch.cuda.stream(self.stream):
            for _ in range(n_steps):
                for g in range(self.groups):
                    if self.first:
                        self._await_tokens(g)
                    else:
                        dist.recv(self.h_in[g], src=self.rank - 1); self.nccl_calls += 1
                    gr = self._graph(g)
                    if gr is not None:
                        gr.replay(); self.kernel_graphs += 1
                    else:
                        self._stage_decode(g)
                    if not self.last:
                        dist.send(self.h_out[g], dst=self.rank + 1); self.nccl_calls += 1
                    self._return_tokens([g])

    def finish(self):
        """order the main stream behind every outstanding token receive (piece 0) / send (last piece)"""
        with torch.cuda.stream(self.stream):
            for g in list(self._tok_ev):
                self._await_tokens(g)
            ev = torch.cuda.Event(); ev.record(self.side)
            self.stream.wait_event(ev)

    def tokens(self) -> torch.Tensor:
        """[groups * gb] newest sampled ids (valid on rank 0 and on the last rank)"""
        return self.tok.reshape(-1)
