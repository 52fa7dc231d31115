"""One *piece* (contiguous layer range) resident on one H100, executed entirely by the
hand-written sm_90a kernels in ``csrc/``.

Per decoder layer (Llama / Mistral) exactly five launches, all on one stream:

    QKV GEMM  [fused: RMSNorm(x) via folded gamma + in-kernel 1/rms, RoPE, paged-KV append]
    attention [paged KV, GQA]
    O GEMM    [fused: + residual]
    gate/up   [fused: RMSNorm, SwiGLU]
    down GEMM [fused: + residual]   <- on the last layer of a piece its epilogue stores the
                                       tiles into the NEXT piece's input buffer on the peer
                                       GPU over NVLink and publishes a release flag

and the first GEMM of the next piece acquires that flag after prefetching its weights.
Gemma-2 adds its post-norms as residual-fused RMSNorm kernels; GPT-2 uses LayerNorm +
bias/GELU epilogues.  Replaces ``build_distilbert_partial`` + the JSON hidden-state hop
of the reference (/root/reference/bee2bee/hf.py:180-205, bee2bee/node.py:249-277).
"""
from __future__ import annotations

from dataclasses import dataclass
import os
from typing import Dict, Iterable, Optional

import torch

from .. import ops
from .config import ModelConfig
from .weights import Tensors


@dataclass
class Handoff:
    """Raw device addresses of one micro-batch slot's handoff endpoints (0 = not used).

    ``in_*`` live in THIS rank's memory (written by the upstream peer); ``out_*`` are the
    downstream peer's ``in_*`` mapped through CUDA IPC / peer access.  For piece 0 the
    "input" is the sampled-token buffer written by the last piece; for the last piece the
    "output" is that token buffer on piece 0."""
    in_x: int = 0            # [max_tokens, H] bf16 staging buffer (local); piece 0: int32 token buffer
    in_h: int = 0            # [max_tokens, F] bf16 staging of the MLP hidden (local): piece starts at a down GEMM
    out_h: int = 0           # downstream in_h (peer): piece ends with a gate/up GEMM
    in_flag: int = 0         # u32: upstream publishes its epoch here (local)
    in_epoch: int = 0        # u32: number of inputs already consumed (local)
    up_ack: int = 0          # u32 on the upstream rank: its out_free for our input slot
    out_x: int = 0           # downstream staging buffer (peer); last piece: piece 0's token buffer
    out_flag: int = 0        # downstream in_flag (peer)
    out_epoch: int = 0       # u32: number of outputs already published (local)
    out_free: int = 0        # u32: downstream acks land here (local)
    done: int = 0            # u32 scratch counter (local)
    free_lag: int = 0        # payloads that may be outstanding on the output slot (1 = double-buffered staging)
    pf_flag: int = 0         # piece 0, decode: counter of prefill chunks completed by the last piece (local)
    pf_need: int = 0         # piece 0, decode: u32 word = chunks that must be complete before this group may embed
    # mxfp8, quantisation fused ACROSS the hop: the producer's tail GEMM (O-proj / down, residual epilogue) also emits the
    # e4m3 copy of the residual stream, its UE8M0 scale-factor chunks and the per-token sum of squares straight into the
    # consumer's memory; the consumer's first GEMM (QKV / gate-up) TMA-loads them after acquiring the hop flag
    in_q: int = 0            # [max_tokens, H] e4m3 (local)
    in_sf: int = 0           # scale-factor chunks of in_q (local)
    in_ss: int = 0           # [max_tokens] fp32 sum of squares (local; zeroed by the consumer after use)
    out_q: int = 0           # downstream in_q / in_sf / in_ss (peer)
    out_sf: int = 0
    out_ss: int = 0
    # ... and for a cut between gate/up and down: the GLU epilogue stores the e4m3 MLP hidden + scale factors INSTEAD of
    # the bf16 hidden (half the bytes on the link); the consumer's down GEMM TMA-loads them
    in_qh: int = 0           # [max_tokens, F] e4m3 (local)
    in_sfh: int = 0
    out_qh: int = 0          # downstream in_qh / in_sfh (peer)
    out_sfh: int = 0


@dataclass
class BatchMeta:
    """Device-resident description of the tokens of one forward call."""
    ids: torch.Tensor          # [T] int32 (piece 0)
    positions: torch.Tensor    # [T] int32
    slots: torch.Tensor        # [T] int32 physical KV slot (-1 = do not store)
    q_start: torch.Tensor      # [S] int32
    q_len: torch.Tensor        # [S] int32
    kv_len: torch.Tensor       # [S] int32
    block_table: torch.Tensor  # [S, max_pages] int32
    n_tokens: int
    n_seqs: int
    max_q: int
    last_idx: Optional[torch.Tensor] = None   # [S] int64 row of each sequence's last token (prefill)
    splits: int = 1


class NativePiece:
    def __init__(self, cfg: ModelConfig, layers: Iterable[int], first: bool, last: bool, tensors: Tensors,
                 device: torch.device, max_tokens: int, max_seqs: int, num_pages: int, quant: str = "bf16",
                 units: Optional[tuple] = None):
        # ``units`` = (u0, u1) in THIRD-of-a-layer units: 3l = attention block of layer l (QKV GEMM, attention, O-proj),
        # 3l+1 = its gate/up GEMM, 3l+2 = its down GEMM (config.piece_units).  A piece may start at any of them (the
        # upstream piece ran the earlier ops of that layer) and end after any of them -- every GEMM can be the fused
        # tail GEMM that stores into the peer, every GEMM can be the head GEMM that acquires the flag.  A cut between
        # gate/up and down hands off TWO payloads: the MLP hidden [T, F] and the residual stream [T, H] (which the
        # O-proj epilogue of that layer dual-stores to the peer).  Default: whole layers.
        if units is not None:
            layers = range(units[0] // 3, (units[1] - 1) // 3 + 1)
            self.head_mode, self.tail_mode = units[0] % 3, (units[1] - 1) % 3
        else:
            self.head_mode, self.tail_mode = 0, 2
        self.cfg, self.layers, self.first, self.last = cfg, list(layers), first, last
        self.head_skip_attn, self.tail_skip_mlp = self.head_mode > 0, self.tail_mode < 2       # (reporting)
        if self.head_mode != 0 or self.tail_mode != 2:
            from .config import supports_half_layer_pieces
            assert supports_half_layer_pieces(cfg), "sub-layer piece boundaries need the fused RMSNorm / GLU graph"
            assert not (self.tail_mode != 2 and last), "the last piece ends with a whole layer"
            assert not (self.head_mode != 0 and first), "the first piece starts with a whole layer"
        self.device = torch.device(device)
        self.max_tokens, self.max_seqs, self.num_pages = max_tokens, max_seqs, num_pages
        self.fused_norm = cfg.norm == "rms"
        # W8A8 e4m3 (Llama / Mistral graphs).  "fp8": per-output-row weight scales x per-token activation scales
        # applied in the epilogue; "mxfp8": OCP-MX block scaling, one UE8M0 scale per 32 K elements on both
        # operands, applied by the GEMM to each 32-K partial product.
        self.fp8 = quant in ("fp8", "mxfp8") and self.fused_norm and not cfg.post_norms and cfg.glu
        self.mx = self.fp8 and quant == "mxfp8"
        self.mx_fuse = False
        self.mx_hand = False         # mxfp8: the quantised residual stream crosses the piece handoff (set with mx_fuse)
        self.wscale: Dict[str, torch.Tensor] = {}
        c = cfg
        assert c.hidden_size % 128 == 0 or c.hidden_size % 64 == 0, "hidden must be a multiple of 64"
        bf = torch.bfloat16
        dev = self.device
        t = {k: v.to(device=dev, dtype=bf) for k, v in tensors.items()}
        self.w: Dict[str, torch.Tensor] = {}
        for l in self.layers:
            p = f"l{l}."
            if not self.has_attn(l):
                self._load_mlp_only(t, p, l)
                continue
            wq, wk, wv = t[p + "wq"], t[p + "wk"], t[p + "wv"]
            if c.rope_theta > 0:
                wq = ops.rope_interleave_rows(wq, c.n_heads, c.head_dim)
                wk = ops.rope_interleave_rows(wk, c.n_kv_heads, c.head_dim)
            wqkv = torch.cat([wq, wk, wv], 0)
            if self.fused_norm:
                wqkv = ops.fold_gamma(wqkv, t[p + "ln1_w"], c.gemma_norm)
            self.w[p + "wqkv"] = wqkv.contiguous()
            self.w[p + "wo"] = t[p + "wo"].contiguous()
            if not self.has_gu(l):
                continue
            if c.glu:
                wgu = ops.glu_interleave_rows(t[p + "w_gate"], t[p + "w_up"])
                if self.fused_norm:
                    wgu = ops.fold_gamma(wgu, t[p + "ln2_w"], c.gemma_norm)
                self.w[p + "wgu"] = wgu
            else:
                self.w[p + "w_up"] = t[p + "w_up"].contiguous()
            if self.has_down(l):
                self.w[p + "w_down"] = t[p + "w_down"].contiguous()
            if not self.fused_norm:
                for n in ("ln1_w", "ln1_b", "ln2_w", "ln2_b"):
                    self.w[p + n] = t[p + n]
            if c.bias:
                self.w[p + "bqkv"] = torch.cat([t[p + "bq"], t[p + "bk"], t[p + "bv"]]).float().contiguous()
                for n in ("bo", "b_up", "b_down"):
                    self.w[p + n] = t[p + n].float().contiguous()
            if c.post_norms:
                self.w[p + "post_attn_w"] = t[p + "post_attn_w"]
                self.w[p + "post_ffn_w"] = t[p + "post_ffn_w"]
        if first:
            self.w["embed"] = t["embed"].contiguous()
            if c.rope_theta <= 0:
                self.w["pos_embed"] = t["pos_embed"].contiguous()
        if last:
            head = t["embed"] if c.tie_embeddings else t["lm_head"]
            if self.fused_norm:
                head = ops.fold_gamma(head, t["final_norm_w"], c.gemma_norm)
            else:
                self.w["final_norm_w"], self.w["final_norm_b"] = t["final_norm_w"], t["final_norm_b"]
            self.w["lm_head"] = ops.pad_rows(head, 128)
            self.vocab_pad = self.w["lm_head"].shape[0]
        del t
        if self.fp8:
            for name in list(self.w):
                if name.split(".")[-1] in ("wqkv", "wo", "wgu", "w_down") or name == "lm_head":
                    quantize = ops.quantize_weight_mxfp8 if self.mx else ops.quantize_weight_fp8
                    self.w[name], self.wscale[name] = quantize(self.w[name])
            widths = {cfg.hidden_size, cfg.q_dim, cfg.ffn_size}
            rows = max(max_tokens, max_seqs)
            self._qbuf = {k: torch.zeros((rows, k), device=self.device, dtype=torch.float8_e4m3fn) for k in widths}
            self._qscale = torch.zeros(rows, device=self.device, dtype=torch.float32)
            if self.mx:
                # activation scale-factor chunks: worst case is 32-row tiles (512 B per tile and 128 K); 127 = 2^0 for
                # rows nobody writes (0xFF would be NaN)
                tiles = (rows + 31) // 32
                self._qsf = {k: torch.full((tiles * (k // 128) * 512,), 127, device=self.device, dtype=torch.uint8)
                             for k in widths}
                # fused quantisation (B2B_MX_FUSE, default on): the O / down epilogues emit the e4m3 copy of the residual
                # stream for the next RMSNorm-fused GEMM (+ per-token sum of squares), the gate/up epilogue emits the
                # e4m3 MLP hidden for the down GEMM -- 3 of the 4 activation-quantiser launches of a layer disappear
                self.mx_fuse = os.environ.get("B2B_MX_FUSE", "1") == "1"
                # ... and ACROSS the handoff (B2B_MX_HANDOFF, default on): a tail O-proj / down GEMM emits that e4m3 copy,
                # the scale-factor chunks and the sum of squares into the downstream piece's memory together with the
                # bf16 residual stream; the downstream head GEMM consumes them (no quantiser launch at a piece head)
                self.mx_hand = self.mx_fuse and os.environ.get("B2B_MX_HANDOFF", "1") == "1"
                H, F = cfg.hidden_size, cfg.ffn_size
                self._fq_x = torch.zeros((rows, H), device=self.device, dtype=torch.float8_e4m3fn)
                self._fq_h = torch.zeros((rows, F), device=self.device, dtype=torch.float8_e4m3fn)
                self._fq_sf_x = torch.full((tiles * (H // 128) * 512,), 127, device=self.device, dtype=torch.uint8)
                self._fq_sf_h = torch.full((tiles * (F // 128) * 512,), 127, device=self.device, dtype=torch.uint8)
                self._sumsq1 = torch.zeros(rows, device=self.device, dtype=torch.float32)   # stream entering an attention block
                self._sumsq2 = torch.zeros(rows, device=self.device, dtype=torch.float32)   # stream entering an MLP block
                self._sumsq_head = torch.zeros(rows, device=self.device, dtype=torch.float32)  # separate-kernel quantiser (piece heads, lm_head)

        # ---- KV cache: one [pages, 64, n_kv, D] pair per layer whose attention block runs on this piece
        self.k_cache = {l: torch.zeros((num_pages, ops.PAGE, c.n_kv_heads, c.head_dim), device=dev, dtype=bf)
                        for l in self.layers if self.has_attn(l)}
        self.v_cache = {l: torch.zeros((num_pages, ops.PAGE, c.n_kv_heads, c.head_dim), device=dev, dtype=bf)
                        for l in self.layers if self.has_attn(l)}
        # ---- activations
        H = c.hidden_size
        self.xa = torch.zeros((max_tokens, H), device=dev, dtype=bf)
        self.xb = torch.zeros((max_tokens, H), device=dev, dtype=bf)
        self.q_buf = torch.zeros((max_tokens, c.q_dim), device=dev, dtype=bf)
        self.attn_buf = torch.zeros((max_tokens, c.q_dim), device=dev, dtype=bf)
        self.h_buf = torch.zeros((max_tokens, c.ffn_size), device=dev, dtype=bf)
        if not self.fused_norm or c.post_norms:
            self.n_buf = torch.zeros((max_tokens, H), device=dev, dtype=bf)
        if not self.fused_norm:
            self.qkv_buf = torch.zeros((max_tokens, c.q_dim + 2 * c.kv_dim), device=dev, dtype=bf)
        if last:
            self.last_x = torch.zeros((max_seqs, H), device=dev, dtype=bf)
            self.logits = torch.zeros((max_seqs, self.vocab_pad), device=dev, dtype=torch.float32)
        self.max_splits = 16
        g = c.n_heads // c.n_kv_heads
        rows = max(4, (g + 3) // 4 * 4)
        self.attn_ws = torch.zeros(max_seqs * c.n_kv_heads * self.max_splits * rows * (c.head_dim + 2), device=dev,
                                   dtype=torch.float32)

    # ------------------------------------------------------------------ helpers
    def has_attn(self, l: int) -> bool:
        return not (self.head_mode > 0 and l == self.layers[0])

    def has_gu(self, l: int) -> bool:
        return not (self.head_mode == 2 and l == self.layers[0]) and not (self.tail_mode == 0 and l == self.layers[-1])

    def has_down(self, l: int) -> bool:
        return not (self.tail_mode < 2 and l == self.layers[-1])

    def has_mlp(self, l: int) -> bool:
        return self.has_gu(l) and self.has_down(l)

    def n_launches(self) -> int:
        """kernel launches of one forward through the layers of this piece (fused-norm graphs; reporting)"""
        n = 0
        for l in self.layers:
            n += (3 if self.has_attn(l) else 0) + (1 if self.has_gu(l) else 0) + (1 if self.has_down(l) else 0)
        return n

    def _load_mlp_only(self, t, p: str, l: int) -> None:
        """first layer of a piece that starts inside the layer (fused-norm GLU graphs only)"""
        c = self.cfg
        if self.has_gu(l):
            wgu = ops.glu_interleave_rows(t[p + "w_gate"], t[p + "w_up"])
            self.w[p + "wgu"] = ops.fold_gamma(wgu, t[p + "ln2_w"], c.gemma_norm)
        if self.has_down(l):
            self.w[p + "w_down"] = t[p + "w_down"].contiguous()

    def _quant(self, x: torch.Tensor, with_rms: bool):
        """bf16 rows -> (e4m3 rows, activation-side gemm kwargs) in the preallocated staging buffers.
        fp8: per-token scale [x 1/rms] rides in ``rstd``; mxfp8: 1/rms is folded into the quantised values and the
        UE8M0 scale-factor chunks go to ``sfb``."""
        T, K = x.shape
        if self.mx and self.mx_fuse and with_rms:
            # same numerics as the epilogue-fused quantisation: raw values, 1/rms applied by the consuming GEMM
            ss = self._sumsq_head[:T]
            xq, sfb = ops.quant_mxfp8_rows(x, 0, self.cfg.norm_eps, out=self._qbuf[K][:T], sf_out=self._qsf[K], sumsq_out=ss)
            return xq, {"sfb": sfb, "sumsq": ss}
        if self.mx:
            xq, sfb = ops.quant_mxfp8_rows(x, 0, self.cfg.norm_eps, with_rms, out=self._qbuf[K][:T], sf_out=self._qsf[K])
            return xq, {"sfb": sfb}
        xq, xs = ops.quant_fp8_rows(x, self.cfg.norm_eps, with_rms, out=self._qbuf[K][:T], scale_out=self._qscale[:T])
        return xq, {"rstd": xs}

    def _wkw(self, name: str) -> dict:
        """weight-side gemm kwargs of a quantised weight"""
        return {"sfa": self.wscale[name]} if self.mx else {"w_scale": self.wscale[name]}

    def weight_bytes(self) -> int:
        return sum(v.numel() * v.element_size() for v in self.w.values())

    def streamed_weight_bytes(self) -> int:
        """Bytes a decode step actually streams from this piece's weights: everything except the embedding tables,
        of which a step only gathers one row per sequence (VERDICT r1: weight_bytes() overstated the roofline)."""
        skip = {"embed", "pos_embed"}
        n = sum(v.numel() * v.element_size() for k, v in self.w.items() if k not in skip)
        return n + sum(v.numel() * v.element_size() for v in self.wscale.values())

    def _use_inline_rstd(self, T: int) -> bool:
        return T <= 64

    # ------------------------------------------------------------------ forward
    def forward(self, m: BatchMeta, x_in: Optional[torch.Tensor] = None, hand: Optional[Handoff] = None,
                out_x: Optional[torch.Tensor] = None, h_in: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Runs the piece for the tokens described by ``m``.

        first piece: embeds ``m.ids``; otherwise reads ``x_in`` ([T, H], may be the peer-written
        staging buffer, guarded by ``hand.in_flag``).  Non-last piece: returns (and, with a
        handoff, peer-stores) the hidden states.  Last piece: returns fp32 logits [S, vocab_pad]."""
        c, T = self.cfg, m.n_tokens
        hand = hand or Handoff()
        eps = c.norm_eps
        if self.first:
            x = self.xa[:T]
            ops.embed(m.ids, self.w["embed"], x, pos_table=self.w.get("pos_embed"),
                      positions=m.positions if c.rope_theta <= 0 else None,
                      scale=float(torch.tensor(c.embed_scale, dtype=torch.bfloat16)) if c.embed_scale != 1.0 else 1.0,
                      tok_flag=hand.in_flag, tok_epoch=hand.in_epoch if hand.in_flag else 0,
                      pf_flag=hand.pf_flag if hand.in_flag else 0, pf_need=hand.pf_need if hand.in_flag else 0)
            wait_flag = wait_epoch = 0
        else:
            x = x_in[:T]
            wait_flag, wait_epoch = hand.in_flag, hand.in_epoch
        inline = self._use_inline_rstd(T)
        n_layers = len(self.layers)
        fuse = self.mx_fuse
        q_bn = ops.pick_bn_mx(T) if fuse else 0
        xq_ready = False       # the residual stream entering the next attention block has a fused e4m3 copy (+ sumsq1)
        # quantised payload of the hop (see Handoff.in_q): consumed by a QKV / gate-up head GEMM, produced by an
        # O-proj / down tail GEMM.  A cut between gate/up and down keeps the bf16 MLP hidden + consumer-side quantiser.
        tfp = ops.native().tensor_from_ptr if self.mx_hand else None
        H = c.hidden_size
        in_q = in_sf = in_ss = None
        if self.mx_hand and not self.first and hand.in_q and wait_flag and self.head_mode in (0, 1):
            di = self.device.index
            in_q = tfp(hand.in_q, [T, H], "u8", di).view(torch.float8_e4m3fn)
            in_sf = tfp(hand.in_sf, [((T + 31) // 32) * (H // 128) * 512], "u8", di)
            in_ss = tfp(hand.in_ss, [T], "f32", di)
        out_fq = {}
        if self.mx_hand and not self.last and hand.out_q and hand.out_x and self.tail_mode in (0, 2):
            di = self.device.index
            out_fq = dict(fq_out=tfp(hand.out_q, [T, H], "u8", di).view(torch.float8_e4m3fn),
                          fq_sf=tfp(hand.out_sf, [((T + 31) // 32) * (H // 128) * 512], "u8", di), fq_bn=q_bn,
                          sumsq_out=tfp(hand.out_ss, [T], "f32", di))
        F = c.ffn_size
        in_qh = in_sfh = None          # quantised MLP hidden of a gate/up | down cut
        if self.mx_hand and not self.first and hand.in_qh and wait_flag and self.head_mode == 2:
            di = self.device.index
            in_qh = tfp(hand.in_qh, [T, F], "u8", di).view(torch.float8_e4m3fn)
            in_sfh = tfp(hand.in_sfh, [((T + 31) // 32) * (F // 128) * 512], "u8", di)
        out_fqh = {}
        if self.mx_hand and not self.last and hand.out_qh and hand.out_x and self.tail_mode == 1:
            di = self.device.index
            out_fqh = dict(fq_out=tfp(hand.out_qh, [T, F], "u8", di).view(torch.float8_e4m3fn),
                           fq_sf=tfp(hand.out_sfh, [((T + 31) // 32) * (F // 128) * 512], "u8", di), fq_bn=q_bn, no_out=True)
        for li, l in enumerate(self.layers):
            p = f"l{l}."
            do_attn, do_gu, do_down = self.has_attn(l), self.has_gu(l), self.has_down(l)
            do_mlp = do_gu          # the piece continues past this layer's attention block
            is_tail = (li == n_layers - 1) and not self.last
            head_wait = wait_flag if li == 0 else 0           # the piece's first GEMM consumes the handoff input
            head_epoch = wait_epoch if li == 0 else 0
            x2 = self.xb[:T]
            xn = self.xa[:T]            # layer output buffer (local)
            tail_kw = {}
            if is_tail and hand.out_x:
                tail_kw = dict(out_ptr=hand.out_x, ld_out=c.hidden_size, signal_flag=hand.out_flag,
                               signal_epoch=hand.out_epoch, done_counter=hand.done, free_flag=hand.out_free,
                               bump_epoch=hand.in_epoch, ack_flag=hand.up_ack, free_lag=hand.free_lag)
            elif is_tail and out_x is not None:
                tail_kw = dict(out_ptr=out_x.data_ptr(), ld_out=c.hidden_size)
            # ---------------- attention block
            if not do_attn:
                x2 = x                  # the upstream piece ran this layer's attention: x is the post-attention stream
            elif self.fused_norm:
                if head_wait and not inline and in_q is None:
                    # wide token tiles use a separate 1/rms kernel that reads the peer-written rows:
                    # acquire the handoff flag first (the GEMM's own wait then passes immediately)
                    ops.native().flag_wait(head_wait, head_epoch, 1)
                qkv_kw = dict(epi=ops.EPI_QKV_ROPE, eps=eps, q_out=self.q_buf, k_cache=self.k_cache[l],
                              v_cache=self.v_cache[l], positions=m.positions, slots=m.slots, n_q_heads=c.n_heads,
                              n_kv_heads=c.n_kv_heads, head_dim=c.head_dim, rope_theta=c.rope_theta,
                              q_scale=c.softmax_scale)
                if self.fp8 and xq_ready:
                    # e4m3 copy + scale factors + sum of squares were produced by the previous layer's down epilogue
                    ops.gemm(self.w[p + "wqkv"], self._fq_x[:T], sfb=self._fq_sf_x, sumsq=self._sumsq1,
                             **self._wkw(p + "wqkv"), **qkv_kw)
                    xq_ready = False
                elif self.fp8 and head_wait and in_q is not None:
                    # piece head: the upstream tail GEMM stored the e4m3 copy, scale factors and sum of squares here; the
                    # GEMM acquires the hop flag itself (weights stream while it waits)
                    ops.gemm(self.w[p + "wqkv"], in_q, sfb=in_sf, sumsq=in_ss, wait_flag=head_wait, wait_epoch=head_epoch,
                             **self._wkw(p + "wqkv"), **qkv_kw)
                elif self.fp8:
                    if head_wait and inline:
                        ops.native().flag_wait(head_wait, head_epoch, 1)     # the quant kernel reads x first
                    xq, akw = self._quant(x, with_rms=True)
                    ops.gemm(self.w[p + "wqkv"], xq, **akw, **self._wkw(p + "wqkv"), **qkv_kw)
                else:
                    r = None if inline else ops.rstd(x, eps)
                    ops.gemm(self.w[p + "wqkv"], x, rstd=r, norm_from_x=inline, wait_flag=head_wait,
                             wait_epoch=head_epoch, **qkv_kw)
            else:
                if head_wait:
                    ops.native().flag_wait(head_wait, head_epoch, 1)
                n = ops.layernorm(x, self.w[p + "ln1_w"], self.w[p + "ln1_b"], self.n_buf[:T], eps)
                ops.gemm(self.w[p + "wqkv"], n, out=self.qkv_buf[:T], epi=ops.EPI_PLAIN, bias=self.w.get(p + "bqkv"))
                ops.kv_append(self.qkv_buf[:T], self.q_buf, self.k_cache[l], self.v_cache[l], m.slots, c.q_dim,
                              c.kv_dim, c.softmax_scale)
            if do_attn:
                # mxfp8: the attention kernel emits the e4m3 copy of its output for the O-proj itself (no quantiser launch)
                a_fused = fuse and not c.post_norms and ops.attention_fuses_quant(m.max_q, c.n_heads, c.n_kv_heads, c.head_dim,
                                                                                 m.splits)
                aq_kw = dict(fq_out=self._qbuf[c.q_dim][:T], fq_sf=self._qsf[c.q_dim], fq_bn=q_bn) if a_fused else {}
                ops.attention(self.q_buf, self.k_cache[l], self.v_cache[l], self.attn_buf, m.block_table, m.q_start,
                              m.q_len, m.kv_len, max_q=m.max_q, n_q=c.n_heads, n_kv=c.n_kv_heads, head_dim=c.head_dim,
                              window=c.layer_window(l), softcap=c.attn_softcap, splits=m.splits, ws=self.attn_ws, **aq_kw)
                a = self.attn_buf[:T]
                okw = {} if do_mlp else tail_kw          # piece ends after this attention block: O-proj is the tail GEMM
                o_out = None if okw else x2
                if is_tail and do_gu and not do_down and hand.out_x:
                    # the piece ends with this layer's gate/up GEMM: the next piece's down GEMM needs the residual stream
                    # too -> the O-proj epilogue stores x2 locally AND into the peer's staging slot (flow-controlled like
                    # the tail GEMM's own payload; the tail GEMM's release flag publishes both)
                    okw = dict(out2_ptr=hand.out_x, free_flag=hand.out_free, signal_epoch=hand.out_epoch,
                               free_lag=hand.free_lag)
                    o_out = x2
                if c.post_norms:
                    o = ops.gemm(self.w[p + "wo"], a, out=self.n_buf[:T], epi=ops.EPI_PLAIN)
                    ops.rmsnorm(o, self.w[p + "post_attn_w"], out=x2, residual=x, eps=eps, plus_one=c.gemma_norm)
                elif self.fp8:
                    if a_fused:
                        aq, akw = self._qbuf[c.q_dim][:T], dict(sfb=self._qsf[c.q_dim])
                    else:
                        aq, akw = self._quant(a, with_rms=False)
                    x2_fused = fuse and do_gu and do_down          # this layer's gate/up and down run here
                    fq = {}
                    if fuse:
                        # (layer 0 of a piece fed by a quantised hop: its QKV read the hop's sum of squares, not sumsq1)
                        fq = dict(zero_buf=in_ss if (li == 0 and in_ss is not None) else self._sumsq1)
                        if x2_fused:
                            fq.update(fq_out=self._fq_x[:T], fq_sf=self._fq_sf_x, fq_bn=q_bn, sumsq_out=self._sumsq2)
                        elif okw is tail_kw and tail_kw and out_fq:
                            fq.update(out_fq)            # tail O-proj: quantised copy for the next piece's gate/up GEMM
                    ops.gemm(self.w[p + "wo"], aq, out=o_out, epi=ops.EPI_RESIDUAL, residual=x, **akw,
                             **self._wkw(p + "wo"), **okw, **fq)
                else:
                    ops.gemm(self.w[p + "wo"], a, out=o_out, epi=ops.EPI_RESIDUAL, residual=x, bias=self.w.get(p + "bo"),
                             **okw)
                if not do_mlp:
                    x = out_x[:T] if (okw and out_x is not None and not hand.out_x) else x2
                    continue
            # ---------------- MLP block
            mlp_wait = head_wait if not do_attn else 0      # piece starts inside this layer: its first GEMM consumes the input
            mlp_epoch = head_epoch if not do_attn else 0
            mlp_q_head = bool(mlp_wait) and do_gu and in_q is not None     # gate/up head GEMM fed by a quantised hop
            down_q_head = bool(mlp_wait) and not do_gu and in_qh is not None   # down head GEMM fed by a quantised hop
            if mlp_wait and (self.fp8 or not inline) and not (mlp_q_head or down_q_head):
                ops.native().flag_wait(mlp_wait, mlp_epoch, 1)   # a separate quant / 1/rms kernel reads the input first
            gu_tail = tail_kw if (do_gu and not do_down) else {}   # piece ends after gate/up: it is the tail GEMM
            if gu_tail and hand.out_h:
                gu_tail = dict(gu_tail, out_ptr=hand.out_h, ld_out=c.ffn_size)
            h_fused = False
            if not do_gu:
                hmid = h_in[:T]                              # the upstream piece ran gate/up: staged MLP hidden
            elif c.glu and self.fp8:
                h_fused = fuse and do_down and not gu_tail   # the down GEMM of this layer consumes the e4m3 hidden directly
                hq_kw = dict(fq_out=self._fq_h[:T], fq_sf=self._fq_sf_h, fq_bn=q_bn, no_out=True) if h_fused else {}
                if gu_tail and out_fqh:
                    hq_kw = out_fqh          # tail gate/up GEMM: e4m3 hidden + scale factors into the peer, no bf16 copy
                if fuse and do_attn and do_down and not c.post_norms:
                    # x2 was quantised by the O-proj epilogue of this layer (sum of squares in sumsq2)
                    x2q, akw = self._fq_x[:T], dict(sfb=self._fq_sf_x, sumsq=self._sumsq2)
                elif mlp_q_head:
                    x2q, akw = in_q, dict(sfb=in_sf, sumsq=in_ss, wait_flag=mlp_wait, wait_epoch=mlp_epoch)
                else:
                    x2q, akw = self._quant(x2, with_rms=True)
                hmid = ops.gemm(self.w[p + "wgu"], x2q, out=None if (gu_tail or h_fused) else self.h_buf[:T], epi=ops.EPI_GLU,
                                eps=eps, **akw, **self._wkw(p + "wgu"), act_gelu=(c.act == "gelu_tanh"), **gu_tail, **hq_kw)
            elif c.glu:
                r2 = None
                if self.fused_norm and not inline:
                    r2 = ops.rstd(x2, eps)
                hmid = ops.gemm(self.w[p + "wgu"], x2, out=None if gu_tail else self.h_buf[:T], epi=ops.EPI_GLU, rstd=r2,
                                norm_from_x=inline and self.fused_norm, eps=eps, act_gelu=(c.act == "gelu_tanh"),
                                wait_flag=mlp_wait, wait_epoch=mlp_epoch, **gu_tail)
            else:
                n2 = ops.layernorm(x2, self.w[p + "ln2_w"], self.w[p + "ln2_b"], self.n_buf[:T], eps)
                hmid = ops.gemm(self.w[p + "w_up"], n2, out=self.h_buf[:T], epi=ops.EPI_GELU, bias=self.w.get(p + "b_up"))
            if not do_down:
                x = x2                   # (not read again: the piece ends here)
                continue
            down_wait = mlp_wait if not do_gu else 0         # piece starts at this down GEMM
            down_epoch = mlp_epoch if not do_gu else 0
            if c.post_norms:
                d = ops.gemm(self.w[p + "w_down"], hmid, out=self.n_buf[:T], epi=ops.EPI_PLAIN)
                if is_tail and hand.out_x:
                    dst = ops.native().tensor_from_ptr(hand.out_x, [T, c.hidden_size], "bf16", self.device.index)
                    if hand.out_free:
                        ops.native().flag_wait(hand.out_free, hand.out_epoch, -hand.free_lag)    # back-pressure
                    ops.rmsnorm(d, self.w[p + "post_ffn_w"], out=dst, residual=x2, eps=eps, plus_one=c.gemma_norm)
                    ops.native().flag_signal(hand.out_flag, hand.out_epoch, hand.in_epoch, hand.up_ack)
                    xn = dst
                else:
                    tgt = out_x[:T] if (is_tail and out_x is not None) else xn
                    ops.rmsnorm(d, self.w[p + "post_ffn_w"], out=tgt, residual=x2, eps=eps, plus_one=c.gemma_norm)
                    xn = tgt
            else:
                if not do_attn and xn.data_ptr() == x2.data_ptr():
                    xn = self.xb[:T]    # x2 aliases the input buffer here: keep the residual source intact
                if self.fp8:
                    if h_fused:
                        hq, akw = self._fq_h[:T], dict(sfb=self._fq_sf_h)
                    elif down_q_head:
                        hq, akw = in_qh, dict(sfb=in_sfh, wait_flag=down_wait, wait_epoch=down_epoch)
                    else:
                        hq, akw = self._quant(hmid, with_rms=False)
                    fq = {}
                    if fuse:
                        fq = dict(zero_buf=in_ss if (li == 0 and mlp_q_head) else self._sumsq2)
                        if tail_kw and out_fq:
                            fq.update(out_fq)            # tail down GEMM: quantised copy for the next piece's QKV GEMM
                        if li + 1 < n_layers and not tail_kw:
                            # the next layer's QKV GEMM (on this piece) reads the e4m3 copy; its RMSNorm uses sumsq1
                            fq.update(fq_out=self._fq_x[:T], fq_sf=self._fq_sf_x, fq_bn=q_bn, sumsq_out=self._sumsq1)
                            xq_ready = True
                    ops.gemm(self.w[p + "w_down"], hq, out=None if tail_kw else xn, epi=ops.EPI_RESIDUAL,
                             residual=x2, **akw, **self._wkw(p + "w_down"), **tail_kw, **fq)
                else:
                    ops.gemm(self.w[p + "w_down"], hmid, out=None if tail_kw else xn, epi=ops.EPI_RESIDUAL,
                             residual=x2, bias=self.w.get(p + "b_down"), wait_flag=down_wait, wait_epoch=down_epoch,
                             **tail_kw)
                if tail_kw and out_x is not None and not hand.out_x:
                    xn = out_x[:T]
            x = xn
        if not self.last:
            return x
        # ---------------- head: last-token gather, final norm fused into the lm_head GEMM
        S = m.n_seqs
        if m.last_idx is not None:
            torch.index_select(x, 0, m.last_idx, out=self.last_x[:S])
            xl = self.last_x[:S]
        else:
            xl = x[:S]
        if not self.first and hand.in_flag:
            # the head GEMM of this piece consumed the input slot; release it to the upstream piece
            ops.native().flag_signal(0, 0, hand.in_epoch, hand.up_ack)
        if self.fused_norm and self.fp8 and "lm_head" in self.wscale:
            lq, akw = self._quant(xl, with_rms=True)
            ops.gemm(self.w["lm_head"], lq, out=self.logits[:S], epi=ops.EPI_PLAIN, eps=eps, **akw, **self._wkw("lm_head"),
                     out_fp32=True)
        elif self.fused_norm:
            ops.gemm(self.w["lm_head"], xl, out=self.logits[:S], epi=ops.EPI_PLAIN, norm_from_x=True, eps=eps,
                     out_fp32=True, bn=ops.pick_bn(S))
        else:
            n = ops.layernorm(xl, self.w["final_norm_w"], self.w["final_norm_b"], self.n_buf[:S], eps)
            ops.gemm(self.w["lm_head"], n, out=self.logits[:S], epi=ops.EPI_PLAIN, out_fp32=True)
        return self.logits[:S]
