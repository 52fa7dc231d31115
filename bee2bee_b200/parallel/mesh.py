"""NVLink mesh: the in-process replacement for the reference's WAN discovery and transport.

``peer = one H100 hosting one piece``.  What the reference does with bootstrap links,
hello/peer_list gossip, DHT lookups, STUN/UPnP and one WebSocket per peer pair
(/root/reference/bee2bee/p2p_runtime.py:308-372,478-523; dht.py; nat.py) collapses into

  * a topology table  rank <-> cuda device <-> piece (layer range), canAccessPeer matrix,
  * symmetric staging buffers + flags whose CUDA IPC handles are exchanged ONCE through
    ``torch.distributed`` (one process per GPU) -- afterwards the token path is pure
    device-to-device: kernels store into peer-mapped memory and publish release flags,
  * ``cudaMemcpyPeerAsync`` for bulk moves (weights, KV migration).

``MeshComm`` also works for world_size == 1 (no peers, no flags).
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from .. import ops
from ..models.native import Handoff

FLAG_WORDS = 16          # u32 slots per channel (64 B, one line per channel)
F_IN_FLAG, F_IN_EPOCH, F_OUT_EPOCH, F_OUT_FREE, F_DONE, F_TOK_DONE = 0, 1, 2, 3, 4, 5
# misc channel (index groups + 1): prefill completion, published by the last rank on rank 0
M_PF_FLAG, M_PF_EPOCH, M_PF_SEEN = 0, 1, 2
M_PF_NEED0 = 4           # misc words 4.. : per micro-batch group, chunks that must be complete before the group may decode (<= 12 groups per line; more groups spill into a dedicated buffer)


@dataclass
class PeerInfo:
    rank: int
    device: int
    pid: int
    host: str
    layers: List[int] = field(default_factory=list)


class MeshComm:
    """Per-rank view of the pipeline ring rank0 -> rank1 -> ... -> rank(W-1) -> rank0 (tokens)."""

    def __init__(self, rank: int, world: int, device: torch.device, hidden: int, max_tokens: int, groups: int,
                 group_batch: int, hist_len: int, control_group=None, ffn: int = 0, mx: bool = False):
        # ffn > 0: some piece boundary lies between a gate/up and a down GEMM -> the hop also carries the MLP hidden
        # mx: block-scaled fp8 pieces -> the hop also carries the e4m3 copy of the residual stream, its scale-factor
        #     chunks and the per-token sum of squares (quantisation fused across the handoff)
        self.mx = mx
        self.rank, self.world, self.device = rank, world, torch.device(device)
        self.hidden, self.max_tokens, self.groups, self.group_batch, self.hist_len = hidden, max_tokens, groups, group_batch, hist_len
        self.control_group = control_group
        self.ffn = ffn
        self.next_rank = (rank + 1) % world
        self.prev_rank = (rank - 1) % world
        self.peers: Dict[int, PeerInfo] = {}
        self._opened: List[int] = []
        self.C = ops.native() if self.device.type == "cuda" else None
        self.local: Dict[str, int] = {}
        self.remote_next: Dict[str, int] = {}
        self.remote_prev: Dict[str, int] = {}
        self.remote_first: Dict[str, int] = {}
        if world > 1:
            self._alloc_and_exchange()

    # ------------------------------------------------------------------ set-up
    def _sf_bytes(self, rows: int, width: int = 0) -> int:
        """scale-factor chunks of ``rows`` tokens x ``width`` (default hidden) -- worst case: 32-row token tiles,
        512 B per tile and 128 K"""
        return ((rows + 31) // 32) * ((width or self.hidden) // 128) * 512

    def _sizes(self) -> Dict[str, int]:
        mxs = {}
        if self.mx:
            mxs = {
                "stage_q": self.groups * self.group_batch * self.hidden,
                "stage_q_pf": 2 * self.max_tokens * self.hidden,
                "stage_sf": self.groups * self._sf_bytes(self.group_batch),
                "stage_sf_pf": 2 * self._sf_bytes(self.max_tokens),
                "stage_ss": self.groups * self.group_batch * 4,
                "stage_ss_pf": 2 * self.max_tokens * 4,
            }
            if self.ffn:
                mxs.update({
                    "stage_qh": self.groups * self.group_batch * self.ffn,
                    "stage_qh_pf": 2 * self.max_tokens * self.ffn,
                    "stage_sfh": self.groups * self._sf_bytes(self.group_batch, self.ffn),
                    "stage_sfh_pf": 2 * self._sf_bytes(self.max_tokens, self.ffn),
                })
        return {
            **mxs,
            "stage": self.groups * self.group_batch * self.hidden * 2,          # decode: one bf16 slot per group
            "stage_pf": 2 * self.max_tokens * self.hidden * 2,                  # prefill chunks: double-buffered
            "stage_h": self.groups * self.group_batch * self.ffn * 2,           # MLP hidden of a gate/up | down cut
            "stage_h_pf": 2 * self.max_tokens * self.ffn * 2,
            "flags": (self.groups + 2) * FLAG_WORDS * 4,                        # groups, prefill channel, misc
            "pf_need": max(64, self.groups * 4),                                # rank 0: chunks each group waits for
            "tok": self.groups * self.group_batch * 4,                          # sampled-token return buffer (rank 0)
            "hist": self.groups * self.group_batch * self.hist_len * 4,         # token history ring (rank 0)
        }

    def _alloc_and_exchange(self) -> None:
        import torch.distributed as dist

        C = self.C
        handles = {}
        for name, nbytes in self._sizes().items():
            p = C.peer_alloc(max(256, nbytes))
            self.local[name] = p
            handles[name] = C.ipc_export(p)
        info = {"rank": self.rank, "device": self.device.index, "pid": os.getpid(), "host": os.uname().nodename,
                "handles": handles}
        gathered: List[Optional[dict]] = [None] * self.world
        dist.all_gather_object(gathered, info, group=self.control_group)
        for g in gathered:
            self.peers[g["rank"]] = PeerInfo(g["rank"], g["device"], g["pid"], g["host"])

        def open_all(rank: int) -> Dict[str, int]:
            if rank == self.rank:
                return dict(self.local)
            out = {}
            for name, h in gathered[rank]["handles"].items():
                p = C.ipc_import(h)
                self._opened.append(p)
                out[name] = p
            return out

        self.remote_next = open_all(self.next_rank)
        self.remote_prev = open_all(self.prev_rank) if self.prev_rank != self.next_rank else self.remote_next
        self.remote_first = self.remote_next if self.next_rank == 0 else (
            self.remote_prev if self.prev_rank == 0 else open_all(0))
        self.init_flags()

    # ------------------------------------------------------------------ endpoints
    def _flag(self, table: Dict[str, int], group: int, word: int) -> int:
        return table["flags"] + (group * FLAG_WORDS + word) * 4

    @property
    def pf_channel(self) -> int:
        return self.groups

    @property
    def misc_channel(self) -> int:
        return self.groups + 1

    def handoff(self, group: int) -> Handoff:
        """Decode endpoints of micro-batch group ``group`` on this rank (all zero for world == 1).  One staging slot
        per group and no back-pressure flags: a group's step k+1 cannot reach a piece before the token loop has
        carried step k through every piece behind it."""
        if self.world == 1:
            return Handoff()
        first, last = self.rank == 0, self.rank == self.world - 1
        stage_off = group * self.group_batch * self.hidden * 2
        tok_off = group * self.group_batch * 4
        h = Handoff()
        h.in_flag = self._flag(self.local, group, F_IN_FLAG)
        h.in_epoch = self._flag(self.local, group, F_IN_EPOCH)
        h.out_epoch = self._flag(self.local, group, F_OUT_EPOCH)
        h.done = self._flag(self.local, group, F_DONE)
        h.in_x = (self.local["tok"] + tok_off) if first else (self.local["stage"] + stage_off)
        if first:
            h.pf_flag = self._flag(self.local, self.misc_channel, M_PF_FLAG)
            h.pf_need = self.local["pf_need"] + group * 4
        h_off = group * self.group_batch * self.ffn * 2
        if self.ffn and not first:
            h.in_h = self.local["stage_h"] + h_off
        q_off, sf_off, ss_off = group * self.group_batch * self.hidden, group * self._sf_bytes(self.group_batch), tok_off
        if self.mx and not first:
            h.in_q, h.in_sf, h.in_ss = self.local["stage_q"] + q_off, self.local["stage_sf"] + sf_off, self.local["stage_ss"] + ss_off
        if self.mx and not last:
            h.out_q, h.out_sf, h.out_ss = (self.remote_next["stage_q"] + q_off, self.remote_next["stage_sf"] + sf_off,
                                           self.remote_next["stage_ss"] + ss_off)
        if self.mx and self.ffn:
            qh_off, sfh_off = group * self.group_batch * self.ffn, group * self._sf_bytes(self.group_batch, self.ffn)
            if not first:
                h.in_qh, h.in_sfh = self.local["stage_qh"] + qh_off, self.local["stage_sfh"] + sfh_off
            if not last:
                h.out_qh, h.out_sfh = self.remote_next["stage_qh"] + qh_off, self.remote_next["stage_sfh"] + sfh_off
        if last:
            h.out_x = self.remote_first["tok"] + tok_off
            h.out_flag = self._flag(self.remote_first, group, F_IN_FLAG)
        else:
            h.out_x = self.remote_next["stage"] + stage_off
            h.out_flag = self._flag(self.remote_next, group, F_IN_FLAG)
            if self.ffn:
                h.out_h = self.remote_next["stage_h"] + h_off
        return h

    def handoff_prefill(self, parity: int) -> Handoff:
        """Prefill-chunk endpoints (own channel, staging double-buffered by chunk parity).  Chunks have no loop
        dependency, so the slot is flow-controlled on the device: the producer's tail GEMM waits until the consumer
        has released payload n-2 before it stores payload n (``free_lag`` = 1), the consumer's tail GEMM (last piece:
        a flag kernel) bumps its input epoch and acks the upstream producer."""
        if self.world == 1:
            return Handoff()
        first, last = self.rank == 0, self.rank == self.world - 1
        c = self.pf_channel
        off = parity * self.max_tokens * self.hidden * 2
        h = Handoff()
        h.done = self._flag(self.local, c, F_DONE)
        h.free_lag = 1
        h_off = parity * self.max_tokens * self.ffn * 2
        q_off, sf_off, ss_off = parity * self.max_tokens * self.hidden, parity * self._sf_bytes(self.max_tokens), parity * self.max_tokens * 4
        if self.mx and not first:
            h.in_q, h.in_sf, h.in_ss = (self.local["stage_q_pf"] + q_off, self.local["stage_sf_pf"] + sf_off,
                                        self.local["stage_ss_pf"] + ss_off)
        if self.mx and not last:
            h.out_q, h.out_sf, h.out_ss = (self.remote_next["stage_q_pf"] + q_off, self.remote_next["stage_sf_pf"] + sf_off,
                                           self.remote_next["stage_ss_pf"] + ss_off)
        if self.mx and self.ffn:
            qh_off, sfh_off = parity * self.max_tokens * self.ffn, parity * self._sf_bytes(self.max_tokens, self.ffn)
            if not first:
                h.in_qh, h.in_sfh = self.local["stage_qh_pf"] + qh_off, self.local["stage_sfh_pf"] + sfh_off
            if not last:
                h.out_qh, h.out_sfh = self.remote_next["stage_qh_pf"] + qh_off, self.remote_next["stage_sfh_pf"] + sfh_off
        if not first:
            h.in_x = self.local["stage_pf"] + off
            if self.ffn:
                h.in_h = self.local["stage_h_pf"] + h_off
            h.in_flag = self._flag(self.local, c, F_IN_FLAG)
            h.in_epoch = self._flag(self.local, c, F_IN_EPOCH)
            h.up_ack = self._flag(self.remote_prev, c, F_OUT_FREE)
        if not last:
            if self.ffn:
                h.out_h = self.remote_next["stage_h_pf"] + h_off
            h.out_x = self.remote_next["stage_pf"] + off
            h.out_flag = self._flag(self.remote_next, c, F_IN_FLAG)
            h.out_epoch = self._flag(self.local, c, F_OUT_EPOCH)
            h.out_free = self._flag(self.local, c, F_OUT_FREE)
        return h

    # prefill completion: the last rank publishes "first tokens of prefill #n are in rank 0's ring"
    def pf_done_signal(self):
        """(remote flag on rank 0, local epoch) for the last rank's flag_signal after a prefill."""
        return (self._flag(self.remote_first, self.misc_channel, M_PF_FLAG),
                self._flag(self.local, self.misc_channel, M_PF_EPOCH))

    def pf_done_flag(self) -> int:
        """Address of rank 0's prefill-completion counter as seen from this rank."""
        table = self.local if self.rank == 0 else self.remote_first
        return self._flag(table, self.misc_channel, M_PF_FLAG)

    def tok_flag(self, group: int) -> int:
        """Address of rank 0's token flag of ``group`` (1 + decode steps published by the sampler) from this rank."""
        table = self.local if self.rank == 0 else self.remote_first
        return self._flag(table, group, F_IN_FLAG)

    def hist_base(self) -> int:
        """Rank 0's history ring [max_batch, hist_len] as seen from this rank."""
        return (self.local if self.rank == 0 else self.remote_first)["hist"]

    def tok_base(self) -> int:
        return (self.local if self.rank == 0 else self.remote_first)["tok"]

    def history_ptr(self, group: int) -> int:
        """Where the sampler of the last rank writes token history (rank 0's ring)."""
        table = self.remote_first if self.world > 1 else self.local
        return table["hist"] + group * self.group_batch * self.hist_len * 4

    def local_view(self, name: str, shape, dtype: str) -> torch.Tensor:
        return self.C.tensor_from_ptr(self.local[name], list(shape), dtype, self.device.index)

    def init_flags(self) -> None:
        """Once, before the first kernel: every counter is a monotonic epoch and is never reset afterwards.  Rank 0's
        token flags start at 1 ("the tokens of step 0 are there": prefill writes them) and so does the last rank's
        count of published token sets."""
        if self.world == 1:
            return
        flags = self.local_view("flags", (self.groups + 2, FLAG_WORDS), "i32")
        flags.zero_()
        if self.rank == 0:
            flags[:self.groups, F_IN_FLAG] = 1
        if self.rank == self.world - 1:
            flags[:self.groups, F_OUT_EPOCH] = 1
        if self.mx:
            sizes = self._sizes()
            for name in ("stage_q", "stage_q_pf", "stage_qh", "stage_qh_pf"):
                if name in sizes:
                    self.local_view(name, (sizes[name],), "u8").zero_()
            for name in ("stage_sf", "stage_sf_pf", "stage_sfh", "stage_sfh_pf"):
                if name in sizes:
                    self.local_view(name, (sizes[name],), "u8").fill_(127)     # 2^0 for rows nobody writes (0xFF would be NaN)
            for name in ("stage_ss", "stage_ss_pf"):
                self.local_view(name, (sizes[name] // 4,), "f32").zero_()
        torch.cuda.synchronize(self.device)
        self.barrier()

    def barrier(self) -> None:
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier(group=self.control_group)

    def topology(self) -> Dict:
        n = torch.cuda.device_count() if self.device.type == "cuda" else 0
        acc = [[bool(i == j or (self.C and self.C.can_access_peer(i, j))) for j in range(n)] for i in range(n)]
        return {"rank": self.rank, "world": self.world, "device": str(self.device), "can_access_peer": acc,
                "peers": {r: vars(p) for r, p in self.peers.items()}}

    def close(self) -> None:
        if self.C is None:
            return
        for p in self._opened:
            try:
                self.C.ipc_close(p)
            except Exception:
                pass
        self._opened.clear()
        for p in self.local.values():
            try:
                self.C.peer_free(p)
            except Exception:
                pass
        self.local.clear()
