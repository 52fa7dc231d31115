"""Pluggable control-plane transports for ``P2PNode``.

* ``ws://`` / ``wss://``  -- ``websockets`` text frames, 32 MiB cap: wire-compatible with the
  reference mesh and its JS bridge (/root/reference/bee2bee/p2p_runtime.py:174-179,350).
* ``inproc://``           -- an in-process hub (pairs of asyncio queues).  On one H100 box all
  peers live in one host, so the control plane does not need sockets at all; also what the
  multi-peer unit tests use (no ports, no NAT probing).

The token path never touches a transport: activations move GPU->GPU through
``parallel.mesh`` (peer stores + flags).
"""
from __future__ import annotations

import asyncio
from typing import AsyncIterator, Awaitable, Callable, Dict, Optional

MAX_FRAME = 32 * 1024 * 1024


class ConnectionClosed(Exception):
    pass


class Connection:
    """Duplex text-frame channel."""

    async def send(self, text: str) -> None:
        raise NotImplementedError

    async def recv(self) -> str:
        raise NotImplementedError

    async def close(self) -> None:
        raise NotImplementedError

    @property
    def closed(self) -> bool:
        raise NotImplementedError

    def __aiter__(self) -> AsyncIterator[str]:
        return self._iter()

    async def _iter(self) -> AsyncIterator[str]:
        while True:
            try:
                yield await self.recv()
            except ConnectionClosed:
                return


Handler = Callable[[Connection], Awaitable[None]]


# ----------------------------------------------------------------------------- in-process
class _QueueConn(Connection):
    _EOF = object()

    def __init__(self, rx: "asyncio.Queue", tx: "asyncio.Queue"):
        self._rx, self._tx, self._closed = rx, tx, False
        self.peer: Optional["_QueueConn"] = None

    async def send(self, text: str) -> None:
        if self._closed or (self.peer is not None and self.peer._closed):
            raise ConnectionClosed()
        if len(text) > MAX_FRAME:
            raise ValueError("frame too large")
        await self._tx.put(text)

    async def recv(self) -> str:
        if self._closed:
            raise ConnectionClosed()
        item = await self._rx.get()
        if item is self._EOF:
            self._closed = True
            raise ConnectionClosed()
        return item

    async def close(self) -> None:
        if not self._closed:
            self._closed = True
            await self._tx.put(self._EOF)      # wake the remote reader
            await self._rx.put(self._EOF)      # and our own, if any

    @property
    def closed(self) -> bool:
        return self._closed


class InProcHub:
    """Process-wide registry of listening nodes: ``inproc://<name>``."""
    _listeners: Dict[str, Handler] = {}

    @classmethod
    def listen(cls, name: str, handler: Handler) -> str:
        cls._listeners[name] = handler
        return f"inproc://{name}"

    @classmethod
    def unlisten(cls, name: str) -> None:
        cls._listeners.pop(name, None)

    @classmethod
    async def connect(cls, addr: str) -> Connection:
        name = addr.split("://", 1)[1]
        handler = cls._listeners.get(name)
        if handler is None:
            raise ConnectionRefusedError(f"no in-process listener at {addr}")
        a2b: asyncio.Queue = asyncio.Queue()
        b2a: asyncio.Queue = asyncio.Queue()
        client, server = _QueueConn(b2a, a2b), _QueueConn(a2b, b2a)
        client.peer, server.peer = server, client
        asyncio.get_running_loop().create_task(handler(server))
        return client


# ------------------------------------------------------------------------------ websockets
class _WSConn(Connection):
    def __init__(self, ws):
        self.ws = ws
        self._closed = False

    async def send(self, text: str) -> None:
        try:
            await self.ws.send(text)
        except Exception as exc:
            self._closed = True
            raise ConnectionClosed() from exc

    async def recv(self) -> str:
        try:
            data = await self.ws.recv()
        except Exception as exc:
            self._closed = True
            raise ConnectionClosed() from exc
        return data if isinstance(data, str) else data.decode("utf-8", "replace")

    async def close(self) -> None:
        self._closed = True
        try:
            await self.ws.close()
        except Exception:
            pass

    @property
    def closed(self) -> bool:
        if self._closed:
            return True
        state = getattr(self.ws, "state", None)
        return getattr(state, "name", "OPEN") not in ("OPEN", "CONNECTING")


class WSServer:
    def __init__(self, server, port: int):
        self.server, self.port = server, port

    async def close(self) -> None:
        self.server.close()
        try:
            await asyncio.wait_for(self.server.wait_closed(), timeout=2)
        except Exception:
            pass


async def ws_listen(host: str, port: int, handler: Handler) -> WSServer:
    import websockets

    async def on_conn(ws):
        await handler(_WSConn(ws))

    server = await websockets.serve(on_conn, host, port, max_size=MAX_FRAME)
    real_port = port
    for sock in getattr(server, "sockets", None) or []:
        real_port = sock.getsockname()[1]
        break
    return WSServer(server, real_port)


async def ws_connect(addr: str, timeout: float = 10.0) -> Connection:
    import websockets

    try:
        ws = await asyncio.wait_for(websockets.connect(addr, max_size=MAX_FRAME), timeout)
    except Exception:
        if addr.startswith("wss://"):          # same downgrade the reference attempts (p2p_runtime.py:353-361)
            ws = await asyncio.wait_for(websockets.connect("ws://" + addr[6:], max_size=MAX_FRAME), timeout)
        else:
            raise
    return _WSConn(ws)


async def connect(addr: str, timeout: float = 10.0) -> Connection:
    if addr.startswith("inproc://"):
        return await InProcHub.connect(addr)
    return await ws_connect(addr, timeout)
