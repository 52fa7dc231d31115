"""NAT traversal (parity: /root/reference/bee2bee/nat.py:19-609): UPnP -> NAT-PMP -> PCP ->
STUN, public-IP discovery with a 5-minute cache, status/manual-instruction helpers and the
legacy wrappers (``try_upnp_map``, ``try_stun``, ``auto_port_forward``, ``get_public_ip``).

On the H100 box peers are GPUs of one host: reachability is a CUDA peer-access question
answered by ``parallel.mesh``; this module exists so WAN deployments keep working and is
completely inert when ``BEE2BEE_OFFLINE`` is set (no sockets are opened)."""
from __future__ import annotations

import asyncio
import ipaddress
import socket
import struct
import time
from typing import Dict, List, Optional, Tuple

from .stun_client import STUNClient
from .utils import get_lan_ip, offline

PUBLIC_IP_SERVICES = ("https://api.ipify.org", "https://ifconfig.me/ip", "https://icanhazip.com",
                      "https://checkip.amazonaws.com", "https://ipinfo.io/ip", "https://ident.me")


class PortForwardingResult:
    def __init__(self, success: bool, method: str = "none", external_ip: Optional[str] = None,
                 external_port: Optional[int] = None, details: str = "", needs_manual: bool = False,
                 fallback_used: bool = False):
        self.success, self.method = success, method
        self.external_ip, self.external_port = external_ip, external_port
        self.details, self.needs_manual, self.fallback_used = details, needs_manual, fallback_used

    def __bool__(self) -> bool:
        return self.success

    def __str__(self) -> str:
        if self.success:
            return f"{self.method}: {self.external_ip}:{self.external_port}"
        return f"{self.method}: Failed - {self.details}"


class PortForwarder:
    def __init__(self):
        self.forwarded_ports: Dict[int, PortForwardingResult] = {}
        self.public_ip_cache: Optional[str] = None
        self.public_ip_cache_time = 0.0

    # ----------------------------------------------------------------- orchestration
    async def auto_forward_port(self, port: int, protocol: str = "TCP",
                                description: str = "Bee2Bee P2P") -> PortForwardingResult:
        if offline():
            res = PortForwardingResult(False, "offline", details="BEE2BEE_OFFLINE set; mesh is node-local")
            self.forwarded_ports[port] = res
            return res
        loop = asyncio.get_running_loop()
        attempts: List[PortForwardingResult] = []
        for name, fn in (("UPnP", self._try_upnp), ("NAT-PMP", self._try_natpmp), ("PCP", self._try_pcp)):
            try:
                res = await asyncio.wait_for(loop.run_in_executor(None, fn, port, protocol, description), timeout=6)
            except Exception as exc:
                res = PortForwardingResult(False, name, details=str(exc))
            attempts.append(res)
            if res.success:
                self.forwarded_ports[port] = res
                return res
        res = await self._try_stun_detection(port, protocol, description)
        if not res.success:
            res.needs_manual = True
            res.details = "; ".join(f"{a.method}: {a.details}" for a in attempts + [res])
        self.forwarded_ports[port] = res
        return res

    # ----------------------------------------------------------------------- methods
    def _try_upnp(self, port: int, protocol: str, description: str) -> PortForwardingResult:
        try:
            import miniupnpc  # type: ignore
        except Exception:
            return PortForwardingResult(False, "UPnP", details="miniupnpc not installed")
        try:
            u = miniupnpc.UPnP()
            u.discoverdelay = 200
            if u.discover() == 0:
                return PortForwardingResult(False, "UPnP", details="no IGD found")
            u.selectigd()
            ok = u.addportmapping(port, protocol, u.lanaddr, port, description, "")
            if ok:
                return PortForwardingResult(True, "UPnP", u.externalipaddress(), port, "mapped")
            return PortForwardingResult(False, "UPnP", details="addportmapping refused")
        except Exception as exc:
            return PortForwardingResult(False, "UPnP", details=str(exc))

    def _try_natpmp(self, port: int, protocol: str, description: str) -> PortForwardingResult:
        """RFC 6886 over a raw UDP socket (no third-party package needed)."""
        gw = self._get_gateway_ip()
        if not gw:
            return PortForwardingResult(False, "NAT-PMP", details="no gateway")
        try:
            with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s:
                s.settimeout(1.0)
                s.sendto(struct.pack("!BB", 0, 0), (gw, 5351))                 # external address request
                data, _ = s.recvfrom(64)
                if len(data) < 12 or struct.unpack("!H", data[2:4])[0] != 0:
                    return PortForwardingResult(False, "NAT-PMP", details="address request refused")
                ext_ip = socket.inet_ntoa(data[8:12])
                op = 2 if protocol.upper() == "TCP" else 1
                s.sendto(struct.pack("!BBHHHI", 0, op, 0, port, port, 3600), (gw, 5351))
                data, _ = s.recvfrom(64)
                if len(data) >= 16 and struct.unpack("!H", data[2:4])[0] == 0:
                    return PortForwardingResult(True, "NAT-PMP", ext_ip, struct.unpack("!H", data[10:12])[0], "mapped")
                return PortForwardingResult(False, "NAT-PMP", details="mapping refused")
        except Exception as exc:
            return PortForwardingResult(False, "NAT-PMP", details=str(exc))

    def _try_pcp(self, port: int, protocol: str, description: str) -> PortForwardingResult:
        """RFC 6887 MAP request."""
        gw = self._get_gateway_ip()
        if not gw:
            return PortForwardingResult(False, "PCP", details="no gateway")
        try:
            local = ipaddress.IPv4Address(self._get_local_ip())
            mapped_local = b"\x00" * 10 + b"\xff\xff" + local.packed
            proto = 6 if protocol.upper() == "TCP" else 17
            req = struct.pack("!BBHI", 2, 1, 0, 3600) + mapped_local
            req += b"\x00" * 12 + struct.pack("!B3xHH", proto, port, port) + b"\x00" * 16
            with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s:
                s.settimeout(1.0)
                s.sendto(req, (gw, 5351))
                data, _ = s.recvfrom(1100)
            if len(data) >= 60 and data[0] == 2 and data[3] == 0:
                ext_port = struct.unpack("!H", data[42:44])[0]
                ext_ip = str(ipaddress.IPv6Address(data[44:60]).ipv4_mapped or "")
                return PortForwardingResult(True, "PCP", ext_ip or None, ext_port, "mapped")
            return PortForwardingResult(False, "PCP", details="MAP refused")
        except Exception as exc:
            return PortForwardingResult(False, "PCP", details=str(exc))

    async def _try_stun_detection(self, port: int, protocol: str, description: str) -> PortForwardingResult:
        info = await STUNClient().get_public_info()
        if info:
            return PortForwardingResult(True, "STUN", info["ip"], info["port"], "public mapping discovered (no port "
                                        "was opened; works for cone NATs)", fallback_used=True)
        return PortForwardingResult(False, "STUN", details="no STUN server answered")

    async def _simple_stun_request(self, server: str, server_port: int, local_port: int) -> Optional[str]:
        res = await STUNClient(local_port=local_port).query_server(server, server_port)
        return res["ip"] if res else None

    # --------------------------------------------------------------------- utilities
    async def get_public_ip(self) -> Optional[str]:
        if offline():
            return None
        if self.public_ip_cache and time.time() - self.public_ip_cache_time < 300:
            return self.public_ip_cache
        import urllib.request

        def fetch(url: str) -> Optional[str]:
            try:
                with urllib.request.urlopen(url, timeout=3) as r:
                    ip = r.read().decode().strip()
                return ip if self._is_valid_ip(ip) else None
            except Exception:
                return None

        loop = asyncio.get_running_loop()
        for url in PUBLIC_IP_SERVICES:
            ip = await loop.run_in_executor(None, fetch, url)
            if ip:
                self.public_ip_cache, self.public_ip_cache_time = ip, time.time()
                return ip
        return None

    def _get_local_ip(self) -> str:
        return get_lan_ip()

    def _get_gateway_ip(self) -> Optional[str]:
        try:
            with open("/proc/net/route") as fh:
                for line in fh.readlines()[1:]:
                    f = line.split()
                    if f[1] == "00000000" and int(f[3], 16) & 2:
                        return socket.inet_ntoa(struct.pack("<L", int(f[2], 16)))
        except Exception:
            pass
        parts = self._get_local_ip().split(".")
        return ".".join(parts[:3] + ["1"]) if len(parts) == 4 else None

    def _is_valid_ip(self, ip: str) -> bool:
        try:
            ipaddress.ip_address(ip)
            return True
        except ValueError:
            return False

    def get_status_table(self):
        from rich.table import Table

        t = Table(title="Port forwarding")
        for col in ("Port", "Method", "External", "Status"):
            t.add_column(col)
        for port, res in self.forwarded_ports.items():
            t.add_row(str(port), res.method, f"{res.external_ip}:{res.external_port}" if res.success else "-",
                      "ok" if res.success else f"failed ({res.details[:40]})")
        return t

    def get_manual_instructions(self, port: int, protocol: str = "TCP"):
        from rich.panel import Panel

        return Panel(f"1. Open your router admin page (usually http://{self._get_gateway_ip()})\n"
                     f"2. Add a port-forward rule: external {protocol} {port} -> {self._get_local_ip()}:{port}\n"
                     f"3. Restart the node with --public-host <your public IP>", title="Manual port forwarding")

    async def cleanup(self) -> None:
        for port, res in list(self.forwarded_ports.items()):
            if res.success and res.method == "UPnP":
                try:
                    import miniupnpc  # type: ignore

                    u = miniupnpc.UPnP()
                    u.discover()
                    u.selectigd()
                    u.deleteportmapping(port, "TCP")
                except Exception:
                    pass
        self.forwarded_ports.clear()


_forwarder = PortForwarder()


async def try_upnp_map(port: int, proto: str = "TCP") -> Tuple[bool, Optional[str]]:
    if offline():
        return False, None
    res = await asyncio.get_running_loop().run_in_executor(None, _forwarder._try_upnp, port, proto, "Bee2Bee P2P")
    return res.success, res.external_ip


async def try_stun() -> Optional[Tuple[str, int]]:
    info = await STUNClient().get_public_info()
    return (info["ip"], info["port"]) if info else None


async def auto_port_forward(port: int, protocol: str = "TCP") -> PortForwardingResult:
    return await _forwarder.auto_forward_port(port, protocol)


async def get_public_ip() -> Optional[str]:
    return await _forwarder.get_public_ip()
