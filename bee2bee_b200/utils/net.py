"""Address discovery (parity: the reference's bee2bee/utils.py:68-98).  On the H100 box the
mesh is node-local, so WAN probing is skipped whenever ``BEE2BEE_OFFLINE`` is set."""
from __future__ import annotations

import os
import socket
import sys
from typing import Optional


def offline() -> bool:
    return os.environ.get("BEE2BEE_OFFLINE", "").lower() in ("1", "true", "yes")


def get_lan_ip() -> str:
    with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s:
        try:
            s.connect(("10.255.255.255", 1))      # no packet is sent for UDP connect
            return s.getsockname()[0]
        except OSError:
            return "127.0.0.1"


def get_public_ip(timeout: float = 3.0) -> Optional[str]:
    if offline():
        return None
    import urllib.request

    try:
        with urllib.request.urlopen("https://api.ipify.org", timeout=timeout) as r:
            return r.read().decode("utf8").strip() or None
    except Exception:
        return None


def is_colab() -> bool:
    return "google.colab" in sys.modules
