"""Three-tier configuration: CLI flag > environment > ``$BEE2BEE_HOME/config.json`` > defaults
(parity: /root/reference/bee2bee/config.py:11-47), extended with validated engine settings
(pieces, dtype, batch, KV budget) that the reference has no notion of."""
from __future__ import annotations

import os
from typing import Any, Dict

from .utils import bee2bee_home, load_json, save_json

CONFIG_FILE = "config.json"

DEFAULT_CONFIG: Dict[str, Any] = {
    "bootstrap_url": "ws://127.0.0.1:4003",
    "p2p_port": 0,
    "api_port": 4002,
    # engine (H100) defaults
    "pieces": 1,
    "max_batch": 32,
    "max_seq_len": 4096,
    "decode_burst": 8,
}

_TYPES = {"bootstrap_url": str, "p2p_port": int, "api_port": int, "pieces": int, "max_batch": int,
          "max_seq_len": int, "decode_burst": int}


def get_config_path():
    return bee2bee_home() / CONFIG_FILE


def _validated(raw: Dict[str, Any]) -> Dict[str, Any]:
    cfg = dict(DEFAULT_CONFIG)
    for k, v in (raw or {}).items():
        want = _TYPES.get(k)
        if want is None:
            cfg[k] = v                      # unknown keys are preserved, not interpreted
        elif isinstance(v, want) and not isinstance(v, bool):
            cfg[k] = v
        else:
            try:
                cfg[k] = want(v)
            except (TypeError, ValueError):
                pass                        # keep the default for malformed values
    return cfg


def load_config() -> Dict[str, Any]:
    return _validated(load_json(get_config_path(), {}))


def save_config(config: Dict[str, Any]) -> None:
    save_json(get_config_path(), _validated(config))


def get_bootstrap_url() -> str:
    return os.getenv("BEE2BEE_BOOTSTRAP") or load_config()["bootstrap_url"]


def set_bootstrap_url(url: str) -> None:
    cfg = load_config()
    cfg["bootstrap_url"] = url
    save_config(cfg)


def get_setting(name: str, default: Any = None) -> Any:
    """``BEE2BEE_<NAME>`` env override, then config file, then ``default``."""
    env = os.getenv("BEE2BEE_" + name.upper())
    if env is not None:
        want = _TYPES.get(name, str)
        try:
            return want(env)
        except (TypeError, ValueError):
            return default
    return load_config().get(name, default)
