"""bee2bee_b200 -- Hopper (H100) peer-mesh inference engine with the Bee2Bee surface.

Public exports mirror the reference package (/root/reference/bee2bee/__init__.py:1-11):
``P2PNode``, ``run_p2p_node``, ``api_server`` (the FastAPI module) and ``__version__``.
Heavy sub-modules are imported lazily so ``import bee2bee_b200`` stays cheap."""
from __future__ import annotations

__version__ = "0.1.0"
REFERENCE_VERSION = "3.7.1"      # surface parity target (pyproject of the reference)

__all__ = ["P2PNode", "run_p2p_node", "api_server", "Engine", "SamplingParams", "__version__"]


def __getattr__(name):
    if name in ("P2PNode", "run_p2p_node"):
        from . import p2p_runtime

        return getattr(p2p_runtime, name)
    if name == "api_server":
        from . import api

        return api
    if name in ("Engine", "SamplingParams"):
        from .engine import core

        return getattr(core, name)
    raise AttributeError(name)
