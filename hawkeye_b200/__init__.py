"""hawkeye_b200 — H100-native (sm_90a) high-order-pooling hot path behind Hawkeye's plugin surface.

``from hawkeye_b200.registry import MODEL`` mirrors ``model.registry.MODEL``; ``install_into`` overrides the
reference's own registry entries.  All compute goes through ``libhawkeye_b200.so`` (no fallback).
"""
from . import _lib  # noqa: F401
from .registry import MODEL, BACKBONE, install_into  # noqa: F401
from . import methods  # noqa: F401  (registers BCNN / CBCNN / MPN by import side effect, like model/__init__.py)

__all__ = ['MODEL', 'BACKBONE', 'install_into']
