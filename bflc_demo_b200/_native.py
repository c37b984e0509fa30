"""Loader for the in-tree native modules (built by ``bflc_demo_b200.build``).

``_C``      CUDA kernels (sm_90a) + symmetric heap + torch bindings
``_ledger`` C++ ledger runtime (host only)

On a GPU box a missing ``_C.so`` is a hard error: ops must never fall back silently to
eager PyTorch (the driver records which in-tree .so files were actually loaded).
"""
from __future__ import annotations

import importlib.util
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
_cache: dict = {}


def _load(name: str):
    if name in _cache:
        return _cache[name]
    path = _HERE / f"{name}.so"
    if not path.exists():
        if os.environ.get("BFLC_NO_AUTOBUILD", "0") == "1":
            raise ImportError(f"{path} missing; run `python -m bflc_demo_b200.build`")
        from . import build as _build

        _build.build_all(verbose=False)
    spec = importlib.util.spec_from_file_location(f"bflc_demo_b200.{name}", str(path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    _cache[name] = mod
    return mod


def C():
    """The CUDA kernel module (imports torch first so libtorch symbols resolve)."""
    import torch  # noqa: F401

    fresh = "_C" not in _cache
    mod = _load("_C")
    if fresh and os.environ.get("BFLC_PDL", "1") == "0":
        mod.set_pdl(False)  # A/B switch: plain stream-ordered launches
    return mod


def ledger():
    return _load("_ledger")


def have_cuda() -> bool:
    import torch

    return torch.cuda.is_available()
