"""Loader for the in-tree sm_90a extension (``_C.so`` → ``torch.ops.rab.*``).

The extension is mandatory on a GPU box: if a CUDA device is visible and the shared object cannot be
loaded we raise instead of silently falling back to eager PyTorch.
"""
from __future__ import annotations

import os
import threading
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parent.parent
_SO = _PKG / "_C.so"
_lock = threading.Lock()
_loaded = False
_error: Exception | None = None


def extension_path() -> Path:
    return _SO


def load(build_if_missing: bool = True) -> bool:
    """Load ``_C.so``; returns True when ``torch.ops.rab`` is usable."""
    global _loaded, _error
    if _loaded:
        return True
    with _lock:
        if _loaded:
            return True
        try:
            if not _SO.exists() and build_if_missing and os.environ.get("RAB_NO_BUILD", "0") != "1":
                # every rank of a torchrun / mp.spawn launch gets here at the same time on a fresh checkout: one process
                # builds under an exclusive file lock, the others wait for it and then find the finished object
                import fcntl

                from ring_attention_pytorch_b200 import build as _build

                with open(str(_PKG / ".build.lock"), "w") as lock:
                    fcntl.flock(lock, fcntl.LOCK_EX)
                    try:
                        if not _SO.exists():
                            _build.build(verbose=False)
                    finally:
                        fcntl.flock(lock, fcntl.LOCK_UN)
            torch.ops.load_library(str(_SO))
            _loaded = True
        except Exception as e:  # pragma: no cover - depends on toolchain
            _error = e
            if torch.cuda.is_available():
                raise RuntimeError(
                    f"ring_attention_pytorch_b200: the sm_90a extension {_SO} failed to load on a CUDA machine: {e}"
                ) from e
            return False
    return True


def is_loaded() -> bool:
    return _loaded


def ops():
    if not load():
        raise RuntimeError(f"sm_90a extension unavailable: {_error}")
    return torch.ops.rab
