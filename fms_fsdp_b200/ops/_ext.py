"""Loader for the in-tree sm_90a extension (``fms_fsdp_b200/_C*.so``).

The extension is built by ``__graft_entry__.build()`` / ``python -m fms_fsdp_b200.build``.
On a machine with a GPU the ops in this package *require* it: there is no silent
ATen fallback on CUDA tensors (``FMS_B200_ALLOW_TORCH_FALLBACK=1`` opts in for debugging).
"""
from __future__ import annotations

import importlib
import os
import threading

_lock = threading.Lock()
_mod = None
_err = None


def load():
    global _mod, _err
    if _mod is not None or _err is not None:
        return _mod
    with _lock:
        if _mod is None and _err is None:
            try:
                import torch  # noqa: F401  (libtorch symbols must be resident first)
                _mod = importlib.import_module("fms_fsdp_b200._C")
            except Exception as e:  # pragma: no cover - depends on build state
                _err = e
    return _mod


def available() -> bool:
    return load() is not None


def require():
    m = load()
    if m is None:
        raise RuntimeError(
            "fms_fsdp_b200._C (sm_90a kernels) is not built/loadable: "
            f"{_err!r}. Run `python -c 'import __graft_entry__ as g; g.build()'`."
        )
    return m


def allow_torch_fallback() -> bool:
    return os.environ.get("FMS_B200_ALLOW_TORCH_FALLBACK", "0") == "1"
