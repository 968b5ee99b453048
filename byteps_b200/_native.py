"""Loads the in-tree native modules, building them on first use if the shared
objects are missing (the normal flow is ``__graft_entry__.build()`` or
``python -m byteps_b200._build``)."""
import importlib
import os
import threading

_lock = threading.Lock()
_core = None
_cuda = None


def _try_import(name):
    try:
        return importlib.import_module("byteps_b200." + name)
    except ImportError:
        return None


def core():
    global _core
    if _core is None:
        with _lock:
            if _core is None:
                m = _try_import("_core")
                if m is None:
                    from . import _build

                    _build.build_core()
                    m = importlib.import_module("byteps_b200._core")
                _core = m
    return _core


def cuda():
    """The sm_90a extension.  Fails loudly if it cannot be built/loaded: a GPU
    box must never silently fall back to eager PyTorch."""
    global _cuda
    if _cuda is None:
        with _lock:
            if _cuda is None:
                import torch  # noqa: F401  (loads libcudart the extension links against)

                m = _try_import("_cuda")
                if m is None:
                    if os.environ.get("BYTEPS_NO_AUTOBUILD"):
                        raise ImportError("byteps_b200._cuda is not built (run __graft_entry__.build())")
                    from . import _build

                    _build.build_cuda()
                    m = importlib.import_module("byteps_b200._cuda")
                _cuda = m
    return _cuda


_torch_ops = None


def torch_ops():
    """The native torch adapter (push_pull on at::Tensor).  Fails loudly like cuda() - building it
    needs the torch headers of the running interpreter."""
    global _torch_ops
    if _torch_ops is None:
        with _lock:
            if _torch_ops is None:
                import torch  # noqa: F401

                m = _try_import("_torch_ops")
                if m is None:
                    if os.environ.get("BYTEPS_NO_AUTOBUILD"):
                        raise ImportError("byteps_b200._torch_ops is not built (run __graft_entry__.build())")
                    from . import _build

                    _build.build_torch()
                    m = importlib.import_module("byteps_b200._torch_ops")
                _torch_ops = m
    return _torch_ops
