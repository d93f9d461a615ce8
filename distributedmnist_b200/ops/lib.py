"""ctypes loader for the sm_90a kernel library.

The library is built in-tree by ``ops/build.py``.  On a box with a GPU a missing
or unloadable library is a hard error -- the CUDA path never silently falls back
to PyTorch ops.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

from . import build as _build

_lib: Optional[ctypes.CDLL] = None


class KernelLibraryError(RuntimeError):
    pass


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    if not os.path.exists(path):
        if not build_if_missing:
            raise KernelLibraryError("kernel library %s is missing; run `python -m distributedmnist_b200.ops.build`" % path)
        _build.build()
    try:
        _lib = ctypes.CDLL(path)
    except OSError as e:
        raise KernelLibraryError("cannot load %s: %s" % (path, e))
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise KernelLibraryError("%s failed with code %d" % (what, rc))


def ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def stream_ptr(stream: Optional[torch.cuda.Stream] = None) -> ctypes.c_void_p:
    s = torch.cuda.current_stream() if stream is None else stream
    return ctypes.c_void_p(s.cuda_stream)


def require_hopper(device: torch.device) -> None:
    """The library holds sm_90a code only (wgmma, TMA): it loads on nothing but a compute capability 9.0 device."""
    cc = load().dm_device_cc(device.index or 0)
    if cc != 90:
        raise KernelLibraryError("device %s has compute capability %d; this library is sm_90a-only" % (device, cc))
