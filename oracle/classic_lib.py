"""TEST INFRASTRUCTURE ONLY: classic.cu's sin / cos helpers on the device (classic_probe.cu).

  libclassic_probe.so   epb::M<double> and epb::M<float>'s sincos_small_, sin_, cos_ and
                        sincos_, compiled from classic.cu itself with classic.cu's nvcc flags

`build()` compiles it when stale (`__graft_entry__.build()` calls it); it is also built on first
use.  The product package envpool_b200 never imports this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
PROBE_SO = os.path.join(_HERE, "libclassic_probe.so")
_SRC = os.path.join(_HERE, "classic_probe.cu")
FUNCS = ("sincos_small", "sin", "cos", "sincos")


def _deps():
    csrc = os.path.join(_ROOT, "envpool_b200", "csrc")
    return [_SRC, os.path.join(csrc, "classic.cu"), os.path.join(csrc, "common.cuh"),
            os.path.join(_ROOT, "envpool_b200", "_build.py")]


def build() -> str:
    """Compile the probe when it is missing or older than classic.cu, common.cuh, its source or
    _build.py (whose flags it follows)."""
    from envpool_b200 import _build

    if not os.path.exists(PROBE_SO) or any(os.path.getmtime(d) > os.path.getmtime(PROBE_SO)
                                           for d in _deps()):
        tmp = PROBE_SO + ".tmp%d" % os.getpid()
        subprocess.check_call([_build._nvcc()] + _build.NVCC_COMMON +
                              _build.CUDA_UNITS["classic.cu"] +
                              ["-shared", "-cudart", "static", "-o", tmp, _SRC])
        os.replace(tmp, PROBE_SO)
    return PROBE_SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        vp = ctypes.c_void_p
        for fn in FUNCS:
            for p in ("f64", "f32"):
                f = getattr(L, f"classic_probe_{fn}_{p}")
                f.restype = ctypes.c_int
                f.argtypes = [vp, vp, vp, ctypes.c_int, vp]
        _lib = L
    return _lib


def device_trig(fn, x):
    """classic.cu's M<R>::<fn>_ of every element of `x` (a numpy float64 or float32 array, R
    from its dtype) on the current CUDA device and torch stream: (sin, cos), either None where
    `fn` does not compute it ("sin" -> (s, None), "cos" -> (None, c))."""
    import torch

    x = np.ascontiguousarray(x)
    tag = {np.dtype(np.float64): "f64", np.dtype(np.float32): "f32"}[x.dtype]
    dx = torch.from_numpy(x.ravel()).cuda()
    ds = torch.empty_like(dx) if fn != "cos" else None
    dc = torch.empty_like(dx) if fn != "sin" else None
    rc = getattr(lib(), f"classic_probe_{fn}_{tag}")(
        dx.data_ptr(), None if ds is None else ds.data_ptr(),
        None if dc is None else dc.data_ptr(), dx.numel(), torch.cuda.current_stream().cuda_stream)
    if rc:
        raise RuntimeError(f"classic_probe_{fn}_{tag}: CUDA error {rc}")
    out = tuple(None if d is None else d.cpu().numpy().reshape(x.shape) for d in (ds, dc))
    return out
