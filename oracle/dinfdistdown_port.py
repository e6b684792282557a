"""TEST INFRASTRUCTURE ONLY — ctypes wrapper of the C restatement of dinfdistdown, oracle/port/dinfdistdown_oracle.c (build: make -C
oracle -f dinfdistdown.mk port).  Only tests/ may import this module."""
import ctypes as C
import os

import numpy as np

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "port", "libdinfdistdown_oracle.so")
_lib = None
_P, _I, _F = C.c_void_p, C.c_int, C.c_float
METHODS = {"h": 0, "v": 1, "p": 2, "s": 3}
STATS = {"ave": 0, "max": 1, "min": 2}
MISSINGFLOAT = -3.4028234663852886e38


def available():
    return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_SO)
        _lib.orc_dinfdistdown.restype = C.c_longlong
        _lib.orc_dinfdistdown.argtypes = [_P, _P, _P, _P, _P, _I, _I, _F, _F, _F, _P, _P, _I, _I, _I]
    return _lib


def _rows(v, ny):
    a = np.asarray(v, dtype=np.float64)
    return np.ascontiguousarray(np.full(ny, float(a)) if a.ndim == 0 else a)


def dinfdistdown(ang, src, fel=None, weights=None, method="h", stat="ave", contcheck=True, dx=30.0, dy=30.0, dxc=None, dyc=None,
                 ang_nodata=MISSINGFLOAT, fel_nodata=-3.0e38, w_nodata=MISSINGFLOAT):
    """dd (float32, nodata MISSINGFLOAT); src is read as int16 (integers saturate)"""
    ang = np.ascontiguousarray(ang, np.float32)
    s = np.asarray(src)
    src = np.ascontiguousarray(np.clip(s, -32768, 32767) if s.dtype.kind in "iu" else s, np.int16)
    ny, nx = ang.shape
    assert src.shape == ang.shape
    fel = None if method == "h" or fel is None else np.ascontiguousarray(fel, np.float32)
    w = None if method == "v" or weights is None else np.ascontiguousarray(weights, np.float32)
    xc, yc = _rows(dx if dxc is None else dxc, ny), _rows(dy if dyc is None else dyc, ny)
    out = np.empty((ny, nx), np.float32)
    ptr = lambda a: None if a is None else a.ctypes.data
    lib().orc_dinfdistdown(ang.ctypes.data, ptr(fel), ptr(w), src.ctypes.data, out.ctypes.data, nx, ny, float(ang_nodata), float(fel_nodata),
                           float(w_nodata), xc.ctypes.data, yc.ctypes.data, STATS[stat], METHODS[method], int(bool(contcheck)))
    return out
