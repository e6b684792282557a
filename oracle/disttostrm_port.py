"""TEST INFRASTRUCTURE ONLY — ctypes wrapper of the C restatement of d8hdisttostrm and d8vdisttostrm, oracle/port/disttostrm_oracle.c
(build: make -C oracle -f disttostrm.mk port).  Only tests/ may import this module."""
import ctypes as C
import os

import numpy as np

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "port", "libdisttostrm_oracle.so")
_lib = None
_P, _I = C.c_void_p, C.c_int


def available():
    return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_SO)
        _lib.orc_disttostrm.argtypes = [_I, _P, _P, _P, _P, _I, _I, C.c_int16, C.c_int32, _I, _P, _P]
    return _lib


def _rows(v, ny):
    a = np.asarray(v, dtype=np.float64)
    return np.ascontiguousarray(np.full(ny, float(a)) if a.ndim == 0 else a)


def disttostrm(p, src, fel=None, thresh=1, dx=30.0, dy=30.0, p_nodata=-32768, src_nodata=-2147483648, dxc=None, dyc=None):
    """dist (float32, nodata MISSINGFLOAT): d8vdisttostrm where fel is given, else d8hdisttostrm"""
    p = np.ascontiguousarray(p, np.int16)
    src = np.ascontiguousarray(src, np.int32)
    ny, nx = p.shape
    assert src.shape == p.shape
    vertical = fel is not None
    fel = np.ascontiguousarray(fel if vertical else np.zeros((1, 1)), np.float32)
    xc, yc = _rows(dx if dxc is None else dxc, ny), _rows(dy if dyc is None else dyc, ny)
    out = np.empty((ny, nx), np.float32)
    lib().orc_disttostrm(int(vertical), p.ctypes.data, fel.ctypes.data, src.ctypes.data, out.ctypes.data, nx, ny, int(p_nodata), int(src_nodata),
                         int(thresh), xc.ctypes.data, yc.ctypes.data)
    return out
