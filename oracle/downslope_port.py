"""TEST INFRASTRUCTURE ONLY — ctypes wrapper of the C restatement of slopeavedown, oracle/port/slopeavedown_oracle.c
(build: make -C oracle -f downslope.mk port).  Only tests/ may import this module."""
import ctypes as C
import os

import numpy as np

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "port", "libslopeavedown_oracle.so")
_lib = None
_P, _I, _F, _D = C.c_void_p, C.c_int, C.c_float, C.c_double


def available():
    return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_SO)
        _lib.orc_slopeavedown.argtypes = [_P, _P, _P, _I, _I, _F, C.c_int16, _P, _P, _D, _D, _D, _P]
        _lib.orc_slopeavedown_niter.argtypes = [_D, _D, _D, _P]
    return _lib


def _rows(v, ny):
    a = np.asarray(v, dtype=np.float64)
    return np.ascontiguousarray(np.full(ny, float(a)) if a.ndim == 0 else a)


def niter(dn, dx, dy):
    """the reference's pass count, or None where it is undefined"""
    n = C.c_int(0)
    return None if lib().orc_slopeavedown_niter(float(dn), float(dx), float(dy), C.byref(n)) else n.value


def slopeavedown(fel, p, dn=50.0, dx=30.0, dy=30.0, nodata=-3.0e38, p_nodata=-32768, dxc=None, dyc=None, passes=False):
    """slpd (float32, nodata MISSINGFLOAT), the signature of taudem_b200.slopeavedown_grid.  passes=True: (slpd, the number of the
    last pass that changed anything)."""
    fel = np.ascontiguousarray(fel, np.float32)
    p = np.ascontiguousarray(p, np.int16)
    ny, nx = fel.shape
    assert p.shape == fel.shape
    xc, yc = _rows(dx if dxc is None else dxc, ny), _rows(dy if dyc is None else dyc, ny)
    sd = np.empty((ny, nx), np.float32)
    last = C.c_int(0)
    rc = lib().orc_slopeavedown(fel.ctypes.data, p.ctypes.data, sd.ctypes.data, nx, ny, float(nodata), int(p_nodata), xc.ctypes.data, yc.ctypes.data,
                                float(dx), float(dy), float(dn), C.byref(last))
    if rc:
        raise ValueError("slopeavedown: dn / min(dx, dy) + 1 is undefined as an int")
    return (sd, last.value) if passes else sd
