"""TEST INFRASTRUCTURE ONLY — ctypes wrapper of the C restatements of flowdircond and retlimflow, oracle/port/conditioning_oracle.c
(build: make -C oracle -f conditioning.mk port).  Only tests/ may import this module."""
import ctypes as C
import os

import numpy as np

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "port", "libconditioning_oracle.so")
_lib = None
_P, _I, _F = C.c_void_p, C.c_int, C.c_float


def available():
    return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_SO)
        _lib.orc_flowdircond.argtypes = [_P, _P, _P, _I, _I, C.c_int16, _F, _P]
        _lib.orc_flowdircond.restype = None
        _lib.orc_retlimflow.argtypes = [_P, _P, _P, _P, _I, _I, _F, _F, _F, _P, _P, _I, _P]
        _lib.orc_retlimflow.restype = None
    return _lib


def flowdircond(p, z, p_nodata=-32768, nodata=-9999.0, processed=False):
    """zfdc (float32, z's nodata), the signature of taudem_b200.flowdircond_grid.  processed=True: (zfdc, the number of cells the
    reference's queue dequeued)."""
    p = np.ascontiguousarray(p, np.int16)
    z = np.ascontiguousarray(z, np.float32)
    ny, nx = z.shape
    assert p.shape == z.shape
    out = np.empty((ny, nx), np.float32)
    n = C.c_longlong(0)
    lib().orc_flowdircond(p.ctypes.data, z.ctypes.data, out.ctypes.data, nx, ny, int(p_nodata), np.float32(nodata), C.byref(n))
    return (out, n.value) if processed else out


def _rows(v, ny):
    a = np.asarray(v, dtype=np.float64)
    return np.ascontiguousarray(np.full(ny, float(a)) if a.ndim == 0 else a)


def retlimflow(ang, wg, rc, dx=30.0, dy=30.0, ang_nodata=-3.4028234663852886e38, wg_nodata=-9999.0, rc_nodata=-9999.0, dxc=None, dyc=None,
               edge_quirk=False, processed=False):
    """qrl (float32, nodata MISSINGFLOAT), the signature of taudem_b200.retlimflow_grid.  edge_quirk=True: also the reference's
    one-rank handling of shares that leave the grid through the top / bottom edge (oracle/port/conditioning_oracle.c); False: the
    contract of the GPU, where they decrement nothing.  processed=True: (qrl, the number of cells the queue dequeued)."""
    ang, wg, rc = (np.ascontiguousarray(a, np.float32) for a in (ang, wg, rc))
    ny, nx = ang.shape
    assert wg.shape == ang.shape == rc.shape
    xc, yc = _rows(dx if dxc is None else dxc, ny), _rows(dy if dyc is None else dyc, ny)
    out = np.empty((ny, nx), np.float32)
    n = C.c_longlong(0)
    lib().orc_retlimflow(ang.ctypes.data, wg.ctypes.data, rc.ctypes.data, out.ctypes.data, nx, ny, np.float32(ang_nodata), np.float32(wg_nodata),
                         np.float32(rc_nodata), xc.ctypes.data, yc.ctypes.data, int(edge_quirk), C.byref(n))
    return (out, n.value) if processed else out
