"""TEST INFRASTRUCTURE ONLY — ctypes wrapper of the C restatement oracle/port/taudem_oracle.c
(build: make -C oracle port).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline
leg may import this module."""
import ctypes as C
import os

import numpy as np

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "port", "libtaudem_oracle.so")
_lib = None
_P, _I, _F = C.c_void_p, C.c_int, C.c_float


def available():
    return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_SO)
        _lib.orc_flood.argtypes = [_P, _P, _P, _I, _I, _F, _I]
        _lib.orc_set_skip_flats.argtypes = [_I]
        _lib.orc_flat_stats.argtypes = [_P]
        _lib.orc_set_outlets.argtypes = [_P, _P, _I]
        _lib.orc_d8.argtypes = [_P, _P, _P, _I, _I, _F, _P, _P]
        _lib.orc_dinf.argtypes = [_P, _P, _P, _I, _I, _F, _P, _P]
        _lib.orc_aread8.argtypes = [_P, _P, _P, _I, _I, C.c_int16, _F, _I, _I]
        _lib.orc_areadinf.argtypes = [_P, _P, _P, _I, _I, _F, _I, _I, _P, _P]
        _lib.orc_flowpathextremeup.argtypes = [_P, _P, _P, _I, _I, C.c_int16, _I, _I]
        _lib.orc_gridnet.argtypes = [_P, _P, _I, _P, _P, _P, _I, _I, C.c_int16, _P, _P]
        _lib.orc_dinfdecayaccum.argtypes = [_P, _P, _P, _P, _I, _I, _F, _F, _I, _I, _P, _P]
        _lib.orc_dinfconclimaccum.argtypes = [_P, _P, _P, _P, _P, _I, _I, _F, _F, _F, _F, _I, _P, _P]
        _lib.orc_dinftranslimaccum.argtypes = [_P, _P, _P, _P, _P, _P, _P, _I, _I, _F, _F, _F, _F, _I, _P, _P]
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(_P)


def _rows(v, ny):
    a = np.asarray(v, dtype=np.float64)
    return np.ascontiguousarray(np.full(ny, float(a)) if a.ndim == 0 else a)


def pitremove(dem, nodata=-9999.0, four_way=False, depmask=None):
    dem = np.ascontiguousarray(dem, np.float32); ny, nx = dem.shape
    out = np.empty_like(dem)
    m = None if depmask is None else np.ascontiguousarray(depmask, np.int16)
    assert lib().orc_flood(_p(dem), _p(out), _p(m), nx, ny, nodata, int(four_way)) == 0
    return out


def d8flowdir(fel, nodata=-3.0e38, dx=30.0, dy=30.0, flats=True):
    """flats=False: stop after the positive-slope stencil (flat cells keep direction 0)."""
    lib().orc_set_skip_flats(0 if flats else 1)
    fel = np.ascontiguousarray(fel, np.float32); ny, nx = fel.shape
    p, sd8 = np.empty((ny, nx), np.int16), np.empty((ny, nx), np.float32)
    dxc, dyc = _rows(dx, ny), _rows(dy, ny)
    assert lib().orc_d8(_p(fel), _p(p), _p(sd8), nx, ny, nodata, _p(dxc), _p(dyc)) == 0
    return p, sd8


def dinfflowdir(fel, nodata=-3.0e38, dx=30.0, dy=30.0, flats=True):
    """flats=False: stop after the facet stencil (flat cells keep angle -1)."""
    lib().orc_set_skip_flats(0 if flats else 1)
    fel = np.ascontiguousarray(fel, np.float32); ny, nx = fel.shape
    ang, slp = np.empty((ny, nx), np.float32), np.empty((ny, nx), np.float32)
    dxc, dyc = _rows(dx, ny), _rows(dy, ny)
    assert lib().orc_dinf(_p(fel), _p(ang), _p(slp), nx, ny, nodata, _p(dxc), _p(dyc)) == 0
    return ang, slp


FLAT_STATS = ("iters", "T", "U", "pits", "fall_level", "rise_level", "elev2")


def flat_stats():
    """What the last d8flowdir / dinfflowdir call's flat resolution reached: iters = outer iterations, T / U = the largest number
    of fall / rise passes, pits = cells marked as pits, fall_level / rise_level = the largest number of cells that stop at one
    fall level / are first marked in one rise pass, elev2 = the largest level + s before it is stored in 16 bits."""
    out = np.zeros(len(FLAT_STATS), np.int64)
    lib().orc_flat_stats(_p(out))
    return dict(zip(FLAT_STATS, (int(v) for v in out)))


class _Outlets:
    """outlets = (cols, rows) grid cells: only the cells upstream of them are evaluated (-o)."""
    def __init__(self, outlets):
        self.o = outlets
    def __enter__(self):
        if self.o is None:
            lib().orc_set_outlets(None, None, -1)
        else:
            self.c = np.ascontiguousarray(self.o[0], np.int32); self.r = np.ascontiguousarray(self.o[1], np.int32)
            lib().orc_set_outlets(_p(self.c), _p(self.r), len(self.c))
    def __exit__(self, *a):
        lib().orc_set_outlets(None, None, -1)


def aread8(p, nodata=-32768, weights=None, w_nodata=-9999.0, contcheck=True, outlets=None):
    with _Outlets(outlets):
        return _aread8(p, nodata, weights, w_nodata, contcheck)


def areadinf(ang, nodata=-3.4028234663852886e38, weights=None, dx=30.0, dy=30.0, contcheck=True, outlets=None):
    with _Outlets(outlets):
        return _areadinf(ang, nodata, weights, dx, dy, contcheck)


def _aread8(p, nodata=-32768, weights=None, w_nodata=-9999.0, contcheck=True):
    p = np.ascontiguousarray(p, np.int16); ny, nx = p.shape
    out = np.empty((ny, nx), np.float32)
    w = None if weights is None else np.ascontiguousarray(weights, np.float32)
    assert lib().orc_aread8(_p(p), _p(w), _p(out), nx, ny, nodata, w_nodata, int(w is not None), int(contcheck)) == 0
    return out


def _areadinf(ang, nodata=-3.4028234663852886e38, weights=None, dx=30.0, dy=30.0, contcheck=True):
    ang = np.ascontiguousarray(ang, np.float32); ny, nx = ang.shape
    out = np.empty((ny, nx), np.float32)
    w = None if weights is None else np.ascontiguousarray(weights, np.float32)
    dxc, dyc = _rows(dx, ny), _rows(dy, ny)
    assert lib().orc_areadinf(_p(ang), _p(w), _p(out), nx, ny, nodata, int(w is not None), int(contcheck), _p(dxc), _p(dyc)) == 0
    return out


# ---- the sibling sweep tools, with the signatures of taudem_b200.api's *_grid functions.  dx / dy: scalars or per-row arrays;
#      dxc / dyc (per-row arrays) take precedence, as in the api.
MISSINGFLOAT = -3.4028234663852886e38


def _sizes(dx, dy, dxc, dyc, ny):
    return _rows(dx if dxc is None else dxc, ny), _rows(dy if dyc is None else dyc, ny)


def _f32(a, shape):
    a = np.ascontiguousarray(a, np.float32)
    assert a.shape == shape
    return a


def d8flowpathextremeup(p, sa, usemax=True, nodata=-32768, contcheck=True, outlets=None):
    p = np.ascontiguousarray(p, np.int16); ny, nx = p.shape
    sa = _f32(sa, p.shape)
    out = np.empty((ny, nx), np.float32)
    with _Outlets(outlets):
        assert lib().orc_flowpathextremeup(_p(p), _p(sa), _p(out), nx, ny, nodata, int(usemax), int(contcheck)) == 0
    return out


def gridnet(p, mask=None, thresh=0, dx=30.0, dy=30.0, nodata=-32768, outlets=None, dxc=None, dyc=None):
    """(plen, tlen, gord)"""
    p = np.ascontiguousarray(p, np.int16); ny, nx = p.shape
    m = None if mask is None else np.ascontiguousarray(mask, np.int32)
    dxc, dyc = _sizes(dx, dy, dxc, dyc, ny)
    plen, tlen, gord = np.empty((ny, nx), np.float32), np.empty((ny, nx), np.float32), np.empty((ny, nx), np.int16)
    with _Outlets(outlets):
        assert lib().orc_gridnet(_p(p), _p(m), int(thresh), _p(plen), _p(tlen), _p(gord), nx, ny, nodata, _p(dxc), _p(dyc)) == 0
    return plen, tlen, gord


def dinfdecayaccum(ang, dm, weights=None, dx=30.0, dy=30.0, nodata=MISSINGFLOAT, dm_nodata=-9999.0, contcheck=True, outlets=None, dxc=None, dyc=None):
    ang = np.ascontiguousarray(ang, np.float32); ny, nx = ang.shape
    dm = _f32(dm, ang.shape)
    w = None if weights is None else _f32(weights, ang.shape)
    dxc, dyc = _sizes(dx, dy, dxc, dyc, ny)
    out = np.empty((ny, nx), np.float32)
    with _Outlets(outlets):
        assert lib().orc_dinfdecayaccum(_p(ang), _p(dm), _p(w), _p(out), nx, ny, nodata, dm_nodata, int(w is not None), int(contcheck), _p(dxc), _p(dyc)) == 0
    return out


def dinfconclimaccum(ang, dm, q, dg, csol=1.0, dx=30.0, dy=30.0, nodata=MISSINGFLOAT, dm_nodata=-9999.0, q_nodata=-9999.0, contcheck=True, outlets=None,
                     dxc=None, dyc=None):
    ang = np.ascontiguousarray(ang, np.float32); ny, nx = ang.shape
    dm, q = _f32(dm, ang.shape), _f32(q, ang.shape)
    dg = np.ascontiguousarray(dg, np.int16); assert dg.shape == ang.shape
    dxc, dyc = _sizes(dx, dy, dxc, dyc, ny)
    out = np.empty((ny, nx), np.float32)
    with _Outlets(outlets):
        assert lib().orc_dinfconclimaccum(_p(ang), _p(dm), _p(q), _p(dg), _p(out), nx, ny, nodata, dm_nodata, q_nodata, csol, int(contcheck),
                                          _p(dxc), _p(dyc)) == 0
    return out


def dinftranslimaccum(ang, tsup, tc, cs=None, dx=30.0, dy=30.0, nodata=MISSINGFLOAT, tsup_nodata=-9999.0, tc_nodata=-9999.0, cs_nodata=-9999.0,
                      contcheck=True, outlets=None, dxc=None, dyc=None):
    """(tla, tdep, ctpt); ctpt is None without cs"""
    ang = np.ascontiguousarray(ang, np.float32); ny, nx = ang.shape
    tsup, tc = _f32(tsup, ang.shape), _f32(tc, ang.shape)
    c = None if cs is None else _f32(cs, ang.shape)
    dxc, dyc = _sizes(dx, dy, dxc, dyc, ny)
    tla, dep = np.empty((ny, nx), np.float32), np.empty((ny, nx), np.float32)
    cout = None if c is None else np.empty((ny, nx), np.float32)
    with _Outlets(outlets):
        assert lib().orc_dinftranslimaccum(_p(ang), _p(tsup), _p(tc), _p(c), _p(tla), _p(dep), _p(cout), nx, ny, nodata, tsup_nodata, tc_nodata, cs_nodata,
                                           int(contcheck), _p(dxc), _p(dyc)) == 0
    return tla, dep, cout
