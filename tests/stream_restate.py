"""Restatements of peukerdouglas and lengtharea in numpy (float32 arithmetic in the reference's order, no contraction), the oracle of
the stream-definition tests.

peukerdouglas (src/PeukerDouglas.cpp:109-212) on one grid: the smoothing pass, then every group of four cells (quad) with origin
(x, y), x in [0, nx-2], y in [-1, ny-1], visited like the reference: emax = the origin's value (the origin is not tested for nodata),
then (x+1, y), (x, y+1), (x+1, y+1) — a nodata cell marks the quad as bound, a larger one becomes the maximum; the maximum is
unflagged, and all four cells of a bound quad or the cells equal to emax of the others.  Rows outside the grid read as nodata.  A
quad only ever clears flags, so the order in which quads are visited does not matter and they are evaluated all at once here.

lengtharea (src/LengthArea.cpp:110-120): 1 where (float)ad8 >= M * powf(plen, y) in float, else 0; -32768 where plen < 0.  ad8 is
read as 32-bit integers, rounded half away from zero.  powf is libm's, like the reference's."""
import ctypes
import ctypes.util

import numpy as np

MINEPS = np.float32(1e-5)

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.powf.restype = ctypes.c_float
_libm.powf.argtypes = [ctypes.c_float, ctypes.c_float]
_powf = np.frompyfunc(lambda x, y: _libm.powf(x, y), 2, 1)


def _isnd(v, nd):
    return np.abs(v - nd) < MINEPS


def peukerdouglas(fel, weights=(0.4, 0.1, 0.05), nodata=-3.0e38):
    """int16 stream sources, 0 / 1 on every cell"""
    fel = np.ascontiguousarray(fel, np.float32)
    ny, nx = fel.shape
    nd = np.float32(nodata)
    wm, ws, wd = (np.float32(w) for w in weights)
    # pass 1: smoothing of the cells off the grid's edge that are not nodata (their eight neighbours are all inside the grid)
    s = fel.copy()
    ss = np.zeros((ny, nx), np.int16)
    if ny > 2 and nx > 2:
        c = fel[1:-1, 1:-1]
        inner = ~_isnd(c, nd)
        acc = wm * c
        wsum = np.full(c.shape, wm, np.float32)
        side = ((0, 1), (-1, 0), (0, -1), (1, 0))            # k = 1 E, 3 N, 5 W, 7 S
        diag = ((-1, 1), (-1, -1), (1, -1), (1, 1))          # k = 2 NE, 4 NW, 6 SW, 8 SE
        for w, group in ((ws, side), (wd, diag)):                # (nodata neighbours are computed, then discarded)
            if not w > 0:
                continue
            for dy, dx in group:
                v = fel[1 + dy:ny - 1 + dy, 1 + dx:nx - 1 + dx]
                ok = ~_isnd(v, nd)
                with np.errstate(all="ignore"):
                    acc = np.where(ok, (acc + (v * w).astype(np.float32)).astype(np.float32), acc)
                wsum = np.where(ok, (wsum + w).astype(np.float32), wsum)
        with np.errstate(all="ignore"):
            s[1:-1, 1:-1] = np.where(inner, (acc / wsum).astype(np.float32), c)
        ss[1:-1, 1:-1] = inner
    # pass 2: the quads on s; P = s with a nodata row above and below, quad origin row y <-> P row y + 1
    if nx < 2:
        return ss
    P = np.full((ny + 2, nx), nd, np.float32)
    P[1:-1] = s
    q = (P[:-1, :-1], P[:-1, 1:], P[1:, :-1], P[1:, 1:])
    emax = q[0].copy()
    am = np.zeros(emax.shape, np.int8)
    bound = np.zeros(emax.shape, bool)
    for i in (1, 2, 3):
        n = _isnd(q[i], nd)
        bound |= n
        up = ~n & (q[i] > emax)
        emax = np.where(up, q[i], emax)
        am = np.where(up, np.int8(i), am)
    clear = np.zeros(P.shape, bool)
    for i, (r, cc) in enumerate(((slice(0, -1), slice(0, -1)), (slice(0, -1), slice(1, None)), (slice(1, None), slice(0, -1)),
                                 (slice(1, None), slice(1, None)))):
        clear[r, cc] |= bound | (am == i) | (q[i] == emax)
    ss[clear[1:-1]] = 0
    return ss


def ad8_int32(ad8):
    """the contributing area as the reference reads it for lengtharea: 32-bit integers, rounded half away from zero"""
    a = np.asarray(ad8, np.float64)
    return np.trunc(a + np.copysign(0.5, a)).astype(np.int32)


def lengtharea(plen, ad8, m=None, y=None):
    """int16: 1 where (float)ad8 >= M * plen^y (M = 0.03, y = 1.3 by default), else 0; -32768 where plen < 0"""
    plen = np.asarray(plen, np.float32)
    a = ad8_int32(ad8)
    m, y = (np.float32(0.03), np.float32(1.3)) if m is None else (np.float32(m), np.float32(y))
    ok = plen >= 0
    out = np.full(plen.shape, -32768, np.int16)
    out[ok] = (a[ok].astype(np.float32) >= (m * _powf(plen[ok], y).astype(np.float32)).astype(np.float32)).astype(np.int16)
    return out
