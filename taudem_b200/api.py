"""Host-side mirror of the reference's interface for the hot path.

File level: ``flood``, ``setdird8``, ``setdir``, ``aread8``, ``area`` take the same
arguments, in the same order and with the same meaning, as the reference functions
(src/flood.cpp:50, src/d8.cpp:181, src/dinf.cpp:109, src/aread8.cpp:56,
src/areadinf.cpp:53) and return 0 on success like they do.

Grid level: ``*_grid`` functions run the same device path on numpy arrays (row 0 =
north).  dx/dy may be scalars (projected grids) or per-row arrays (geographic grids,
tiffIO::getdxc/getdyc).
"""
import ctypes as C

import numpy as np

from ._lib import check, lib

_DT = {np.dtype(np.int16): 0, np.dtype(np.int32): 1, np.dtype(np.float32): 2}

FEL_NODATA = np.float32(-3.0e38)            # src/flood.cpp:136
MISSINGFLOAT = np.float32(-3.4028234663852886e38)   # src/commonLib.h:80
MISSINGSHORT = np.int16(-32768)             # src/commonLib.h:77


def _b(s):
    return (s or "").encode()


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _rows(v, ny):
    a = np.asarray(v, dtype=np.float64)
    if a.ndim == 0:
        a = np.full(ny, float(a), dtype=np.float64)
    if a.shape != (ny,):
        raise ValueError("per-row cell sizes must have one value per row")
    return np.ascontiguousarray(a)


def _grid(a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    if a.ndim != 2:
        raise ValueError("rasters are 2-D arrays")
    return a


# --------------------------------------------------------------------- file level
def flood(demfile, felfile, sfdrfile="", usesfdr=0, verbose=False, is_4Point=False, use_mask=False, maskfile=""):
    return lib().td_flood(_b(demfile), _b(felfile), _b(sfdrfile), int(usesfdr), int(verbose), int(is_4Point), int(use_mask), _b(maskfile))


def setdird8(demfile, pointfile, slopefile, flowfile="", useflowfile=0):
    return lib().td_setdird8(_b(demfile), _b(pointfile), _b(slopefile), _b(flowfile), int(useflowfile))


def setdir(demfile, angfile, slopefile, flowfile="", useflowfile=0):
    return lib().td_setdir(_b(demfile), _b(angfile), _b(slopefile), _b(flowfile), int(useflowfile))


def aread8(pfile, afile, datasrc="", lyrname="", uselyrname=0, lyrno=0, wfile="", useOutlets=0, usew=0, contcheck=1):
    return lib().td_aread8(_b(pfile), _b(afile), _b(datasrc), _b(lyrname), int(uselyrname), int(lyrno), _b(wfile), int(useOutlets), int(usew), int(contcheck))


def area(angfile, scafile, datasrc="", lyrname="", uselyrname=0, lyrno=0, wfile="", useOutlets=0, usew=0, contcheck=1):
    return lib().td_area(_b(angfile), _b(scafile), _b(datasrc), _b(lyrname), int(uselyrname), int(lyrno), _b(wfile), int(useOutlets), int(usew), int(contcheck))


def nameadd(arg, suff):
    buf = C.create_string_buffer(4096)
    lib().td_nameadd(buf, _b(arg), _b(suff))
    return buf.value.decode()


# --------------------------------------------------------------------- raster files
def raster_info(path):
    nx, ny, hn, geo, bits, fmt = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
    nd, dx, dy = C.c_double(), C.c_double(), C.c_double()
    check(lib().td_raster_info(_b(path), C.byref(nx), C.byref(ny), C.byref(nd), C.byref(hn), C.byref(dx), C.byref(dy),
                               C.byref(geo), C.byref(bits), C.byref(fmt)))
    return dict(nx=nx.value, ny=ny.value, nodata=nd.value, has_nodata=bool(hn.value), dx=dx.value, dy=dy.value,
                is_geographic=bool(geo.value), bits=bits.value, sample_format=fmt.value)


def read_raster(path, dtype=np.float32):
    info = raster_info(path)
    out = np.empty((info["ny"], info["nx"]), dtype=dtype)
    check(lib().td_raster_read(_b(path), _DT[np.dtype(dtype)], _ptr(out), info["nx"], info["ny"]))
    return out


def write_raster(path, arr, nodata, like=None, dx=30.0, dy=30.0, compression=1):
    arr = np.ascontiguousarray(arr)
    check(lib().td_raster_write(_b(path), _DT[arr.dtype], _ptr(arr), arr.shape[1], arr.shape[0], float(nodata),
                                _b(like) if like else None, float(dx), float(dy), int(compression)))


# --------------------------------------------------------------------- grid level
def pitremove_grid(dem, nodata=-9999.0, depmask=None, is_4Point=False, out=None):
    dem = _grid(dem, np.float32)
    ny, nx = dem.shape
    fel = out if out is not None else np.empty_like(dem)
    m = None if depmask is None else _grid(depmask, np.int16)
    check(lib().td_flood_host(_ptr(dem), _ptr(fel), _ptr(m), nx, ny, np.float32(nodata), int(is_4Point)))
    return fel


def d8flowdir_grid(fel, nodata=float(FEL_NODATA), dx=30.0, dy=30.0, out=None):
    fel = _grid(fel, np.float32)
    ny, nx = fel.shape
    p, sd8 = out if out is not None else (np.empty((ny, nx), np.int16), np.empty((ny, nx), np.float32))
    dxc, dyc = _rows(dx, ny), _rows(dy, ny)
    check(lib().td_setdird8_host(_ptr(fel), _ptr(p), _ptr(sd8), nx, ny, np.float32(nodata), _ptr(dxc), _ptr(dyc)))
    return p, sd8


def dinfflowdir_grid(fel, nodata=float(FEL_NODATA), dx=30.0, dy=30.0, out=None):
    fel = _grid(fel, np.float32)
    ny, nx = fel.shape
    ang, slp = out if out is not None else (np.empty((ny, nx), np.float32), np.empty((ny, nx), np.float32))
    dxc, dyc = _rows(dx, ny), _rows(dy, ny)
    check(lib().td_setdir_host(_ptr(fel), _ptr(ang), _ptr(slp), nx, ny, np.float32(nodata), _ptr(dxc), _ptr(dyc)))
    return ang, slp


def _outlet_args(outlets):
    """outlets = (cols, rows) of the outlet cells -> (cols array, rows array, n); None -> no outlets (n = -1)."""
    if outlets is None:
        return None, None, -1
    c = np.ascontiguousarray(outlets[0], np.int32); r = np.ascontiguousarray(outlets[1], np.int32)
    assert c.shape == r.shape and c.ndim == 1
    return c, r, len(c)


def read_outlets(datasrc, lyrname="", uselyrname=0, lyrno=0):
    """Outlet points (x, y) of a shapefile / GeoJSON data source (readoutlets, src/ReadOutlets.cpp)."""
    n = C.c_int(0)
    check(lib().td_outlets_read(_b(datasrc), _b(lyrname), int(uselyrname), int(lyrno), None, None, 0, C.byref(n)))
    x = np.empty(max(n.value, 1), np.float64); y = np.empty(max(n.value, 1), np.float64)
    check(lib().td_outlets_read(_b(datasrc), _b(lyrname), int(uselyrname), int(lyrno), _ptr(x), _ptr(y), n.value, C.byref(n)))
    return x[:n.value], y[:n.value]


def aread8_grid(p, nodata=int(MISSINGSHORT), weights=None, w_nodata=-9999.0, contcheck=True, out=None, outlets=None):
    p = _grid(p, np.int16)
    ny, nx = p.shape
    ad8 = out if out is not None else np.empty((ny, nx), np.float32)
    w = None if weights is None else _grid(weights, np.float32)
    oc, orow, nout = _outlet_args(outlets)
    check(lib().td_aread8_outlets_host(_ptr(p), _ptr(w), _ptr(ad8), nx, ny, int(nodata), np.float32(w_nodata), int(contcheck),
                                       _ptr(oc), _ptr(orow), nout))
    return ad8


def d8flowpathextremeup_grid(p, sa, usemax=True, nodata=int(MISSINGSHORT), contcheck=True, outlets=None):
    """The largest (smallest) value of `sa` on the D8 flow paths above each cell (td_d8flowpathextremeup_host;
    src/D8flowpathextremeup.cpp:182-215).  nodata = -FLT_MAX."""
    p = _grid(p, np.int16); sa = _grid(sa, np.float32)
    ny, nx = p.shape
    assert sa.shape == p.shape
    ssa = np.empty((ny, nx), np.float32)
    oc, orow, nout = _outlet_args(outlets)
    check(lib().td_d8flowpathextremeup_host(_ptr(p), _ptr(sa), _ptr(ssa), nx, ny, int(nodata), int(usemax), int(contcheck), _ptr(oc), _ptr(orow), nout))
    return ssa


def gridnet_grid(p, mask=None, thresh=0, dx=30.0, dy=30.0, nodata=int(MISSINGSHORT), outlets=None, dxc=None, dyc=None):
    """(plen, tlen, gord): longest and total upstream path length and Strahler order of the D8 flow field (td_gridnet_host;
    src/gridnet.cpp:383-420).  mask (int32): only cells with mask >= thresh are evaluated and contribute.  nodata = -1."""
    p = _grid(p, np.int16)
    ny, nx = p.shape
    m = None if mask is None else _grid(mask, np.int32)
    dxc = _rows(dx, ny) if dxc is None else np.ascontiguousarray(dxc, np.float64)
    dyc = _rows(dy, ny) if dyc is None else np.ascontiguousarray(dyc, np.float64)
    plen = np.empty((ny, nx), np.float32); tlen = np.empty((ny, nx), np.float32); gord = np.empty((ny, nx), np.int16)
    oc, orow, nout = _outlet_args(outlets)
    check(lib().td_gridnet_host(_ptr(p), _ptr(m), int(thresh), _ptr(plen), _ptr(tlen), _ptr(gord), nx, ny, int(nodata), _ptr(dxc), _ptr(dyc),
                                _ptr(oc), _ptr(orow), nout))
    return plen, tlen, gord


def dinfdecayaccum_grid(ang, dm, weights=None, dx=30.0, dy=30.0, nodata=float(MISSINGFLOAT), dm_nodata=-9999.0, contcheck=True, outlets=None,
                        dxc=None, dyc=None):
    """Decaying accumulation on the D-infinity flow field (td_dinfdecayaccum_host; src/dinfdecayaccum.cpp:205-235): a cell starts from
    its weight (or dx) and receives (float)(dm * area * p) from every contributor.  nodata = -FLT_MAX."""
    ang = _grid(ang, np.float32); dm = _grid(dm, np.float32)
    ny, nx = ang.shape
    assert dm.shape == ang.shape
    w = None if weights is None else _grid(weights, np.float32)
    dxc = _rows(dx, ny) if dxc is None else np.ascontiguousarray(dxc, np.float64)
    dyc = _rows(dy, ny) if dyc is None else np.ascontiguousarray(dyc, np.float64)
    out = np.empty((ny, nx), np.float32)
    oc, orow, nout = _outlet_args(outlets)
    check(lib().td_dinfdecayaccum_host(_ptr(ang), _ptr(dm), _ptr(w), _ptr(out), nx, ny, np.float32(nodata), np.float32(dm_nodata), _ptr(dxc), _ptr(dyc),
                                       int(contcheck), _ptr(oc), _ptr(orow), nout))
    return out


def dinfconclimaccum_grid(ang, dm, q, dg, csol=1.0, dx=30.0, dy=30.0, nodata=float(MISSINGFLOAT), dm_nodata=-9999.0, q_nodata=-9999.0, contcheck=True,
                          outlets=None, dxc=None, dyc=None):
    """Concentration limited accumulation on the D-infinity flow field (td_dinfconclimaccum_host; src/DinfConcLimAccum.cpp:242-270):
    cells with q > 0 only; an indicator cell (dg > 0) has the concentration csol, any other the float sum of p * ctpt * q * dm over its
    contributors divided by its own q.  nodata = -FLT_MAX."""
    ang = _grid(ang, np.float32); dm = _grid(dm, np.float32); q = _grid(q, np.float32); dg = _grid(dg, np.int16)
    ny, nx = ang.shape
    assert dm.shape == ang.shape and q.shape == ang.shape and dg.shape == ang.shape
    dxc = _rows(dx, ny) if dxc is None else _rows(dxc, ny)
    dyc = _rows(dy, ny) if dyc is None else _rows(dyc, ny)
    out = np.empty((ny, nx), np.float32)
    oc, orow, nout = _outlet_args(outlets)
    check(lib().td_dinfconclimaccum_host(_ptr(ang), _ptr(dm), _ptr(q), _ptr(dg), _ptr(out), nx, ny, np.float32(nodata), np.float32(dm_nodata), np.float32(q_nodata),
                                         np.float32(csol), _ptr(dxc), _ptr(dyc), int(contcheck), _ptr(oc), _ptr(orow), nout))
    return out


def dinftranslimaccum_grid(ang, tsup, tc, cs=None, dx=30.0, dy=30.0, nodata=float(MISSINGFLOAT), tsup_nodata=-9999.0, tc_nodata=-9999.0, cs_nodata=-9999.0,
                           contcheck=True, outlets=None, dxc=None, dyc=None):
    """Transport limited accumulation on the D-infinity flow field (td_dinftranslimaccum_host; src/DinfTransLimAccum.cpp:237-302):
    returns (tla, tdep, ctpt) — ctpt is None without a supply concentration grid `cs`.  nodata = -FLT_MAX."""
    ang = _grid(ang, np.float32); tsup = _grid(tsup, np.float32); tc = _grid(tc, np.float32)
    ny, nx = ang.shape
    assert tsup.shape == ang.shape and tc.shape == ang.shape
    c = None if cs is None else _grid(cs, np.float32)
    dxc = _rows(dx, ny) if dxc is None else _rows(dxc, ny)
    dyc = _rows(dy, ny) if dyc is None else _rows(dyc, ny)
    tla = np.empty((ny, nx), np.float32); dep = np.empty((ny, nx), np.float32)
    cout = None if cs is None else np.empty((ny, nx), np.float32)
    oc, orow, nout = _outlet_args(outlets)
    check(lib().td_dinftranslimaccum_host(_ptr(ang), _ptr(tsup), _ptr(tc), _ptr(c), _ptr(tla), _ptr(dep), _ptr(cout), nx, ny, np.float32(nodata),
                                          np.float32(tsup_nodata), np.float32(tc_nodata), np.float32(cs_nodata), _ptr(dxc), _ptr(dyc), int(contcheck),
                                          _ptr(oc), _ptr(orow), nout))
    return tla, dep, cout


def threshold_grid(ssa, thresh=100.0, mask=None, nodata=-1.0):
    """src = (ssa >= thresh [& mask >= 0]) ? 1 : 0, -32768 where ssa is nodata (td_threshold_host; src/Threshold.cpp:109-131)."""
    ssa = _grid(ssa, np.float32)
    ny, nx = ssa.shape
    m = None if mask is None else _grid(mask, np.float32)
    src = np.empty((ny, nx), np.int16)
    check(lib().td_threshold_host(_ptr(ssa), _ptr(m), _ptr(src), nx, ny, np.float32(thresh), np.float32(nodata)))
    return src


def twi_grid(slp, sca, slp_nodata=-1.0, sca_nodata=-1.0):
    """twi = ln(sca / slp) where both are data and positive, else -1 (td_twi_host; src/TWI.cpp:108-124)."""
    slp = _grid(slp, np.float32); sca = _grid(sca, np.float32)
    ny, nx = slp.shape
    assert sca.shape == slp.shape
    twi = np.empty((ny, nx), np.float32)
    check(lib().td_twi_host(_ptr(slp), _ptr(sca), _ptr(twi), nx, ny, np.float32(slp_nodata), np.float32(sca_nodata)))
    return twi


def slopearea_grid(slp, sca, m=2.0, n=1.0):
    """sa = slp^m * sca^n where slp >= 0 and sca >= 0, else -1 (td_slopearea_host; src/SlopeArea.cpp:114-125)."""
    slp = _grid(slp, np.float32); sca = _grid(sca, np.float32)
    ny, nx = slp.shape
    assert sca.shape == slp.shape
    sa = np.empty((ny, nx), np.float32)
    check(lib().td_slopearea_host(_ptr(slp), _ptr(sca), _ptr(sa), nx, ny, np.float32(m), np.float32(n)))
    return sa


def slopearearatio_grid(slp, sca, sca_nodata=-1.0):
    """sar = slp / sca where sca is data, else -1 (td_slopearearatio_host; src/SlopeAreaRatio.cpp:107-118)."""
    slp = _grid(slp, np.float32); sca = _grid(sca, np.float32)
    ny, nx = slp.shape
    assert sca.shape == slp.shape
    sar = np.empty((ny, nx), np.float32)
    check(lib().td_slopearearatio_host(_ptr(slp), _ptr(sca), _ptr(sar), nx, ny, np.float32(sca_nodata)))
    return sar


def peukerdouglas_grid(fel, weights=(0.4, 0.1, 0.05), nodata=-3.0e38):
    """Peuker-Douglas stream sources (td_peukerdouglas_host; src/PeukerDouglas.cpp:109-212): the elevations smoothed with the centre,
    side and diagonal weights, then 1 on every cell that is not the highest of any group of four cells around it (and not on the
    grid's edge, not nodata, not next to nodata), else 0.  int16, 0 / 1 everywhere (the file's nodata tag is -2)."""
    fel = _grid(fel, np.float32)
    ny, nx = fel.shape
    w = np.ascontiguousarray(weights, np.float32)
    if w.shape != (3,):
        raise ValueError("peukerdouglas_grid: three weights (middle, side, diagonal)")
    ss = np.empty((ny, nx), np.int16)
    check(lib().td_peukerdouglas_host(_ptr(fel), _ptr(ss), nx, ny, np.float32(nodata), _ptr(w)))
    return ss


def lengtharea_grid(plen, ad8, m=0.03, y=1.3):
    """Length-area stream sources (td_lengtharea_host; src/LengthArea.cpp:110-120): 1 where ad8 >= m * plen^y, else 0, and -32768
    where plen < 0.  ad8 must be int32 (the reference reads the contributing area as 32-bit integers, rounding half away from zero:
    read_raster(path, np.int32) does the same)."""
    plen = _grid(plen, np.float32)
    a = np.asarray(ad8)
    if a.dtype != np.int32:
        raise TypeError(f"lengtharea_grid: ad8 must be int32, not {a.dtype}")
    a = np.ascontiguousarray(a)
    ny, nx = plen.shape
    if a.shape != plen.shape:
        raise ValueError("lengtharea_grid: plen and ad8 differ in shape")
    ss = np.empty((ny, nx), np.int16)
    check(lib().td_lengtharea_host(_ptr(plen), _ptr(a), _ptr(ss), nx, ny, np.float32(m), np.float32(y)))
    return ss


def slopeavedown_grid(fel, p, dn=50.0, dx=30.0, dy=30.0, nodata=float(FEL_NODATA), p_nodata=int(MISSINGSHORT), dxc=None, dyc=None):
    """D8 slope averaged over the downslope distance dn (td_slopeavedown_host; src/SlopeAveDown.cpp:59-330): for every cell the
    aread8 queue reaches, (fel - the elevation at the end of its flow path dn further down) / that path's length, float32, nodata
    MISSINGFLOAT.  dx / dy: the header's cell sizes, from which the pass count dn / min(dx, dy) + 1 comes; dxc / dyc: per-row cell
    sizes for the distances (default dx / dy on every row)."""
    fel = _grid(fel, np.float32)
    p = _grid(p, np.int16)
    ny, nx = fel.shape
    if p.shape != fel.shape:
        raise ValueError("slopeavedown_grid: fel and p differ in shape")
    dxc = _rows(dx if dxc is None else dxc, ny)
    dyc = _rows(dy if dyc is None else dyc, ny)
    slpd = np.empty((ny, nx), np.float32)
    check(lib().td_slopeavedown_host(_ptr(fel), _ptr(p), _ptr(slpd), nx, ny, np.float32(nodata), int(p_nodata), _ptr(dxc), _ptr(dyc), float(dx),
                                     float(dy), float(dn)))
    return slpd


def _stream_args(p, src, what):
    p = _grid(p, np.int16)
    src = _grid(src, np.int32)
    if src.shape != p.shape:
        raise ValueError(f"{what}: p and src differ in shape")
    return p, src


def d8hdisttostrm_grid(p, src, thresh=1, dx=30.0, dy=30.0, p_nodata=int(MISSINGSHORT), src_nodata=-2147483648, dxc=None, dyc=None):
    """D8 horizontal distance down to the stream (td_d8hdisttostrm_host; src/D8HDistToStrm.cpp:57-226): the length of every cell's D8
    path to the first stream cell (src >= thresh where src, read as int32, is not src_nodata), float32, 0 on the stream, nodata
    MISSINGFLOAT where the path never reaches one.  dxc / dyc: per-row cell sizes (default dx / dy on every row)."""
    p, src = _stream_args(p, src, "d8hdisttostrm_grid")
    ny, nx = p.shape
    dxc = _rows(dx if dxc is None else dxc, ny)
    dyc = _rows(dy if dyc is None else dyc, ny)
    dist = np.empty((ny, nx), np.float32)
    check(lib().td_d8hdisttostrm_host(_ptr(p), _ptr(src), _ptr(dist), nx, ny, int(p_nodata), int(src_nodata), int(thresh), _ptr(dxc), _ptr(dyc)))
    return dist


def d8vdisttostrm_grid(p, fel, src, thresh=1, p_nodata=int(MISSINGSHORT), src_nodata=-2147483648):
    """D8 vertical distance down to the stream, the height above the nearest drainage (td_d8vdisttostrm_host;
    src/D8VDistToStrm.cpp:58-240): fel minus the elevation of the first stream cell down every cell's D8 path, summed step by step in
    float32 as the reference does, 0 on the stream, nodata MISSINGFLOAT where the path never reaches one.  fel's nodata is not
    tested: its values go through the arithmetic."""
    p, src = _stream_args(p, src, "d8vdisttostrm_grid")
    fel = _grid(fel, np.float32)
    if fel.shape != p.shape:
        raise ValueError("d8vdisttostrm_grid: p and fel differ in shape")
    ny, nx = p.shape
    dist = np.empty((ny, nx), np.float32)
    check(lib().td_d8vdisttostrm_host(_ptr(p), _ptr(fel), _ptr(src), _ptr(dist), nx, ny, int(p_nodata), int(src_nodata), int(thresh)))
    return dist


_DDD_METHODS = {"h": 0, "v": 1, "p": 2, "s": 3}
_DDD_STATS = {"ave": 0, "max": 1, "min": 2}


def dinfdistdown_grid(ang, src, fel=None, weights=None, method="h", stat="ave", contcheck=True, dx=30.0, dy=30.0, dxc=None, dyc=None,
                      ang_nodata=float(MISSINGFLOAT), fel_nodata=float(FEL_NODATA), w_nodata=float(MISSINGFLOAT)):
    """D-infinity distance down to the stream (td_dinfdistdown_host; src/DinfDistDown.cpp:66-1398): for every cell the average,
    maximum or minimum (`stat`) over its D-infinity flow of the horizontal (`method` "h"), vertical ("v": the height above the
    nearest drainage), Pythagoras ("p") or surface ("s") distance to the first stream cell, float32, 0 on the stream, nodata
    MISSINGFLOAT.  Stream cells: src >= 1, src read as int16 (integers outside int16 saturate, as the reference's reader narrows
    them).  fel: needed by v, p and s; weights: multiply the horizontal step (h, p, s).  contcheck: a receiver that is off the grid
    or nodata (or whose fel or weight is nodata) makes the cell nodata.  dxc / dyc: ang's per-row cell sizes (default dx / dy)."""
    if method not in _DDD_METHODS or stat not in _DDD_STATS:
        raise ValueError(f"dinfdistdown_grid: method is one of {sorted(_DDD_METHODS)}, stat one of {sorted(_DDD_STATS)}")
    ang = _grid(ang, np.float32)
    s = np.asarray(src)
    if s.dtype.kind in "iu":
        s = np.clip(s, -32768, 32767)
    src = _grid(s, np.int16)
    if src.shape != ang.shape:
        raise ValueError("dinfdistdown_grid: ang and src differ in shape")
    if method != "h":
        if fel is None:
            raise ValueError(f"dinfdistdown_grid: method {method} needs fel")
        fel = _grid(fel, np.float32)
        if fel.shape != ang.shape:
            raise ValueError("dinfdistdown_grid: ang and fel differ in shape")
    else:
        fel = None
    if weights is not None and method != "v":
        weights = _grid(weights, np.float32)
        if weights.shape != ang.shape:
            raise ValueError("dinfdistdown_grid: ang and weights differ in shape")
    else:
        weights = None
    ny, nx = ang.shape
    dxc = _rows(dx if dxc is None else dxc, ny)
    dyc = _rows(dy if dyc is None else dyc, ny)
    dd = np.empty((ny, nx), np.float32)
    check(lib().td_dinfdistdown_host(_ptr(ang), _ptr(fel), _ptr(weights), _ptr(src), _ptr(dd), nx, ny, float(ang_nodata), float(fel_nodata),
                                     float(w_nodata), _ptr(dxc), _ptr(dyc), _DDD_STATS[stat], _DDD_METHODS[method], int(bool(contcheck))))
    return dd


def flowdircond_grid(p, z, p_nodata=int(MISSINGSHORT), nodata=-9999.0):
    """D8-conditioned elevations (td_flowdircond_host; src/flowdircond.cpp:143-194): every cell the aread8 queue of `p` reaches gets
    the smallest conditioned elevation among the cells that drain into it, or its own z if that is smaller, so that elevations never
    rise downstream along `p`; every other cell keeps its z.  A cell whose z is nodata (within 1e-5 of `nodata`) keeps it.  float32,
    the nodata value of z."""
    p = _grid(p, np.int16)
    z = _grid(z, np.float32)
    ny, nx = z.shape
    if p.shape != z.shape:
        raise ValueError("flowdircond_grid: p and z differ in shape")
    zfdc = np.empty((ny, nx), np.float32)
    check(lib().td_flowdircond_host(_ptr(p), _ptr(z), _ptr(zfdc), nx, ny, int(p_nodata), np.float32(nodata)))
    return zfdc


def retlimflow_grid(ang, wg, rc, dx=30.0, dy=30.0, ang_nodata=float(MISSINGFLOAT), wg_nodata=-9999.0, rc_nodata=-9999.0, dxc=None, dyc=None):
    """D-infinity retention-limited runoff (td_retlimflow_host; src/RetlimFlow.cpp:147-200): qrl = max(0, sum of p * qrl of the
    contributors + wg - rc) in float.  A cell whose wg or rc is nodata gets nodata and passes nothing on.  float32, nodata
    MISSINGFLOAT.  dxc / dyc: per-row cell sizes (default dx / dy on every row).  An angle nodata value that prop() reads as a
    direction raises TaudemError (code 1)."""
    ang = _grid(ang, np.float32)
    wg = _grid(wg, np.float32)
    rc = _grid(rc, np.float32)
    ny, nx = ang.shape
    if wg.shape != ang.shape or rc.shape != ang.shape:
        raise ValueError("retlimflow_grid: ang, wg and rc differ in shape")
    dxc = _rows(dx if dxc is None else dxc, ny)
    dyc = _rows(dy if dyc is None else dyc, ny)
    qrl = np.empty((ny, nx), np.float32)
    check(lib().td_retlimflow_host(_ptr(ang), _ptr(wg), _ptr(rc), _ptr(qrl), nx, ny, np.float32(ang_nodata), np.float32(wg_nodata), np.float32(rc_nodata),
                                   _ptr(dxc), _ptr(dyc)))
    return qrl


def contributing_areas_grid(p, ang, p_nodata=int(MISSINGSHORT), ang_nodata=float(MISSINGFLOAT), dx=30.0, dy=30.0, contcheck=True, out_ad8=None, out_sca=None):
    """aread8 + areadinf of one DEM in one call, copies overlapped with the kernels (td_contributing_areas_host)."""
    p = _grid(p, np.int16); ang = _grid(ang, np.float32)
    ny, nx = p.shape
    assert ang.shape == p.shape
    ad8 = out_ad8 if out_ad8 is not None else np.empty((ny, nx), np.float32)
    sca = out_sca if out_sca is not None else np.empty((ny, nx), np.float32)
    dxc, dyc = _rows(dx, ny), _rows(dy, ny)
    check(lib().td_contributing_areas_host(_ptr(p), _ptr(ang), _ptr(ad8), _ptr(sca), nx, ny, int(p_nodata), np.float32(ang_nodata), _ptr(dxc), _ptr(dyc), int(contcheck)))
    return ad8, sca


def areadinf_grid(ang, nodata=float(MISSINGFLOAT), weights=None, w_nodata=-9999.0, dx=30.0, dy=30.0, contcheck=True, out=None, outlets=None):
    ang = _grid(ang, np.float32)
    ny, nx = ang.shape
    sca = out if out is not None else np.empty((ny, nx), np.float32)
    w = None if weights is None else _grid(weights, np.float32)
    dxc, dyc = _rows(dx, ny), _rows(dy, ny)
    oc, orow, nout = _outlet_args(outlets)
    check(lib().td_area_outlets_host(_ptr(ang), _ptr(w), _ptr(sca), nx, ny, np.float32(nodata), np.float32(w_nodata), _ptr(dxc), _ptr(dyc),
                                     int(contcheck), _ptr(oc), _ptr(orow), nout))
    return sca
