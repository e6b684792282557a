"""The reference tools' outputs that the tests compare against, without the reference tools (oracle/_ref is built only
where the reference sources are).  tests/golden/reference.json stores a digest of each output, keyed by a digest of the
call.  `RefPipeline` has refrun.RefPipeline's interface and writes the same input files; it replays: every tool is recomputed
— pitremove, d8flowdir, dinfflowdir, aread8, areadinf and the five sibling sweep tools (d8flowpathextremeup, gridnet,
dinfdecayaccum, dinfconclimaccum, dinftranslimaccum) by the C restatement (oracle/port), twi, slopearea, threshold and
slopearearatio in numpy with libm's logf / powf — and must match the stored digest bit for bit.  `replayed` collects the keys
of the calls whose outputs were recomputed and matched.
TD_RECORD_REFERENCE=<file> with oracle/_ref built runs the tools instead, requires the recomputed outputs to be theirs too, and
writes the digests to <file> at exit.
"""
import atexit
import ctypes
import ctypes.util
import hashlib
import json
import os
import tempfile

import numpy as np

import port
import refrun

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference.json")
RECORD = os.environ.get("TD_RECORD_REFERENCE")
_recorded = {}
_stored = None
replayed = {}          # call key -> tool, for every call whose recomputed outputs matched the stored digests


class Digest:
    """What the reference returned, by digest (dtype, shape and bytes)."""

    def __init__(self, hexdigest, what):
        self.hexdigest, self.what = hexdigest, what

    def __repr__(self):
        return f"<reference {self.what} {self.hexdigest[:12]}>"


def _sha256(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def digest(a):
    """the stored form: the first 48 bits of the SHA-256 of dtype, shape and bytes"""
    return a.hexdigest if isinstance(a, Digest) else _sha256(a)[:12]


def _arg(v):
    if isinstance(v, np.ndarray):
        return _sha256(v)
    if isinstance(v, str) and os.path.isfile(v):                # an outlets shapefile: its content
        with open(v, "rb") as f:
            return hashlib.sha256(f.read()).hexdigest()
    return repr(v)


def call_key(tool, dx, dy, ranks, args, kw):
    parts = [tool, repr(float(dx)), repr(float(dy)), str(ranks)] + [_arg(a) for a in args] + [f"{k}={_arg(kw[k])}" for k in sorted(kw)]
    return hashlib.sha256("\n".join(parts).encode()).hexdigest()[:12]


def stored():
    global _stored
    if _stored is None:
        with open(GOLDEN) as f:
            _stored = json.load(f)
    return _stored


def _save():
    if _recorded:
        with open(RECORD, "w") as f:           # one call per line
            f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, separators=(',', ':'))}" for k, v in sorted(_recorded.items())) + "\n}\n")


if RECORD:
    atexit.register(_save)


def _outlet_cells(shp, ny, dx, dy):
    """(cols, rows) of a point shapefile on a RefPipeline raster (origin (0, dy * ny)), like the reference's geoToGlobalXY"""
    import taudem_b200 as td
    xs, ys = td.read_outlets(shp)
    return [int(x / dx) for x in xs], [int((dy * ny - y) / dy) for y in ys]


_libm = ctypes.CDLL(ctypes.util.find_library("m"))
for _name in ("logf", "powf"):
    getattr(_libm, _name).restype = ctypes.c_float
_libm.logf.argtypes = [ctypes.c_float]
_libm.powf.argtypes = [ctypes.c_float, ctypes.c_float]
_logf = np.frompyfunc(lambda x: _libm.logf(x), 1, 1)
_powf = np.frompyfunc(lambda x, y: _libm.powf(x, y), 2, 1)


def _twi(slp, sca, nodata=-1.0):
    """TWI: ln(sca / slp) in float where both are data and positive, else nodata (-1)"""
    slp, sca = np.asarray(slp, np.float32), np.asarray(sca, np.float32)
    nd = np.float32(nodata)
    ok = (slp != nd) & (sca != nd) & (slp > 0) & (sca > 0)
    out = np.full(slp.shape, -1.0, np.float32)
    with np.errstate(all="ignore"):
        out[ok] = _logf(sca[ok] / slp[ok]).astype(np.float32)
    return out


def _slopearea(slp, sca, m=None, n=None):
    """SlopeArea: slp^m * sca^n in float (m = 2, n = 1 by default) where both are >= 0, else nodata (-1)"""
    slp, sca = np.asarray(slp, np.float32), np.asarray(sca, np.float32)
    m, n = (np.float32(2.0), np.float32(1.0)) if m is None else (np.float32(m), np.float32(n))
    ok = (slp >= 0) & (sca >= 0)
    out = np.full(slp.shape, -1.0, np.float32)
    out[ok] = (_powf(slp[ok], m).astype(np.float32) * _powf(sca[ok], n).astype(np.float32)).astype(np.float32)
    return out


def _threshold(ssa, thresh, mask=None, nodata=-1.0):
    """Threshold: 1 where ssa >= thresh (and mask >= 0), else 0; MISSINGSHORT where ssa is nodata"""
    ssa = np.asarray(ssa, np.float32)
    ok = (ssa >= np.float32(thresh)) & (True if mask is None else np.asarray(mask, np.float32) >= 0)
    return np.where(np.abs(ssa - np.float32(nodata)) < np.float32(1e-5), np.int16(-32768), ok.astype(np.int16)).astype(np.int16)


def _slopearearatio(slp, sca, nodata=-1.0):
    """SlopeAreaRatio: slp / sca in float where sca is data, else nodata (-1)"""
    slp, sca = np.asarray(slp, np.float32), np.asarray(sca, np.float32)
    with np.errstate(all="ignore"):
        return np.where(np.abs(sca - np.float32(nodata)) < np.float32(1e-5), np.float32(-1.0), slp / sca).astype(np.float32)


class RefPipeline:
    """refrun.RefPipeline's calls: the reference tools when recording, their stored outputs otherwise (module docstring)."""

    TOOLS = ("pitremove", "d8flowdir", "dinfflowdir", "aread8", "areadinf", "d8flowpathextremeup", "gridnet", "dinfdecayaccum",
             "dinfconclimaccum", "dinftranslimaccum", "threshold", "slopearea", "slopearearatio", "twi")

    def __init__(self, workdir=None, dx=30.0, dy=30.0, np_ranks=1):
        if workdir is None:
            self._tmp = tempfile.TemporaryDirectory(prefix="tdref_")
            workdir = self._tmp.name
        if RECORD and not refrun.available():
            raise RuntimeError("TD_RECORD_REFERENCE needs the reference tools in oracle/_ref (make -C oracle ref)")
        refrun.INPUTS_ONLY = not RECORD
        self.files = refrun.RefPipeline(workdir=workdir, dx=dx, dy=dy, np_ranks=np_ranks)
        self.dir, self.dx, self.dy, self.np_ranks = workdir, dx, dy, np_ranks

    def path(self, name):
        return self.files.path(name)

    def __getattr__(self, tool):
        if tool not in self.TOOLS:
            raise AttributeError(tool)
        return lambda *args, **kw: self._call(tool, args, kw)

    def _restate(self, tool, args, kw):
        dx, dy = self.dx, self.dy
        kw = dict(kw)
        if kw.get("outlets") is not None:
            kw["outlets"] = _outlet_cells(kw["outlets"], args[0].shape[0], dx, dy)
        if tool == "pitremove":
            return port.pitremove(*args, **kw)
        if tool in ("d8flowdir", "dinfflowdir"):
            return getattr(port, tool)(*args, dx=dx, dy=dy, **kw)
        if tool == "aread8":
            return port.aread8(*args, **kw)
        if tool == "areadinf":
            kw.pop("w_nodata", None)
            return port.areadinf(*args, dx=dx, dy=dy, **kw)
        if tool == "d8flowpathextremeup":
            kw.pop("sa_nodata", None)                       # the sa values are taken as they are, nodata or not
            return port.d8flowpathextremeup(*args, **kw)
        if tool == "gridnet":
            return port.gridnet(*args, dx=dx, dy=dy, **kw)
        if tool == "dinfdecayaccum":
            kw.pop("w_nodata", None)                        # (likewise the weights)
            return port.dinfdecayaccum(*args, dx=dx, dy=dy, **kw)
        if tool == "dinfconclimaccum":                      # nodata: of dm and q (the angles' is MISSINGFLOAT)
            nd = kw.pop("nodata", -9999.0)
            return port.dinfconclimaccum(*args, dx=dx, dy=dy, dm_nodata=nd, q_nodata=nd, **kw)
        if tool == "dinftranslimaccum":                     # nodata: of tsup, tc and cs
            nd = kw.pop("nodata", -9999.0)
            return port.dinftranslimaccum(*args, dx=dx, dy=dy, tsup_nodata=nd, tc_nodata=nd, cs_nodata=nd, **kw)
        if tool == "twi":
            return _twi(*args, **kw)
        if tool == "slopearea":
            return _slopearea(*args, **kw)
        if tool == "threshold":
            return _threshold(*args, **kw)
        if tool == "slopearearatio":
            return _slopearearatio(*args, **kw)
        raise AssertionError(f"{tool}: no restatement")

    def _call(self, tool, args, kw):
        key = call_key(tool, self.dx, self.dy, self.np_ranks, args, kw)
        out = getattr(self.files, tool)(*args, **kw)          # writes the input files (and runs the tool when recording)
        many = isinstance(out, tuple)
        if RECORD:
            _recorded[key] = [None if o is None else digest(o) for o in (out if many else (out,))]
            mine = self._restate(tool, args, kw)
            if [None if m is None else digest(m) for m in (mine if many else (mine,))] != _recorded[key]:
                raise AssertionError(f"{tool}: the restatement does not reproduce the reference's output")
            return out
        want = stored().get(key)
        if want is None:
            raise AssertionError(f"{tool}: no stored reference output for these inputs in {GOLDEN} "
                                 "(record it with TD_RECORD_REFERENCE=<file> where oracle/_ref is built)")
        mine = self._restate(tool, args, kw)
        res = mine if isinstance(mine, tuple) else (mine,)
        assert len(res) == len(want), f"{tool}: {len(res)} outputs, {len(want)} stored"
        for i, (r, h) in enumerate(zip(res, want)):
            assert (None if r is None else digest(r)) == h, f"{tool}[{i}]: the restatement no longer reproduces the reference's output"
        replayed[key] = tool
        return res if many else res[0]


def run_tool_outputs(tool, args, outputs, dtypes, inputs):
    """refrun.run_tool's output rasters: arrays when recording, Digests when replaying.  inputs: the arrays of its input files."""
    names = [os.path.basename(a) for a in args if a not in outputs]          # file names, not the directories they are in
    key = hashlib.sha256("\n".join([tool] + names + [_sha256(a) for a in inputs]).encode()).hexdigest()[:12]
    if RECORD:
        import taudem_b200 as td
        refrun.run_tool(tool, args)
        res = [td.read_raster(o, dt) for o, dt in zip(outputs, dtypes)]
        _recorded[key] = [digest(r) for r in res]
        return res
    want = stored().get(key)
    if want is None:
        raise AssertionError(f"{tool}: no stored reference output for these inputs in {GOLDEN}")
    return [Digest(w, f"{tool} {os.path.basename(o)}") for w, o in zip(want, outputs)]
