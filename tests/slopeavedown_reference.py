"""slopeavedown's test inputs and the reference's outputs on them.

Cases: (name, fel, fel nodata, p, p nodata, dx, dy, dn), each run at 1 rank (and the strip cases at 3), covering rough DEMs with
flats, nodata holes in fel only, in p only and in both, direction codes 0, 9, -1, 2-cycles, longer cycles and a code 0 north-west
of a cell (the phantom contributor of initNeighborD8up), rivers that leave the grid on every edge, dn = 0, dn below one cell, dn
equal to an exact path sum (the strict >), dn past the longest path, dn that gives no pass at all, oblong cells, and a DEM whose
nodata is -FLT_MAX with cells whose slope lands on the nodata test.

tests/golden/slopeavedown_reference.json stores a digest of each reference output, keyed like tests/reference.py's.
`RefPipeline` replays: slopeavedown is recomputed by the C restatement (oracle/port/slopeavedown_oracle.c), pitremove and
d8flowdir of the workflow by oracle/port, and each result must match its stored digest bit for bit.
TD_RECORD_REFERENCE=<file> with oracle/_ref built (make -C oracle ref && make -C oracle -f downslope.mk ref) runs the reference's
tools instead, requires the restatements to reproduce them, and writes this module's digests to <file> at exit."""
import atexit
import json
import os

import numpy as np

import downslope_port
import port
import reference
import refrun
from taudem_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "slopeavedown_reference.json")
FEL_ND = np.float32(-3.0e38)
MISSINGFLOAT = np.float32(-3.4028234663852886e38)
P_ND = np.int16(-32768)
_recorded = {}
_stored = None
replayed = {}


def stored():
    global _stored
    if _stored is None:
        with open(GOLDEN) as f:
            _stored = json.load(f)
    return _stored


def available():
    return os.access(os.path.join(refrun.REF, "slopeavedown"), os.X_OK)


def _save():
    if _recorded:
        with open(reference.RECORD, "w") as f:
            f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, separators=(',', ':'))}" for k, v in sorted(_recorded.items())) + "\n}\n")


if reference.RECORD:
    atexit.register(_save)


# ---------------------------------------------------------------------------------------------------------------- inputs
def flow(ny, nx, seed, quant=None, hurst=0.7, tilt=1.0):
    """(fel, p) of a synthetic DEM by the C restatement: pitremove and d8flowdir; quant: round the DEM to that step first (flats)"""
    dem = synth.gen_dem(ny, nx, hurst=hurst, tilt=tilt, seed=seed)
    if quant:
        dem = (np.round(dem / quant) * quant).astype(np.float32)
    fel = port.pitremove(dem)
    p, _ = port.d8flowdir(fel)
    return fel.astype(np.float32), p.astype(np.int16)


def junk_codes(p, seed, frac=0.25):
    """codes 0, 9, -1, 10, a nodata code, 2-cycles, a 4-cycle, and code 0 north-west of cells (phantom contributors)"""
    rng = np.random.default_rng(seed)
    p = p.copy()
    ny, nx = p.shape
    m = rng.random(p.shape) < frac
    p[m] = rng.choice(np.array([0, 9, -1, 10, -2, 1, 5, 3, 7], np.int16), m.sum())
    p[rng.random(p.shape) < 0.03] = P_ND
    for j in range(2, ny - 2, 7):                 # 2-cycles: E <-> W
        p[j, 3], p[j, 4] = 1, 5
    for j in range(4, ny - 3, 9):                 # 4-cycles: E, S, W, N
        i = nx // 2
        p[j, i], p[j, i + 1], p[j + 1, i + 1], p[j + 1, i] = 1, 7, 5, 3
    for j in range(6, ny - 1, 5):                 # code 0 north-west of (j, i)
        p[j - 1, nx - 6] = 0
    return p


def edge_rivers(p):
    """every cell of the rim drains off the grid (N along the top, S along the bottom, W / E along the sides, the corners diagonally)"""
    p = p.copy()
    p[0, :] = 3; p[-1, :] = 7; p[:, 0] = 5; p[:, -1] = 1
    p[0, 0], p[0, -1], p[-1, 0], p[-1, -1] = 4, 2, 6, 8
    return p


def holes(a, nd, seed, frac=0.06):
    a = a.copy()
    rng = np.random.default_rng(seed)
    a[rng.random(a.shape) < frac] = nd
    a[0, 2] = a[-1, 3] = a[4, 0] = a[5, -1] = nd
    return a


def cases():
    """(name, fel, fel_nodata, p, p_nodata, dx, dy, dn, ranks) of every recorded reference call"""
    out = []
    fel, p = flow(29, 37, 1, quant=0.5)
    big_fel, big_p = flow(70, 261, 2)
    for dn in (50.0, 0.0, 10.0, 60.0, 600.0, 5000.0, -10.0):
        out.append((f"rough dn={dn}", fel, FEL_ND, p, P_ND, 30.0, 30.0, dn, 1))
    out.append(("fel holes", holes(fel, FEL_ND, 3), FEL_ND, p, P_ND, 30.0, 30.0, 100.0, 1))
    out.append(("p holes", fel, FEL_ND, holes(p, P_ND, 4), P_ND, 30.0, 30.0, 100.0, 1))
    out.append(("both holes", holes(fel, FEL_ND, 5), FEL_ND, holes(p, P_ND, 6), P_ND, 30.0, 30.0, 100.0, 1))
    out.append(("junk codes", holes(fel, FEL_ND, 7), FEL_ND, junk_codes(p, 8), P_ND, 30.0, 30.0, 120.0, 1))
    out.append(("edge rivers", fel, FEL_ND, edge_rivers(p), P_ND, 30.0, 30.0, 45.0, 1))
    out.append(("oblong", fel, FEL_ND, p, P_ND, 10.0, 7.0, 45.0, 1))
    # DEM nodata -FLT_MAX: a processed cell whose own elevation is the nodata value and that drains north gets (-FLT_MAX - zi) / 1 =
    # -FLT_MAX in its first slope, which tests as nodata, so the next pass computes it again
    f2 = fel.copy()
    f2[3:26:4, 5:33:6] = MISSINGFLOAT
    out.append(("fel -FLT_MAX", f2, MISSINGFLOAT, p, P_ND, 0.5, 1.0, 0.9, 1))
    out.append(("fel -9999", holes(fel, np.float32(-9999.0), 9), np.float32(-9999.0), p, P_ND, 30.0, 30.0, 70.0, 1))
    # strips: tiles and row strips crossed, at 1 and 3 ranks
    for ranks in (1, 3):
        out.append(("strips", big_fel, FEL_ND, big_p, P_ND, 30.0, 30.0, 300.0, ranks))
        out.append(("strips junk", holes(big_fel, FEL_ND, 10), FEL_ND, junk_codes(big_p, 11, 0.1), P_ND, 30.0, 30.0, 600.0, ranks))
    return out


def workflow_dem():
    return synth.gen_dem(83, 97, hurst=0.7, tilt=2.0, seed=31)


def large():
    """2000 x 1500 with dn = 1470 at 30 m: niter = 50"""
    fel, p = flow(2000, 1500, 41, hurst=0.8, tilt=2.0)
    return fel, p, 1470.0


# ------------------------------------------------------------------------------------------------------- reference calls
class Files(refrun.RefPipeline):
    """the reference's slopeavedown on arrays, through a scratch directory"""

    def slopeavedown(self, fel, p, dn=None, fel_nodata=float(FEL_ND), p_nodata=int(P_ND)):
        self.put("felsad.tif", fel, fel_nodata)
        self.put("psad.tif", np.asarray(p, np.int16), p_nodata)
        args = ["-fel", self.path("felsad.tif"), "-p", self.path("psad.tif"), "-slpd", self.path("slpd.tif")]
        if dn is not None:
            args += ["-dn", repr(float(dn))]
        _, self.times["slopeavedown"] = refrun.run_tool("slopeavedown", args, self.np_ranks)
        return self.get("slpd.tif", np.float32)


class RefPipeline:
    """slopeavedown, pitremove and d8flowdir: the reference tools when recording, their stored outputs otherwise"""

    def __init__(self, workdir, dx=30.0, dy=30.0, np_ranks=1):
        if reference.RECORD and not (available() and refrun.available()):
            raise RuntimeError("TD_RECORD_REFERENCE needs oracle/_ref (make -C oracle ref && make -C oracle -f downslope.mk ref)")
        refrun.INPUTS_ONLY = not reference.RECORD
        self.files = Files(workdir=workdir, dx=dx, dy=dy, np_ranks=np_ranks)
        self.dx, self.dy, self.np_ranks = dx, dy, np_ranks

    def slopeavedown(self, *args, **kw):
        return self._call("slopeavedown", args, kw)

    def pitremove(self, *args, **kw):
        return self._call("pitremove", args, kw)

    def d8flowdir(self, *args, **kw):
        return self._call("d8flowdir", args, kw)

    def _restate(self, tool, args, kw):
        if tool == "slopeavedown":
            kw = dict(kw)
            dn = kw.pop("dn", None)
            nd, pnd = kw.pop("fel_nodata", float(FEL_ND)), kw.pop("p_nodata", int(P_ND))
            return downslope_port.slopeavedown(*args, dn=50.0 if dn is None else dn, dx=self.dx, dy=self.dy, nodata=nd, p_nodata=pnd)
        if tool == "pitremove":
            return port.pitremove(*args, **kw)
        return port.d8flowdir(*args, dx=self.dx, dy=self.dy, **kw)

    def _call(self, tool, args, kw):
        key = reference.call_key(tool, self.dx, self.dy, self.np_ranks, args, kw)
        out = getattr(self.files, tool)(*args, **kw)
        many = isinstance(out, tuple)
        if reference.RECORD:
            _recorded[key] = [reference.digest(o) for o in (out if many else (out,))]
            mine = self._restate(tool, args, kw)
            if [reference.digest(m) for m in (mine if many else (mine,))] != _recorded[key]:
                raise AssertionError(f"{tool}: the restatement does not reproduce the reference's output")
            return out
        want = stored().get(key)
        if want is None:
            raise AssertionError(f"{tool}: no stored reference output for these inputs in {GOLDEN} "
                                 "(record it with TD_RECORD_REFERENCE=<file> where oracle/_ref is built)")
        mine = self._restate(tool, args, kw)
        res = mine if many else (mine,)
        assert len(res) == len(want), f"{tool}: {len(res)} outputs, {len(want)} stored"
        for i, (r, h) in enumerate(zip(res, want)):
            assert reference.digest(r) == h, f"{tool}[{i}]: the restatement no longer reproduces the reference's output"
        replayed[key] = tool
        return mine


def reference_case(R, case):
    """the reference's slpd of one case on a RefPipeline made with the case's dx, dy and ranks"""
    name, fel, fnd, p, pnd, dx, dy, dn, ranks = case
    return R.slopeavedown(fel, p, dn=dn, fel_nodata=float(fnd), p_nodata=int(pnd))


def pipeline(tmp, case):
    name, fel, fnd, p, pnd, dx, dy, dn, ranks = case
    return RefPipeline(workdir=str(tmp), dx=dx, dy=dy, np_ranks=ranks)


def workflow(R, dem):
    """pitremove -> d8flowdir -> slopeavedown (dn 50) on a RefPipeline: (fel, p, slpd)"""
    fel = R.pitremove(dem)
    p, _ = R.d8flowdir(fel)
    return fel, p, R.slopeavedown(fel, p)
