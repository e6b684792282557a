"""d8hdisttostrm's and d8vdisttostrm's test inputs and the reference's outputs on them.

Cases: (name, p, fel, src, thresh, dx, dy, ranks), each run through both tools, covering: rough DEMs with src = the D8 contributing
area at a low and a high threshold; stream cells whose p is nodata; chains of stream cells; a threshold above every src (all
nodata); src nodata holes; codes 0, 9, -1, 10 and nodata away from the queue and on it, 2- and 4-cycles; rivers that leave the grid
on every edge; oblong cells; fel with -FLT_MAX holes, NaN, +0 / -0 and a stream cell at -FLT_MAX; a spiral whose one path to its one
stream cell is far longer than one batch of BFS levels; a column serpentine whose path crosses every row boundary once per column;
and a real DEM at 1 and 3 ranks.

tests/golden/disttostrm_reference.json stores a digest of each reference output, keyed like tests/reference.py's.  `RefPipeline`
replays: the distances are recomputed by the C restatement (oracle/port/disttostrm_oracle.c), pitremove, d8flowdir and aread8 of
the workflow by oracle/port and threshold by tests/pointwise_cases.py, and each result must match its stored digest bit for bit.
TD_RECORD_REFERENCE=<file> with oracle/_ref built (make -C oracle ref && make -C oracle -f stream.mk && make -C oracle -f
disttostrm.mk ref) runs the reference's tools instead, requires the restatements to reproduce them, and writes this module's
digests to <file> at exit."""
import atexit
import json
import os

import numpy as np

import disttostrm_port
import pointwise_cases
import port
import reference
import refrun
from taudem_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "disttostrm_reference.json")
MISSINGFLOAT = np.float32(-3.4028234663852886e38)
P_ND = np.int16(-32768)
SRC_ND = np.int32(-1)
TOOLS = ("d8hdisttostrm", "d8vdisttostrm")
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
    return all(os.access(os.path.join(refrun.REF, t), os.X_OK) for t in TOOLS)


def _save():
    if _recorded:
        with open(reference.RECORD, "w") as f:
            f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, separators=(',', ':'))}" for k, v in sorted(_recorded.items())) + "\n}\n")


if reference.RECORD:
    atexit.register(_save)


# ---------------------------------------------------------------------------------------------------------------- inputs
def flow(ny, nx, seed, hurst=0.7, tilt=1.0):
    """(fel, p, src) of a synthetic DEM by the C restatement: pitremove, d8flowdir, and src = the D8 contributing area (int32)"""
    dem = synth.gen_dem(ny, nx, hurst=hurst, tilt=tilt, seed=seed)
    fel = port.pitremove(dem).astype(np.float32)
    p, _ = port.d8flowdir(fel)
    ad8 = port.aread8(p)
    src = np.where(ad8 < 0, SRC_ND, np.round(ad8)).astype(np.int32)
    return fel, p.astype(np.int16), src


def junk_codes(p, seed, frac=0.15):
    """codes 0, 9, -1, 10, -3, 12 and nodata, 2-cycles, 4-cycles"""
    rng = np.random.default_rng(seed)
    p = p.copy()
    ny, nx = p.shape
    m = rng.random(p.shape) < frac
    p[m] = rng.choice(np.array([0, 9, -1, 10, -3, 12, 1, 5, 3, 7], np.int16), m.sum())
    p[rng.random(p.shape) < 0.03] = P_ND
    for j in range(2, ny - 2, 7):                 # 2-cycles: E <-> W
        p[j, 3], p[j, 4] = 1, 5
    for j in range(4, ny - 3, 9):                 # 4-cycles: E, S, W, N
        i = nx // 2
        p[j, i], p[j, i + 1], p[j + 1, i + 1], p[j + 1, i] = 1, 7, 5, 3
    return p


def edge_rivers(p):
    p = p.copy()
    p[0, :] = 3; p[-1, :] = 7; p[:, 0] = 5; p[:, -1] = 1
    p[0, 0], p[0, -1], p[-1, 0], p[-1, -1] = 4, 2, 6, 8
    return p


_STEP = {(0, 1): 1, (-1, 1): 2, (-1, 0): 3, (-1, -1): 4, (0, -1): 5, (1, -1): 6, (1, 0): 7, (1, 1): 8}   # (drow, dcol) -> code


def path_grid(cells, shape):
    """p where every cell of `cells` drains to the next; the last one is the one stream cell (src 1, elsewhere 0)"""
    p = np.full(shape, P_ND, np.int16)
    src = np.zeros(shape, np.int32)
    for (r0, c0), (r1, c1) in zip(cells[:-1], cells[1:]):
        p[r0, c0] = _STEP[(r1 - r0, c1 - c0)]
    r, c = cells[-1]
    p[r, c] = 0
    src[r, c] = 1
    return p, src


def spiral(ny, nx):
    """clockwise from the north-west corner inwards: one path through every cell"""
    cells, top, bot, lef, rig = [], 0, ny - 1, 0, nx - 1
    while top <= bot and lef <= rig:
        cells += [(top, c) for c in range(lef, rig + 1)]
        cells += [(r, rig) for r in range(top + 1, bot + 1)]
        if top < bot:
            cells += [(bot, c) for c in range(rig - 1, lef - 1, -1)]
        if lef < rig:
            cells += [(r, lef) for r in range(bot - 1, top, -1)]
        top, bot, lef, rig = top + 1, bot - 1, lef + 1, rig - 1
    return path_grid(cells, (ny, nx))


def serpentine(ny, nx):
    """down column 0, up column 1, ...: a path that crosses every row boundary once per column"""
    cells = []
    for c in range(nx):
        cells += [(r, c) for r in (range(ny) if c % 2 == 0 else range(ny - 1, -1, -1))]
    return path_grid(cells, (ny, nx))


def ramp(shape, seed):
    rng = np.random.default_rng(seed)
    return (np.arange(shape[0] * shape[1]).reshape(shape) * 0.37 + rng.random(shape) * 3).astype(np.float32)


def cases():
    """(name, p, fel, src, thresh, dx, dy, ranks) of every recorded reference call (each through both tools)"""
    out = []
    fel, p, src = flow(29, 37, 1)
    big_fel, big_p, big_src = flow(70, 261, 2)
    for t in (1, 5, 40, 10 ** 6):                 # 1: every cell with an area is a stream cell; 10**6: none is
        out.append((f"rough thresh={t}", p, fel, src, t, 30.0, 30.0, 1))
    s2 = src.copy(); p2 = p.copy()
    st = s2 >= 20
    p2[st & (np.random.default_rng(3).random(p.shape) < 0.3)] = P_ND          # stream cells whose p is nodata
    out.append(("stream p nodata", p2, fel, s2, 20, 30.0, 30.0, 1))
    s3 = src.copy()
    s3[np.random.default_rng(4).random(p.shape) < 0.08] = SRC_ND               # src nodata holes
    out.append(("src holes", p, fel, s3, 20, 30.0, 30.0, 1))
    out.append(("junk codes", junk_codes(p, 5), fel, src, 20, 30.0, 30.0, 1))
    out.append(("edge rivers", edge_rivers(p), fel, src, 60, 30.0, 30.0, 1))
    out.append(("oblong", p, fel, src, 20, 10.0, 7.0, 1))
    f4 = fel.copy()
    f4[3:26:4, 5:33:6] = MISSINGFLOAT
    f4[2:27:5, 2:35:7] = np.nan
    f4[1::6, 1::9] = 0.0
    f4[4::6, 3::9] = -0.0
    f4[src >= 20] = np.where(np.random.default_rng(6).random((src >= 20).sum()) < 0.2, MISSINGFLOAT, f4[src >= 20])
    out.append(("fel float range", p, f4, src, 20, 30.0, 30.0, 1))
    sp, ss = spiral(23, 31)
    out.append(("spiral", sp, ramp(sp.shape, 7), ss, 1, 30.0, 30.0, 1))
    # (the serpentine at one rank only: on several ranks the reference adds an uninitialised border row to the counts of rank 0's
    # first row in every exchange round, which stops this path there; DESIGN.md section 2)
    sv, sr = serpentine(30, 11)
    out.append(("serpentine", sv, ramp(sv.shape, 8), sr, 1, 30.0, 30.0, 1))
    for ranks in (1, 3):
        out.append(("strips", big_p, big_fel, big_src, 30, 30.0, 30.0, ranks))
    return out


def workflow_dem():
    return synth.gen_dem(83, 97, hurst=0.7, tilt=2.0, seed=31)


def large():
    """2000 x 1500: (p, fel, src, thresh)"""
    fel, p, src = flow(2000, 1500, 41, hurst=0.8, tilt=2.0)
    return p, fel, src, 200


# ------------------------------------------------------------------------------------------------------- reference calls
class Files(refrun.RefPipeline):
    """the reference's two tools on arrays, through a scratch directory"""

    def _dist(self, tool, p, src, fel, thresh, p_nodata, src_nodata):
        self.put("pdts.tif", np.asarray(p, np.int16), p_nodata)
        src = np.asarray(src)
        self.put("srcdts.tif", src, src_nodata)
        args = ["-p", self.path("pdts.tif"), "-src", self.path("srcdts.tif"), "-dist", self.path("dts.tif")]
        if fel is not None:
            self.put("feldts.tif", np.asarray(fel, np.float32), float(MISSINGFLOAT))
            args += ["-fel", self.path("feldts.tif")]
        if thresh is not None:
            args += ["-thresh", str(int(thresh))]
        _, self.times[tool] = refrun.run_tool(tool, args, self.np_ranks)
        return self.get("dts.tif", np.float32)

    def d8hdisttostrm(self, p, src, thresh=None, p_nodata=int(P_ND), src_nodata=int(SRC_ND)):
        return self._dist("d8hdisttostrm", p, src, None, thresh, p_nodata, src_nodata)

    def d8vdisttostrm(self, p, fel, src, thresh=None, p_nodata=int(P_ND), src_nodata=int(SRC_ND)):
        return self._dist("d8vdisttostrm", p, src, fel, thresh, p_nodata, src_nodata)


class RefPipeline:
    """both distance tools, and pitremove, d8flowdir, aread8 and threshold of the workflow: the reference tools when recording,
    their stored outputs otherwise"""

    def __init__(self, workdir, dx=30.0, dy=30.0, np_ranks=1):
        if reference.RECORD and not (available() and refrun.available()):
            raise RuntimeError("TD_RECORD_REFERENCE needs oracle/_ref (make -C oracle ref && make -C oracle -f disttostrm.mk ref)")
        refrun.INPUTS_ONLY = not reference.RECORD
        self.files = Files(workdir=workdir, dx=dx, dy=dy, np_ranks=np_ranks)
        self.dx, self.dy, self.np_ranks = dx, dy, np_ranks

    def d8hdisttostrm(self, *args, **kw):
        return self._call("d8hdisttostrm", args, kw)

    def d8vdisttostrm(self, *args, **kw):
        return self._call("d8vdisttostrm", args, kw)

    def pitremove(self, *args, **kw):
        return self._call("pitremove", args, kw)

    def d8flowdir(self, *args, **kw):
        return self._call("d8flowdir", args, kw)

    def aread8(self, *args, **kw):
        return self._call("aread8", args, kw)

    def threshold(self, *args, **kw):
        return self._call("threshold", args, kw)

    def _restate(self, tool, args, kw):
        if tool in TOOLS:
            kw = dict(kw)
            thresh = kw.pop("thresh", None)
            fel = args[1] if tool == "d8vdisttostrm" else None
            src = args[-1]
            return disttostrm_port.disttostrm(args[0], src, fel=fel, thresh=1 if thresh is None else thresh, dx=self.dx, dy=self.dy,
                                              p_nodata=kw.pop("p_nodata", int(P_ND)), src_nodata=kw.pop("src_nodata", int(SRC_ND)))
        if tool == "pitremove":
            return port.pitremove(*args, **kw)
        if tool == "aread8":
            return port.aread8(*args, **kw)
        if tool == "threshold":
            return pointwise_cases.threshold(*args, **kw)
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
    """the reference's (horizontal, vertical) distances of one case on a RefPipeline made with the case's dx, dy and ranks"""
    name, p, fel, src, thresh, dx, dy, ranks = case
    return R.d8hdisttostrm(p, src, thresh=thresh), R.d8vdisttostrm(p, fel, src, thresh=thresh)


def pipeline(tmp, case):
    name, p, fel, src, thresh, dx, dy, ranks = case
    return RefPipeline(workdir=str(tmp), dx=dx, dy=dy, np_ranks=ranks)


def workflow(R, dem, thresh=30.0):
    """pitremove -> d8flowdir -> aread8 -> threshold -> d8hdisttostrm / d8vdisttostrm on a RefPipeline: (fel, p, ad8, src, h, v)"""
    fel = R.pitremove(dem)
    p, _ = R.d8flowdir(fel)
    ad8 = R.aread8(p)
    src = R.threshold(ad8, thresh)
    return (fel, p, ad8, src, R.d8hdisttostrm(p, src, src_nodata=-32768), R.d8vdisttostrm(p, fel, src, src_nodata=-32768))
