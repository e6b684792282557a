"""flowdircond's and retlimflow's test inputs and the reference's outputs on them.

Cases: (name, p, p nodata, z, z nodata, ranks).  The directions mostly disagree with z, because conditioning changes nothing when p
was derived from the same filled DEM: p of a burned DEM applied to the raw DEM with its pits, p of another DEM altogether, random
direction fields with 2- and 4-cycles, code 0 and codes outside 0..8 (tests/slopeavedown_reference.junk_codes), nodata holes in z
only, in p only and in both, z nodata -FLT_MAX and -9999, a nodata value that cells lie within 1e-5 of, +-0 and NaN elevations,
rivers that leave the grid on every edge, and a grid whose rivers cross tiles and (at 3 ranks) row strips.

retlimflow cases: (name, ang, ang nodata, wg, wg nodata, rc, rc nodata, dx, dy, ranks): angles of a filled DEM and of the rivers of
tests/dinf_fields.river_comb, wg / rc nodata holes whose blocked downstream closures cross tiles and (at 3 ranks) row strips, rc
larger than the inflow (the clip at 0), NaN wg, the angle torture of tests/util.py (shares near 1e-5, the wrap sector) and oblong
cells.

tests/golden/conditioning_reference.json stores a digest of each reference output, keyed like tests/reference.py's.
`RefPipeline` replays: flowdircond and retlimflow are recomputed by the C restatements (oracle/port/conditioning_oracle.c), pitremove and d8flowdir
of the workflow by oracle/port, and each result must match its stored digest bit for bit.
TD_RECORD_REFERENCE=<file> with oracle/_ref built (make -C oracle ref && make -C oracle -f conditioning.mk ref) runs the
reference's tools instead, requires the restatements to reproduce them, and writes this module's digests to <file> at exit."""
import atexit
import json
import os

import numpy as np

import conditioning_port
import port
import reference
import refrun
from slopeavedown_reference import edge_rivers, holes, junk_codes
from taudem_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conditioning_reference.json")
MISSINGFLOAT = np.float32(-3.4028234663852886e38)
Z_ND = np.float32(-9999.0)
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
    return os.access(os.path.join(refrun.REF, "flowdircond"), os.X_OK)


def _save():
    if _recorded:
        with open(reference.RECORD, "w") as f:
            f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, separators=(',', ':'))}" for k, v in sorted(_recorded.items())) + "\n}\n")


if reference.RECORD:
    atexit.register(_save)


# ---------------------------------------------------------------------------------------------------------------- inputs
def burned(ny, nx, seed, depth=40.0):
    """(raw dem, p): p is d8flowdir of the filled DEM with a meandering channel burned `depth` deep, so it disagrees with the raw DEM
    (its pits, and cells the channel makes drain uphill)"""
    dem = synth.gen_dem(ny, nx, hurst=0.7, tilt=1.0, seed=seed)
    rng = np.random.default_rng(seed)
    b = dem.copy()
    c = nx // 2
    for j in range(ny):
        c = int(np.clip(c + rng.integers(-1, 2), 1, nx - 2))
        b[j, c] -= depth
    fel = port.pitremove(b)
    p, _ = port.d8flowdir(fel)
    return dem.astype(np.float32), p.astype(np.int16)


def other_p(ny, nx, seed):
    """p of an unrelated DEM"""
    fel = port.pitremove(synth.gen_dem(ny, nx, hurst=0.8, tilt=2.0, seed=seed + 1000))
    p, _ = port.d8flowdir(fel)
    return p.astype(np.int16)


def random_p(ny, nx, seed):
    """a random direction field: codes 1..8 everywhere, then tests/slopeavedown_reference.junk_codes on top"""
    rng = np.random.default_rng(seed)
    return junk_codes(rng.integers(1, 9, (ny, nx)).astype(np.int16), seed + 1, 0.2)


def signed_zeros_nan(z, seed):
    """+0, -0 and NaN elevations scattered over z (next to each other too)"""
    z = z.copy()
    rng = np.random.default_rng(seed)
    r = rng.random(z.shape)
    z[r < 0.05] = 0.0
    z[(r >= 0.05) & (r < 0.1)] = -0.0
    z[(r >= 0.1) & (r < 0.13)] = np.nan
    z[2, 2:8] = [0.0, -0.0, np.nan, -0.0, 0.0, np.nan]
    return z


def near_nodata(z, nd, seed):
    """cells at nd + 4e-6, nd - 9e-6 (within 1e-5: nodata) and nd + 2e-5 (not) around a nodata value of 0.25"""
    z = (z - z.min()).astype(np.float32) * np.float32(0.001) + np.float32(0.2)
    rng = np.random.default_rng(seed)
    r = rng.random(z.shape)
    z[r < 0.05] = nd
    z[(r >= 0.05) & (r < 0.1)] = nd + np.float32(4e-6)
    z[(r >= 0.1) & (r < 0.15)] = nd - np.float32(9e-6)
    z[(r >= 0.15) & (r < 0.2)] = nd + np.float32(2e-5)
    return z


def cases():
    """(name, p, p_nodata, z, z_nodata, ranks) of every recorded reference call"""
    out = []
    z, p = burned(29, 37, 1)
    big_z, big_p = burned(70, 261, 2)
    out.append(("burned", p, P_ND, z, Z_ND, 1))
    out.append(("other p", other_p(29, 37, 3), P_ND, z, Z_ND, 1))
    out.append(("random p", random_p(29, 37, 4), P_ND, z, Z_ND, 1))
    out.append(("z holes", p, P_ND, holes(z, Z_ND, 5), Z_ND, 1))
    out.append(("p holes", holes(p, P_ND, 6), P_ND, z, Z_ND, 1))
    out.append(("both holes", holes(random_p(29, 37, 7), P_ND, 8), P_ND, holes(z, Z_ND, 9), Z_ND, 1))
    zf = holes(z, MISSINGFLOAT, 10)
    out.append(("z -FLT_MAX", other_p(29, 37, 11), P_ND, zf, MISSINGFLOAT, 1))
    nd = np.float32(0.25)
    out.append(("near nodata", random_p(29, 37, 12), P_ND, near_nodata(z, nd, 13), nd, 1))
    out.append(("zeros nan", random_p(29, 37, 14), P_ND, signed_zeros_nan(z, 15), Z_ND, 1))
    out.append(("edge rivers", edge_rivers(other_p(29, 37, 16)), P_ND, z, Z_ND, 1))
    # tiles and row strips crossed, at 1 and 3 ranks
    for ranks in (1, 3):
        out.append(("strips", big_p, P_ND, big_z, Z_ND, ranks))
        out.append(("strips other", other_p(70, 261, 17), P_ND, holes(big_z, Z_ND, 18), Z_ND, ranks))
        out.append(("strips random", holes(random_p(70, 261, 19), P_ND, 20), P_ND, signed_zeros_nan(big_z, 21), Z_ND, ranks))
    return out


def rl_inputs(ang, seed, wmax=1.0, rmax=0.5):
    """(wg, rc): uniform in [0, wmax) and [0, rmax)"""
    rng = np.random.default_rng(seed)
    return rng.random(ang.shape).astype(np.float32) * np.float32(wmax), rng.random(ang.shape).astype(np.float32) * np.float32(rmax)


def dinf_angles(ny, nx, seed, dx=30.0, dy=30.0):
    fel = port.pitremove(synth.gen_dem(ny, nx, hurst=0.7, tilt=1.0, seed=seed))
    ang, _ = port.dinfflowdir(fel, dx=dx, dy=dy)
    return ang.astype(np.float32)


def rl_cases():
    """(name, ang, ang_nodata, wg, wg_nodata, rc, rc_nodata, dx, dy, ranks) of every recorded retlimflow call"""
    from dinf_fields import river_comb
    from util import angle_torture
    out = []
    ang = dinf_angles(29, 37, 51)
    wg, rc = rl_inputs(ang, 52)
    out.append(("rl basic", ang, MISSINGFLOAT, wg, Z_ND, rc, Z_ND, 30.0, 30.0, 1))
    wg2, rc2 = rl_inputs(ang, 53, 1.0, 6.0)
    wg2[np.random.default_rng(54).random(ang.shape) < 0.04] = np.nan
    out.append(("rl clip nan", ang, MISSINGFLOAT, wg2, Z_ND, rc2, Z_ND, 30.0, 30.0, 1))
    out.append(("rl wg holes", ang, MISSINGFLOAT, holes(wg, Z_ND, 55), Z_ND, rc, Z_ND, 30.0, 30.0, 1))
    out.append(("rl rc holes", ang, MISSINGFLOAT, wg, Z_ND, holes(rc, np.float32(-1.0), 56), np.float32(-1.0), 30.0, 30.0, 1))
    out.append(("rl all holes", holes(ang, MISSINGFLOAT, 57), MISSINGFLOAT, holes(wg, Z_ND, 58), Z_ND, holes(rc, Z_ND, 59), Z_ND, 30.0, 30.0, 1))
    t = angle_torture(48, 60)
    wt, rt = rl_inputs(t, 60, 1.0, 0.2)
    out.append(("rl torture", t, MISSINGFLOAT, wt, Z_ND, rt, Z_ND, 30.0, 30.0, 1))
    ob = dinf_angles(29, 37, 61, 10.0, 7.0)
    wo, ro = rl_inputs(ob, 62)
    out.append(("rl oblong", ob, MISSINGFLOAT, holes(wo, Z_ND, 63), Z_ND, ro, Z_ND, 10.0, 7.0, 1))
    big = dinf_angles(70, 261, 64)
    wb, rb = rl_inputs(big, 65, 1.0, 0.6)
    comb = river_comb(70, 261, (12, 35, 58), 66)
    wc, rcb = rl_inputs(comb, 67, 1.0, 0.3)
    for ranks in (1, 3):
        out.append(("rl strips", big, MISSINGFLOAT, holes(wb, Z_ND, 68, 0.01), Z_ND, holes(rb, Z_ND, 69, 0.01), Z_ND, 30.0, 30.0, ranks))
        out.append(("rl comb", comb, MISSINGFLOAT, holes(wc, Z_ND, 70, 0.005), Z_ND, rcb, Z_ND, 30.0, 30.0, ranks))
    return out


def rl_large():
    """2000 x 1500 angles of a DEM, wg / rc with sparse nodata holes"""
    ang = dinf_angles(2000, 1500, 71)
    wg, rc = rl_inputs(ang, 72, 1.0, 0.5)
    return ang, holes(wg, Z_ND, 73, 0.0005), rc


def workflow_dem():
    return synth.gen_dem(83, 97, hurst=0.7, tilt=2.0, seed=32)


def large():
    """2000 x 1500: p of a burned DEM on the raw DEM"""
    return burned(2000, 1500, 41)


# ------------------------------------------------------------------------------------------------------- reference calls
class Files(refrun.RefPipeline):
    """the reference's flowdircond on arrays, through a scratch directory"""

    def flowdircond(self, p, z, p_nodata=int(P_ND), z_nodata=float(Z_ND)):
        self.put("pfdc.tif", np.asarray(p, np.int16), p_nodata)
        self.put("zfdcin.tif", np.asarray(z, np.float32), z_nodata)
        args = ["-p", self.path("pfdc.tif"), "-z", self.path("zfdcin.tif"), "-zfdc", self.path("zfdc.tif")]
        _, self.times["flowdircond"] = refrun.run_tool("flowdircond", args, self.np_ranks)
        return self.get("zfdc.tif", np.float32)

    def retlimflow(self, ang, wg, rc, ang_nodata=float(MISSINGFLOAT), wg_nodata=float(Z_ND), rc_nodata=float(Z_ND)):
        self.put("angrl.tif", np.asarray(ang, np.float32), ang_nodata)
        self.put("wgrl.tif", np.asarray(wg, np.float32), wg_nodata)
        self.put("rcrl.tif", np.asarray(rc, np.float32), rc_nodata)
        args = ["-ang", self.path("angrl.tif"), "-wg", self.path("wgrl.tif"), "-rc", self.path("rcrl.tif"), "-qrl", self.path("qrl.tif")]
        _, self.times["retlimflow"] = refrun.run_tool("retlimflow", args, self.np_ranks)
        return self.get("qrl.tif", np.float32)


class RefPipeline:
    """flowdircond, pitremove and d8flowdir: the reference tools when recording, their stored outputs otherwise"""

    def __init__(self, workdir, dx=30.0, dy=30.0, np_ranks=1):
        if reference.RECORD and not (available() and refrun.available()):
            raise RuntimeError("TD_RECORD_REFERENCE needs oracle/_ref (make -C oracle ref && make -C oracle -f conditioning.mk ref)")
        refrun.INPUTS_ONLY = not reference.RECORD
        self.files = Files(workdir=workdir, dx=dx, dy=dy, np_ranks=np_ranks)
        self.dx, self.dy, self.np_ranks = dx, dy, np_ranks

    def flowdircond(self, *args, **kw):
        return self._call("flowdircond", args, kw)

    def retlimflow(self, *args, **kw):
        return self._call("retlimflow", args, kw)

    def pitremove(self, *args, **kw):
        return self._call("pitremove", args, kw)

    def d8flowdir(self, *args, **kw):
        return self._call("d8flowdir", args, kw)

    def dinfflowdir(self, *args, **kw):
        return self._call("dinfflowdir", args, kw)

    def _restate(self, tool, args, kw):
        if tool == "flowdircond":
            kw = dict(kw)
            pnd, znd = kw.pop("p_nodata", int(P_ND)), kw.pop("z_nodata", float(Z_ND))
            return conditioning_port.flowdircond(*args, p_nodata=pnd, nodata=znd)
        if tool == "retlimflow":
            kw = dict(kw)
            return conditioning_port.retlimflow(*args, dx=self.dx, dy=self.dy, edge_quirk=self.np_ranks == 1, ang_nodata=kw.pop("ang_nodata", float(MISSINGFLOAT)),
                                                wg_nodata=kw.pop("wg_nodata", float(Z_ND)), rc_nodata=kw.pop("rc_nodata", float(Z_ND)))
        if tool == "pitremove":
            return port.pitremove(*args, **kw)
        if tool == "dinfflowdir":
            return port.dinfflowdir(*args, dx=self.dx, dy=self.dy, **kw)
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
    """the reference's zfdc of one case on a RefPipeline made with the case's ranks"""
    name, p, pnd, z, znd, ranks = case
    return R.flowdircond(p, z, p_nodata=int(pnd), z_nodata=float(znd))


def pipeline(tmp, case):
    return RefPipeline(workdir=str(tmp), np_ranks=case[5])


def rl_reference_case(R, case):
    """the reference's qrl of one retlimflow case on a RefPipeline made with rl_pipeline"""
    name, ang, andv, wg, wnd, rc, rcnd, dx, dy, ranks = case
    return R.retlimflow(ang, wg, rc, ang_nodata=float(andv), wg_nodata=float(wnd), rc_nodata=float(rcnd))


def rl_pipeline(tmp, case):
    return RefPipeline(workdir=str(tmp), dx=case[7], dy=case[8], np_ranks=case[9])


def rl_workflow(R, dem, wg, rc):
    """pitremove -> dinfflowdir -> retlimflow on a RefPipeline: qrl"""
    ang, _ = R.dinfflowdir(R.pitremove(dem))
    return R.retlimflow(ang, wg, rc)


def workflow(R, dem):
    """pitremove -> d8flowdir -> flowdircond of the raw DEM on a RefPipeline: (fel, p, zfdc)"""
    fel = R.pitremove(dem)
    p, _ = R.d8flowdir(fel)
    return fel, p, R.flowdircond(p, dem)
