"""dinfdistdown's recorded cases and the reference's outputs on them.

Cases (name, ang, fel, src, w, dx, dy), each through the 12 method / statistic pairs, with and without -nc, and with the case's
weights where it has them (tests/dinfdistdown_cases.py for the shapes): rough DEMs through pitremove -> dinfflowdir with src = the
D-infinity contributing area thresholded low and high; the random grids with junk angles, nodata, int32 src beyond int16, fel holes,
NaN and +-0, weights of every sign; cycles; angles on the sector boundaries; oblong cells; a long path of more than 10 batches of
levels; a serpentine; a 2000 x 1500 grid (ave only); and the HAND chain pitremove -> dinfflowdir -> d8flowdir -> aread8 -> threshold
-> dinfdistdown -m ave v (its inputs computed by the C restatements of those tools, oracle/port).

tests/golden/dinfdistdown_reference.json stores a digest of each reference output (tests/reference.py's digest), keyed by the case,
method, statistic, weights, -nc and cell size.  The replay recomputes every output with the C restatement
(oracle/port/dinfdistdown_oracle.c) and compares digests.  TD_RECORD_REFERENCE=<file> with oracle/_ref built (make -C oracle -f
dinfdistdown.mk ref) runs the reference's executable instead, requires the restatement to reproduce it, and writes the digests to
<file>."""
import json
import os

import numpy as np

import dinfdistdown_cases as DC
import pointwise_cases
import port
import reference
from taudem_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dinfdistdown_reference.json")
EXPECTED = 393          # stored digests
_stored = None


def stored():
    global _stored
    if _stored is None:
        with open(GOLDEN) as f:
            _stored = json.load(f)
    return _stored


def want(key):
    """the reference's output of one recorded call, by digest"""
    return reference.Digest(stored()[key], key)


def rough(ny, nx, seed, thresh):
    """(ang, fel, src) of a synthetic DEM by the C restatement: pitremove, dinfflowdir, src = areadinf >= thresh (int16, nodata -32768)"""
    dem = synth.gen_dem(ny, nx, hurst=0.7, tilt=1.0, seed=seed)
    fel = port.pitremove(dem).astype(np.float32)
    ang, _ = port.dinfflowdir(fel)
    sca = port.areadinf(ang)
    return ang.astype(np.float32), fel, pointwise_cases.threshold(sca, thresh)


def hand_chain(dem, thresh=20.0):
    """pitremove -> dinfflowdir -> d8flowdir -> aread8 -> threshold: (ang, fel, src) for dinfdistdown -m ave v"""
    fel = port.pitremove(dem).astype(np.float32)
    ang, _ = port.dinfflowdir(fel)
    p, _ = port.d8flowdir(fel)
    src = pointwise_cases.threshold(port.aread8(p), thresh)
    return ang.astype(np.float32), fel, src


def hand_dem():
    return synth.gen_dem(83, 97, hurst=0.7, tilt=2.0, seed=31)


def cases():
    """(name, ang, fel, src, w, dx, dy) of every recorded case"""
    out = []
    for t in (3.0, 60.0):
        ang, fel, src = rough(29, 37, 1, t)
        w = np.random.default_rng(2).random(ang.shape).astype(np.float32) + 0.5
        out.append((f"rough thresh={t:g}", ang, fel, src, w, 30.0, 30.0))
    for s in range(2):
        out.append((f"random {s}", *DC.random_case(s), 30.0, 30.0))
    out.append(("oblong", *DC.random_case(3), 10.0, 7.0))
    ang, fel, src, w = DC.random_case(4, junk=False)
    ang = DC._boundaries(np.random.default_rng(9), ang.shape)
    ang[::5, ::3] = np.float32(6.2)                              # the wrap sector: receivers 8 and 1
    out.append(("sector boundaries", ang, fel, src, w, 30.0, 30.0))
    src_nd = src.copy()
    st = src_nd >= 1
    ang2 = ang.copy()
    ang2[st & (np.random.default_rng(10).random(ang.shape) < 0.5)] = DC.ANG_ND  # stream cells whose ang is nodata
    out.append(("stream ang nodata", ang2, fel, src_nd, w, 30.0, 30.0))
    out.append(("cycles", *DC.cycles(), 30.0, 30.0))
    out.append(("long path", *DC.long_path(), 30.0, 30.0))
    out.append(("serpentine", *DC.serpentine(), 30.0, 30.0))
    out.append(("hand", *hand_chain(hand_dem()), None, 30.0, 30.0))
    return out


def large():
    """2000 x 1500: (ang, fel, src)"""
    return rough(2000, 1500, 41, 200.0)


def _key(name, method, stat, usew, cc, dx, dy):
    return f"{name} -m {stat} {method}{' -wg' if usew else ''}{'' if cc else ' -nc'} {dx:g}x{dy:g}"


def runs(with_large=True):
    """(key, (ang, fel, src, w, method, stat, cc, dx, dy)) of every recorded call"""
    for name, ang, fel, src, w, dx, dy in cases():
        for m in DC.METHODS:
            for st in DC.STATS:
                for usew in ((False, True) if w is not None and m != "v" else (False,)):
                    for cc in (True, False):
                        yield _key(name, m, st, usew, cc, dx, dy), (ang, fel, src, w if usew else None, m, st, cc, dx, dy)
    if with_large:
        ang, fel, src = large()
        for m in ("h", "v", "p"):
            yield _key("large", m, "ave", False, True, 30.0, 30.0), (ang, fel, src, None, m, "ave", True, 30.0, 30.0)


def record(path):
    """the reference's outputs of every run, checked against the restatement, into path"""
    import dinfdistdown_port
    out = {}
    for key, (ang, fel, src, w, m, st, cc, dx, dy) in runs():
        ref = DC.Files(dx=dx, dy=dy).dinfdistdown(ang, fel, src, w, m, st, cc)
        mine = dinfdistdown_port.dinfdistdown(ang, src, fel, w, m, st, cc, dx=dx, dy=dy, fel_nodata=DC.FEL_ND, w_nodata=DC.W_ND)
        if reference.digest(ref) != reference.digest(mine):
            raise AssertionError(f"{key}: the restatement does not reproduce the reference's output")
        out[key] = reference.digest(ref)
    with open(path, "w") as f:
        f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v)}" for k, v in sorted(out.items())) + "\n}\n")
    return len(out)


if __name__ == "__main__":
    import sys
    print(record(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("TD_RECORD_REFERENCE", GOLDEN)))
