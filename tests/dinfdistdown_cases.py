"""dinfdistdown's test inputs, and the reference's own executable run on them through TIFF files (oracle/_ref/dinfdistdown).

Cases: (name, ang, fel, src, w, dx, dy), each run through the 12 method / statistic pairs (with weights where the case has them)
and with and without -nc, covering: rough DEMs through pitremove -> dinfflowdir with src = the D-infinity contributing area at a low
and a high threshold; stream cells whose ang is nodata; receivers whose ang is nodata and receivers off every edge; angles on every
sector boundary and in the wrap sector (receivers 8 and 1); angles below 0, at and above 2 pi and NaN; 2- and 4-cycles of angles;
weights that are negative, zero and nodata; fel with nodata holes, -FLT_MAX, NaN and +-0, and stream cells whose fel is nodata;
src values above 32767 and below -32768 (narrowed to int16 as the reference's reader does); oblong cells; a long D-infinity path
of more than 10 batches of levels; and a serpentine that crosses the rows of a strip split many times."""
import os

import numpy as np

import refrun
from taudem_b200 import synth

MISSINGFLOAT = np.float32(-3.4028234663852886e38)
FEL_ND = np.float32(-3.0e38)
W_ND = np.float32(-1.0)
ANG_ND = MISSINGFLOAT
SRC_ND = np.int32(-32768)
METHODS = ("h", "v", "p", "s")
STATS = ("ave", "max", "min")
TWO_PI = np.float32(2 * np.pi)


def available():
    return os.access(os.path.join(refrun.REF, "dinfdistdown"), os.X_OK)


def _boundaries(rng, shape):
    """angles exactly on the sector boundaries of square cells (k pi / 4 in float) and just beside them"""
    b = (np.arange(9) * (np.pi / 4)).astype(np.float32)
    a = rng.choice(b, shape)
    nudge = rng.integers(-2, 3, shape)
    return np.where(nudge == 0, a, np.nextafter(a, np.where(nudge > 0, np.float32(9), np.float32(-9)))).astype(np.float32)


def random_case(seed, ny=23, nx=31, junk=True):
    """the D-infinity angles of a pit-filled synthetic DEM (oracle/port), a tenth of them replaced by random angles and angles on or
    beside the sector boundaries; with junk, angles below 0, at and above 2 pi, NaN and nodata; random stream cells, src nodata and
    int32 src outside int16; fel holes, -FLT_MAX, NaN and -0; weights of every sign and nodata"""
    import port
    rng = np.random.default_rng(seed)
    fel = port.pitremove(synth.gen_dem(ny, nx, hurst=0.7, tilt=0.5, seed=seed)).astype(np.float32)
    ang = port.dinfflowdir(fel)[0].astype(np.float32)
    m = rng.random(ang.shape) < 0.03
    ang[m] = (rng.random(m.sum()) * 2 * np.pi).astype(np.float32)
    m = rng.random(ang.shape) < 0.06
    ang[m] = _boundaries(rng, ang.shape)[m]
    if junk:
        ang[rng.random(ang.shape) < 0.02] = np.float32(-0.3)
        ang[rng.random(ang.shape) < 0.02] = TWO_PI
        ang[rng.random(ang.shape) < 0.01] = np.float32(7.0)
        ang[rng.random(ang.shape) < 0.01] = np.nan
        ang[rng.random(ang.shape) < 0.03] = ANG_ND
    src = np.where(rng.random(ang.shape) < 0.08, rng.integers(1, 5, ang.shape), 0).astype(np.int32)
    src[rng.random(ang.shape) < 0.02] = 40000
    src[rng.random(ang.shape) < 0.02] = -40000
    src[rng.random(ang.shape) < 0.02] = SRC_ND
    fel[rng.random(ang.shape) < 0.02] = FEL_ND
    fel[rng.random(ang.shape) < 0.01] = MISSINGFLOAT
    fel[rng.random(ang.shape) < 0.02] = np.nan
    fel[rng.random(ang.shape) < 0.02] = np.float32(-0.0)
    w = (rng.random(ang.shape) * 2).astype(np.float32)
    w[rng.random(ang.shape) < 0.05] = np.float32(-0.7)
    w[rng.random(ang.shape) < 0.05] = np.float32(0.0)
    w[rng.random(ang.shape) < 0.05] = W_ND
    return ang, fel, src, w


def cycles():
    """2- and 4-cycles of angles (E <-> W, and N -> W -> S -> E around a square), with cells draining into them and a stream"""
    ny, nx = 9, 12
    ang = np.full((ny, nx), np.float32(np.pi / 2))      # north everywhere: every column drains off the top edge ...
    src = np.zeros((ny, nx), np.int32)
    ang[4, 2], ang[4, 3] = 0.0, np.float32(np.pi)        # a 2-cycle
    ang[5:, 2] = np.float32(np.pi / 2)
    sq = {(4, 7): np.pi, (4, 6): 1.5 * np.pi, (5, 6): 0.0, (5, 7): np.pi / 2}   # a 4-cycle
    for (r, c), a in sq.items():
        ang[r, c] = np.float32(a)
    ang[0, :] = 0.0                                     # ... except the top row, which drains east to a stream cell
    src[0, nx - 1] = 1
    ang[0, nx - 1] = ANG_ND                             # the stream cell's ang is nodata: it never starts the queue
    src[0, nx - 2] = 1
    fel = (np.arange(ny * nx, dtype=np.float32).reshape(ny, nx) * 0.5 + 100).astype(np.float32)
    return ang, fel, src, None


def long_path(n=720):
    """one D-infinity path of n cells (a boustrophedon along the rows, every angle splitting between two directions at the turns) to
    one stream cell: more than 10 batches of 64 levels"""
    nx = 24
    ny = (n + nx - 1) // nx
    ang = np.empty((ny, nx), np.float32)
    for r in range(ny):
        ang[r, :] = 0.0 if r % 2 == 0 else np.float32(np.pi)
        if r % 2 == 0:
            ang[r, nx - 1] = np.float32(1.5 * np.pi)                 # south at the east end
        else:
            ang[r, 0] = np.float32(1.5 * np.pi)                      # south at the west end
    ang[ny - 1, :] = np.float32(0.0) if (ny - 1) % 2 == 0 else np.float32(np.pi)
    src = np.zeros((ny, nx), np.int32)
    src[ny - 1, nx - 1 if (ny - 1) % 2 == 0 else 0] = 1
    fel = np.arange(ny * nx, 0, -1, dtype=np.float32).reshape(ny, nx)
    return ang, fel, src, None


def serpentine(ny=30, nx=16):
    """a column serpentine: down one column, up the next, so the path crosses every row boundary once per column; the angles lean
    a little off the direction so that every step splits with a diagonal neighbour"""
    ang = np.empty((ny, nx), np.float32)
    for c in range(nx):
        ang[:, c] = np.float32(1.5 * np.pi + 0.2) if c % 2 == 0 else np.float32(np.pi / 2 - 0.2)
        ang[ny - 1 if c % 2 == 0 else 0, c] = 0.0
    src = np.zeros((ny, nx), np.int32)
    src[ny - 1 if (nx - 1) % 2 == 0 else 0, nx - 1] = 1
    fel = np.linspace(500, 0, ny * nx, dtype=np.float32).reshape(ny, nx)
    return ang, fel, src, None


class Files(refrun.RefPipeline):
    """the reference's dinfdistdown on arrays, through TIFF files"""

    def dinfdistdown(self, ang, fel, src, w=None, method="h", stat="ave", contcheck=True):
        """src is written as int32: the reference reads it as int16 through its reader's narrowing"""
        self.put("ang.tif", np.asarray(ang, np.float32), ANG_ND)
        self.put("fel.tif", np.asarray(fel if fel is not None else np.zeros_like(ang), np.float32), FEL_ND)
        self.put("src.tif", np.asarray(src, np.int32), SRC_ND)
        args = ["-ang", self.path("ang.tif"), "-fel", self.path("fel.tif"), "-slp", self.path("slp.tif"), "-src", self.path("src.tif"),
                "-dd", self.path("dd.tif"), "-m", stat, method]
        if w is not None:
            self.put("w.tif", np.asarray(w, np.float32), W_ND)
            args += ["-wg", self.path("w.tif")]
        if not contcheck:
            args.append("-nc")
        refrun.run_tool("dinfdistdown", args, self.np_ranks)
        return self.get("dd.tif", np.float32)
