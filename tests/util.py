import glob
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FEL_ND = -3.0e38
ANG_ND = -3.4028234663852886e38


def golden_cases():
    # (siblings.npz holds the outputs of the nine tools of SURVEY.md 8(f) on the hills_holes case: not a pipeline case of its own)
    return sorted(n for n in (os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "*.npz"))) if n != "siblings")


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype == np.float32:
        return bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))
    return bool(np.array_equal(a, b))


def assert_bits(a, b, what):
    from reference import Digest, digest
    if isinstance(a, Digest) or isinstance(b, Digest):       # a stored reference output (tests/reference.py)
        assert digest(a) == digest(b), f"{what}: differs from the reference's output ({a!r} vs {b!r})"
        return
    if not bits_equal(a, b):
        raise AssertionError(f"{what}: {bits_report(a, b)}")


def ulp_distance(a, b):
    """per cell: how many float32 values lie between a and b (0 where the bits are equal; +0 and -0 are 1 apart)"""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff) - 1, i)
    return np.abs(ordered(a) - ordered(b))


def bits_report(a, b, first=5):
    """what differs between two rasters: the number of differing cells, for floats the largest ulp distance, and the first
    cells as (row, column, got, want)"""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return f"{a.dtype}{a.shape} vs {b.dtype}{b.shape}"
    if a.dtype == np.float32:
        diff = a.view(np.uint32) != b.view(np.uint32)
    else:
        diff = a != b
    bad = np.argwhere(diff)
    msg = f"{len(bad)} of {a.size} cells differ"
    if a.dtype == np.float32 and len(bad):
        msg += f", by up to {int(ulp_distance(a[diff], b[diff]).max())} ulp"
    return msg + f"; first {[(*map(int, i), a[tuple(i)].item(), b[tuple(i)].item()) for i in bad[:first]]}"


def write_geographic_dem(path, dem, lon0=-111.8, lat0=41.9, cell=0.001, nodata=-9999.0):
    """A GeoTIFF in geographic coordinates (GTModelTypeGeoKey = 2) written with libtiff (PIL): the reference
    then derives per-row metric cell sizes on the WGS84 ellipsoid (src/tiffIO.cpp:118-151, 434-445)."""
    from PIL import Image, TiffImagePlugin
    info = TiffImagePlugin.ImageFileDirectory_v2()
    info[33550] = (cell, cell, 0.0)
    info[33922] = (0.0, 0.0, 0.0, lon0, lat0, 0.0)
    info[34735] = (1, 1, 0, 2, 1024, 0, 1, 2, 1025, 0, 1, 1)
    info.tagtype[33550] = 12; info.tagtype[33922] = 12; info.tagtype[34735] = 3
    info[42113] = repr(float(nodata))
    Image.fromarray(np.ascontiguousarray(dem, np.float32)).save(path, tiffinfo=info)


def write_point_shapefile(path, xs, ys, shape_type=1):
    """Minimal ESRI shapefile (.shp + .shx) with Point (1), PointZ (11) or PointM (21) records."""
    import struct
    recs = b""
    offsets = []
    for i, (x, y) in enumerate(zip(xs, ys)):
        content = struct.pack("<idd", shape_type, float(x), float(y))
        if shape_type == 11: content += struct.pack("<dd", 0.0, 0.0)
        if shape_type == 21: content += struct.pack("<d", 0.0)
        offsets.append((50 + len(recs) // 2, len(content) // 2))
        recs += struct.pack(">ii", i + 1, len(content) // 2) + content
    bbox = (min(xs), min(ys), max(xs), max(ys)) if len(xs) else (0.0, 0.0, 0.0, 0.0)
    def header(nwords):
        return struct.pack(">iiiiiii", 9994, 0, 0, 0, 0, 0, nwords) + struct.pack("<ii", 1000, shape_type) + struct.pack("<dddddddd", *bbox, 0, 0, 0, 0)
    open(path, "wb").write(header(50 + len(recs) // 2) + recs)
    open(path[:-4] + ".shx", "wb").write(header(50 + 4 * len(offsets)) + b"".join(struct.pack(">ii", o, l) for o, l in offsets))


def write_point_geojson(path, xs, ys):
    import json
    feats = [{"type": "Feature", "properties": {"id": i + 1}, "geometry": {"type": "Point", "coordinates": [float(x), float(y)]}} for i, (x, y) in enumerate(zip(xs, ys))]
    json.dump({"type": "FeatureCollection", "features": feats}, open(path, "w"))


def angle_torture(ny=96, nx=120, dx=30.0, dy=30.0, seed=5):
    """A D-infinity angle grid made of the values where prop() changes its mind: the eight directions' angles and their float
    neighbours, angles whose share for one direction lies within a few ulps of the 1e-5 threshold on either side (one of the
    two receivers is dropped), the wrap sector below 2 PI, 0, 2 PI, angles beyond 2 PI, flats (-1) and nodata.  Mostly cyclic
    nonsense as a flow field, which is fine: every tool leaves the cells of a cycle unevaluated."""
    import numpy as np
    PI = 3.14159265359
    t = np.arctan2(dy, dx)
    edges = [0.0, t, 0.5 * PI, PI - t, PI, PI + t, 1.5 * PI, 2 * PI - t, 2 * PI]
    vals = []
    for i, e in enumerate(edges):
        f = np.float32(e)
        vals += [f, np.nextafter(f, np.float32(10)), np.nextafter(f, np.float32(-10))]
        if i + 1 < len(edges):
            w = edges[i + 1] - e
            for frac in (1e-5, 1e-5 * (1 + 2e-7), 1e-5 * (1 - 2e-7), 0.999e-5, 1.001e-5, 0.3, 0.5, 0.77, 1e-7, 1e-6, 0.4e-5, 0.449e-5, 0.45e-5, 0.5e-5, 0.6e-5, 2e-5, 3.9e-5, 4.1e-5):
                vals += [np.float32(e + frac * w), np.float32(edges[i + 1] - frac * w)]
    vals += [np.float32(2 * PI + 1e-4), np.float32(6.5), np.float32(1e-30), np.float32(-1.0)]
    vals = np.array(vals, np.float32)
    rng = np.random.default_rng(seed)
    ang = vals[rng.integers(0, len(vals), size=(ny, nx))]
    ang[rng.random((ny, nx)) < 0.02] = np.float32(-3.4028234663852886e38)
    return np.ascontiguousarray(ang, np.float32)
