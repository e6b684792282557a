"""d8hdisttostrm and d8vdisttostrm on the GPU against the reference's outputs (tests/golden/disttostrm_reference.json, replayed by the
C restatement: tests/disttostrm_reference.py) and the restatement itself, bit for bit: the grid level on every recorded case (stream
cells with nodata p, chains of stream cells, a threshold above every src, src nodata, junk codes and cycles, rivers leaving every edge,
oblong cells, fel with -FLT_MAX holes, NaN and +-0, a spiral longer than one batch of levels, a serpentine), geographic per-row cell
sizes, the file level and both usages of both executables, TAUDEM_B200_GPUS = 1, 2 and 3, the pitremove -> d8flowdir -> aread8 ->
threshold -> d8hdisttostrm / d8vdisttostrm workflow with our executables, and a 2000 x 1500 grid."""
import os
import subprocess

import numpy as np
import pytest

import disttostrm_port
import disttostrm_reference as DR
from util import assert_bits, write_geographic_dem

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")


def _exe(*args, gpus=None):
    env = dict(os.environ)
    if gpus is not None:
        env["TAUDEM_B200_GPUS"] = str(gpus)
    r = subprocess.run([os.path.join(BIN, args[0]), *map(str, args[1:])], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0 and " error" not in r.stdout and "Error" not in r.stdout, r.stdout
    return r.stdout


def _grid(case):
    import taudem_b200 as td
    name, p, fel, src, thresh, dx, dy, _ = case
    h = td.d8hdisttostrm_grid(p, src, thresh=thresh, dx=dx, dy=dy, src_nodata=int(DR.SRC_ND))
    v = td.d8vdisttostrm_grid(p, fel, src, thresh=thresh, src_nodata=int(DR.SRC_ND))
    return h, v


def _restated(case):
    name, p, fel, src, thresh, dx, dy, _ = case
    return (disttostrm_port.disttostrm(p, src, thresh=thresh, dx=dx, dy=dy, src_nodata=int(DR.SRC_ND)),
            disttostrm_port.disttostrm(p, src, fel=fel, thresh=thresh, dx=dx, dy=dy, src_nodata=int(DR.SRC_ND)))


def test_grid_level_matches_the_reference(tmp_path):
    import taudem_b200 as td
    for case in DR.cases():
        want = DR.reference_case(DR.pipeline(tmp_path, case), case)
        got = _grid(case)
        for w, g, r, what in zip(want, got, _restated(case), ("h", "v")):
            assert_bits(g, w, f"{case[0]} {what} ({case[7]} reference ranks)")
            assert_bits(g, r, f"{case[0]} {what} (restatement)")
        if case[0] == "spiral":
            assert td.lib().td_disttostrm_last_levels() == case[1].size > 10 * 64


def test_grid_level_geographic_rows(tmp_path):
    """per-row cell sizes of a geographic raster for the horizontal distances"""
    import taudem_b200 as td
    name, p, fel, src, thresh, dx, dy, _ = [c for c in DR.cases() if c[0] == "strips"][0]
    f = str(tmp_path / "geo.tif")
    write_geographic_dem(f, fel)
    ny = fel.shape[0]
    xc, yc = np.empty(ny), np.empty(ny)
    assert td.lib().td_raster_cell_sizes(f.encode(), xc.ctypes.data, yc.ctypes.data, ny) == 0
    want = disttostrm_port.disttostrm(p, src, thresh=thresh, src_nodata=int(DR.SRC_ND), dxc=xc, dyc=yc)
    assert (want != DR.MISSINGFLOAT).sum() > 1000
    assert_bits(td.d8hdisttostrm_grid(p, src, thresh=thresh, src_nodata=int(DR.SRC_ND), dxc=xc, dyc=yc), want, "geographic")


def _files(tmp_path, case):
    import taudem_b200 as td
    name, p, fel, src, thresh, dx, dy, _ = case
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("basep.tif"), p, int(DR.P_ND), dx=dx, dy=dy)
    td.write_raster(d("basefel.tif"), fel, float(DR.MISSINGFLOAT), dx=dx, dy=dy)
    td.write_raster(d("basesrc.tif"), src, int(DR.SRC_ND), dx=dx, dy=dy)
    return d


def test_file_level_and_executables(tmp_path):
    """td_distgrid / td_d8vdistdown through the binding, both executables with flags and in simple usage (thresh 1): float32, nodata
    MISSINGFLOAT, p's georeference"""
    import taudem_b200 as td
    case = [c for c in DR.cases() if c[0] == "junk codes"][0]
    name, p, fel, src, thresh, dx, dy, _ = case
    (tmp_path / "r").mkdir()
    wh, wv = DR.reference_case(DR.pipeline(tmp_path / "r", case), case)
    d = _files(tmp_path, case)
    out = _exe("d8hdisttostrm", "-p", d("basep.tif"), "-src", d("basesrc.tif"), "-dist", d("h1.tif"), "-thresh", thresh)
    assert "D8HDistToStrm version" in out and "Compute time" in out, out
    out = _exe("d8vdisttostrm", "-p", d("basep.tif"), "-fel", d("basefel.tif"), "-src", d("basesrc.tif"), "-dist", d("v1.tif"), "-thresh", thresh)
    assert "D8VDistToStrm version" in out and "Compute time" in out, out
    assert td.lib().td_distgrid(d("basep.tif").encode(), d("basesrc.tif").encode(), d("h2.tif").encode(), thresh) == 0
    assert td.lib().td_d8vdistdown(d("basep.tif").encode(), d("basefel.tif").encode(), d("basesrc.tif").encode(), d("v2.tif").encode(), thresh) == 0
    c1 = case[:4] + (1,) + case[5:]
    h1, v1 = _restated(c1)
    _exe("d8hdisttostrm", d("base.tif"))                               # simple usage: basep.tif, basesrc.tif -> basedist.tif, thresh 1
    assert_bits(td.read_raster(d("basedist.tif"), np.float32), h1, "h simple usage")
    _exe("d8vdisttostrm", d("base.tif"))                               # ... and basefel.tif
    for f, w in (("h1.tif", wh), ("h2.tif", wh), ("v1.tif", wv), ("v2.tif", wv), ("basedist.tif", v1)):
        assert_bits(td.read_raster(d(f), np.float32), w, f)
        info = td.raster_info(d(f))
        assert np.float32(info["nodata"]) == DR.MISSINGFLOAT and info["bits"] == 32 and (info["dx"], info["dy"]) == (dx, dy), info
    # sizes that do not match: exit status 5, no output
    td.write_raster(d("small.tif"), src[:, :-1].copy(), int(DR.SRC_ND), dx=dx, dy=dy)
    r = subprocess.run([os.path.join(BIN, "d8hdisttostrm"), "-p", d("basep.tif"), "-src", d("small.tif"), "-dist", d("h4.tif")], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 5 and "File sizes do not match" in r.stdout, r.stdout
    assert not os.path.exists(d("h4.tif"))


@pytest.mark.parametrize("which", ["strips", "serpentine"])
def test_on_1_2_and_3_gpus(tmp_path, which):
    """TAUDEM_B200_GPUS=N: levels per strip, the value raster's edge rows exchanged, the edge-row cells they reach seeding the next
    levels; identical for every N, to the reference and to the restatement"""
    import taudem_b200 as td
    case = [c for c in DR.cases() if c[0] == which][-1]
    name, p, fel, src, thresh, dx, dy, _ = case
    (tmp_path / "r").mkdir()
    wh, wv = DR.reference_case(DR.pipeline(tmp_path / "r", case), case)
    rh, rv = _restated(case)
    d = _files(tmp_path, case)
    for n in (1, 2, 3):
        outh = _exe("d8hdisttostrm", "-p", d("basep.tif"), "-src", d("basesrc.tif"), "-dist", d(f"h{n}.tif"), "-thresh", thresh, gpus=n)
        _exe("d8vdisttostrm", "-p", d("basep.tif"), "-fel", d("basefel.tif"), "-src", d("basesrc.tif"), "-dist", d(f"v{n}.tif"), "-thresh", thresh, gpus=n)
        if n > 1:
            assert f"Processors: {n}" in outh, outh
            rounds = int(outh.split("Exchange rounds:")[1].split()[0])
            if which == "serpentine":
                assert rounds > 11, outh                 # a round per crossing of the path
        assert_bits(td.read_raster(d(f"h{n}.tif"), np.float32), wh, f"h at {n} GPUs")
        assert_bits(td.read_raster(d(f"v{n}.tif"), np.float32), wv, f"v at {n} GPUs")
    assert_bits(wh, rh, "h restatement")
    assert_bits(wv, rv, "v restatement")


def test_workflow_with_the_executables(tmp_path):
    """pitremove -> d8flowdir -> aread8 -> threshold -> d8hdisttostrm / d8vdisttostrm with our executables, equal to the reference's
    chain"""
    import taudem_b200 as td
    dem = DR.workflow_dem()
    (tmp_path / "r").mkdir()
    fel_r, p_r, ad8_r, src_r, h_r, v_r = DR.workflow(DR.RefPipeline(workdir=str(tmp_path / "r")), dem)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("dem.tif"), dem, -9999.0)
    _exe("pitremove", "-z", d("dem.tif"), "-fel", d("fel.tif"))
    _exe("d8flowdir", "-fel", d("fel.tif"), "-p", d("p.tif"), "-sd8", d("sd8.tif"))
    _exe("aread8", "-p", d("p.tif"), "-ad8", d("ad8.tif"))
    _exe("threshold", "-ssa", d("ad8.tif"), "-src", d("src.tif"), "-thresh", "30")
    _exe("d8hdisttostrm", "-p", d("p.tif"), "-src", d("src.tif"), "-dist", d("h.tif"))
    _exe("d8vdisttostrm", "-p", d("p.tif"), "-fel", d("fel.tif"), "-src", d("src.tif"), "-dist", d("v.tif"))
    assert_bits(td.read_raster(d("src.tif"), np.int16), src_r, "threshold")
    h = td.read_raster(d("h.tif"), np.float32)
    assert_bits(h, h_r, "d8hdisttostrm")
    assert_bits(td.read_raster(d("v.tif"), np.float32), v_r, "d8vdisttostrm")
    assert (h != DR.MISSINGFLOAT).sum() > h.size // 2


def test_large_grid(tmp_path):
    """2000 x 1500 at a threshold of 200 cells"""
    import taudem_b200 as td
    p, fel, src, thresh = DR.large()
    R = DR.RefPipeline(workdir=str(tmp_path))
    assert_bits(td.d8hdisttostrm_grid(p, src, thresh=thresh, src_nodata=int(DR.SRC_ND)), R.d8hdisttostrm(p, src, thresh=thresh), "h 2000 x 1500")
    v = td.d8vdisttostrm_grid(p, fel, src, thresh=thresh, src_nodata=int(DR.SRC_ND))
    assert_bits(v, R.d8vdisttostrm(p, fel, src, thresh=thresh), "v 2000 x 1500")
    assert (v != DR.MISSINGFLOAT).sum() > v.size // 2
