"""slopeavedown on the GPU against the reference's outputs (tests/golden/slopeavedown_reference.json, replayed by the C restatement:
tests/slopeavedown_reference.py) and the restatement itself, bit for bit: the grid level on every recorded case (flats, nodata holes
in fel, in p and in both, junk codes, cycles and phantom contributors, rivers leaving every edge, the dn edge cases, oblong cells,
DEM nodata -FLT_MAX), geographic per-row cell sizes, the file level and the executable in both usages, TAUDEM_B200_GPUS = 1, 2
and 3, the pitremove -> d8flowdir -> slopeavedown workflow with our executables, and a 2000 x 1500 grid with niter = 50."""
import os
import subprocess

import numpy as np
import pytest

import downslope_port
import slopeavedown_reference as SR
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


def test_grid_level_matches_the_reference(tmp_path):
    import taudem_b200 as td
    for case in SR.cases():
        name, fel, fnd, p, pnd, dx, dy, dn, ranks = case
        want = SR.reference_case(SR.pipeline(tmp_path, case), case)
        got = td.slopeavedown_grid(fel, p, dn=dn, dx=dx, dy=dy, nodata=float(fnd), p_nodata=int(pnd))
        assert_bits(got, want, f"{name} ({ranks} reference ranks)")
        assert_bits(got, downslope_port.slopeavedown(fel, p, dn=dn, dx=dx, dy=dy, nodata=fnd, p_nodata=pnd), f"{name} (restatement)")


def test_grid_level_geographic_rows(tmp_path):
    """per-row cell sizes of a geographic raster for the distances, the middle row's for niter (tiffIO's dxA / dyA)"""
    import taudem_b200 as td
    name, fel, fnd, p, pnd, dx, dy, dn, r = [c for c in SR.cases() if c[0] == "strips junk"][0]
    f = str(tmp_path / "geo.tif")
    write_geographic_dem(f, fel)
    ny = fel.shape[0]
    xc, yc = np.empty(ny), np.empty(ny)
    assert td.lib().td_raster_cell_sizes(f.encode(), xc.ctypes.data, yc.ctypes.data, ny) == 0
    dxa, dya = abs(xc[ny // 2]), abs(yc[ny // 2])
    want = downslope_port.slopeavedown(fel, p, dn=700.0, dx=dxa, dy=dya, nodata=fnd, dxc=xc, dyc=yc)
    assert (want != SR.MISSINGFLOAT).sum() > 100
    assert_bits(td.slopeavedown_grid(fel, p, dn=700.0, dx=dxa, dy=dya, nodata=float(fnd), dxc=xc, dyc=yc), want, "geographic")


def test_undefined_niter_is_refused():
    import taudem_b200 as td
    fel, p = SR.flow(8, 9, 3)
    for dn in (float("nan"), float("inf"), 1e300):
        with pytest.raises(td.TaudemError) as e:
            td.slopeavedown_grid(fel, p, dn=dn)
        assert e.value.code == 1


def test_file_level_and_executable(tmp_path):
    """td_sloped through the binding, the executable with flags and in simple usage: float32, nodata MISSINGFLOAT, p's georeference"""
    import taudem_b200 as td
    case = [c for c in SR.cases() if c[0] == "both holes"][0]
    name, fel, fnd, p, pnd, dx, dy, dn, _ = case
    (tmp_path / "r").mkdir()
    want = SR.reference_case(SR.pipeline(tmp_path / "r", case), case)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("basefel.tif"), fel, float(fnd), dx=dx, dy=dy)
    td.write_raster(d("basep.tif"), p, int(pnd), dx=dx, dy=dy)
    out = _exe("slopeavedown", "-p", d("basep.tif"), "-fel", d("basefel.tif"), "-slpd", d("s1.tif"), "-dn", dn)
    assert "SlopeAveDown version" in out and "Compute time" in out, out
    assert td.lib().td_sloped(d("basep.tif").encode(), d("basefel.tif").encode(), d("s2.tif").encode(), dn) == 0
    want50 = downslope_port.slopeavedown(fel, p, dn=50.0, dx=dx, dy=dy, nodata=fnd, p_nodata=pnd)
    _exe("slopeavedown", d("base.tif"))                               # simple usage: basefel.tif, basep.tif -> baseslpd.tif, dn 50
    for f, w in (("s1.tif", want), ("s2.tif", want), ("baseslpd.tif", want50)):
        assert_bits(td.read_raster(d(f), np.float32), w, f)
        info = td.raster_info(d(f))
        assert np.float32(info["nodata"]) == SR.MISSINGFLOAT and info["bits"] == 32 and (info["dx"], info["dy"]) == (dx, dy), info
    # the output takes p's georeference: a p raster with other (matching within the tolerance) cell sizes shows through
    td.write_raster(d("p2.tif"), p, int(pnd), like=d("basefel.tif"))
    _exe("slopeavedown", "-p", d("p2.tif"), "-fel", d("basefel.tif"), "-slpd", d("s3.tif"), "-dn", dn)
    assert_bits(td.read_raster(d("s3.tif"), np.float32), want, "s3")
    # sizes that do not match
    td.write_raster(d("small.tif"), p[:, :-1].copy(), int(pnd), dx=dx, dy=dy)
    r = subprocess.run([os.path.join(BIN, "slopeavedown"), "-p", d("small.tif"), "-fel", d("basefel.tif"), "-slpd", d("s4.tif")], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=120)
    assert "File sizes do not match" in r.stdout and "sloped error 5" in r.stdout, r.stdout
    assert not os.path.exists(d("s4.tif"))


@pytest.mark.parametrize("which", ["strips", "strips junk"])
def test_on_1_2_and_3_gpus(tmp_path, which):
    """TAUDEM_B200_GPUS=N: the D8 sweep on row strips, then the passes with the state's edge rows exchanged; identical for every N
    and to the reference on 3 ranks."""
    import taudem_b200 as td
    case = [c for c in SR.cases() if c[0] == which and c[8] == 3][0]
    name, fel, fnd, p, pnd, dx, dy, dn, _ = case
    (tmp_path / "r").mkdir()
    want = SR.reference_case(SR.pipeline(tmp_path / "r", case), case)
    td.write_raster(str(tmp_path / "fel.tif"), fel, float(fnd), dx=dx, dy=dy)
    td.write_raster(str(tmp_path / "p.tif"), p, int(pnd), dx=dx, dy=dy)
    outs = []
    for n in (1, 2, 3):
        out = _exe("slopeavedown", "-p", tmp_path / "p.tif", "-fel", tmp_path / "fel.tif", "-slpd", tmp_path / f"s{n}.tif", "-dn", dn, gpus=n)
        if n > 1:
            assert f"Processors: {n}" in out, out
        outs.append(td.read_raster(str(tmp_path / f"s{n}.tif"), np.float32))
    for n, o in zip((1, 2, 3), outs):
        assert_bits(o, outs[0], f"{n} GPUs vs 1")
        assert_bits(o, want, f"{n} GPUs vs the reference")


def test_workflow_with_the_executables(tmp_path):
    """pitremove -> d8flowdir -> slopeavedown with our executables, equal to the reference's chain"""
    import taudem_b200 as td
    dem = SR.workflow_dem()
    (tmp_path / "r").mkdir()
    fel_r, p_r, s_r = SR.workflow(SR.RefPipeline(workdir=str(tmp_path / "r")), dem)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("dem.tif"), dem, -9999.0)
    _exe("pitremove", "-z", d("dem.tif"), "-fel", d("fel.tif"))
    _exe("d8flowdir", "-fel", d("fel.tif"), "-p", d("p.tif"), "-sd8", d("sd8.tif"))
    _exe("slopeavedown", "-p", d("p.tif"), "-fel", d("fel.tif"), "-slpd", d("slpd.tif"))
    assert_bits(td.read_raster(d("fel.tif"), np.float32), fel_r, "pitremove")
    assert_bits(td.read_raster(d("p.tif"), np.int16), p_r, "d8flowdir")
    s = td.read_raster(d("slpd.tif"), np.float32)
    assert_bits(s, s_r, "slopeavedown")
    assert (s != SR.MISSINGFLOAT).sum() > s.size // 2


def test_large_grid_many_passes(tmp_path):
    """2000 x 1500, dn = 1470 at 30 m: niter = 50, all of them changing cells"""
    import taudem_b200 as td
    fel, p, dn = SR.large()
    want = SR.RefPipeline(workdir=str(tmp_path)).slopeavedown(fel, p, dn=dn)
    got = td.slopeavedown_grid(fel, p, dn=dn)
    assert_bits(got, want, "2000 x 1500")
    assert (got != SR.MISSINGFLOAT).sum() > 0
