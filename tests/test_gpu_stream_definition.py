"""peukerdouglas and lengtharea on the GPU against the reference's outputs (tests/golden/stream_reference.json, replayed by
the restatements: tests/stream_reference.py), bit for bit: the grid level on a rough DEM with plateaus and on an odd-shaped DEM with nodata
holes (default and custom -par), the file level and the executables, peukerdouglas on 1, 2 and 3 GPUs (TAUDEM_B200_GPUS), and the
two documented workflows with our executables:

    pitremove -> d8flowdir -> peukerdouglas -> aread8 -wg ss -> threshold
    pitremove -> d8flowdir -> gridnet (plen) + aread8 -> lengtharea"""
import os
import subprocess

import numpy as np
import pytest

import stream_cases as S
import stream_reference as SR
import stream_restate
from util import assert_bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")


def _exe(tool, *args, gpus=None):
    env = dict(os.environ)
    if gpus is not None:
        env["TAUDEM_B200_GPUS"] = str(gpus)
    r = subprocess.run([os.path.join(BIN, tool), *map(str, args)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0 and " Error" not in r.stdout and "error" not in r.stdout, r.stdout
    return r.stdout


def test_peukerdouglas_grid_matches_the_reference(tmp_path):
    import taudem_b200 as td
    for name, dem, w, ranks in S.pd_calls():
        want = SR.RefPipeline(workdir=str(tmp_path), np_ranks=ranks).peukerdouglas(dem, **({} if w is None else {"weights": w}))
        got = td.peukerdouglas_grid(dem, nodata=float(S.ND)) if w is None else td.peukerdouglas_grid(dem, weights=w, nodata=float(S.ND))
        assert 0 < int((got == 1).sum()) < got.size // 2, name                  # sources exist, and not everywhere
        assert_bits(got, want, f"peukerdouglas_grid {name} {w} ({ranks} reference ranks)")


def test_lengtharea_grid_matches_the_reference(tmp_path):
    import taudem_b200 as td
    plen, ad8, ad8w = S.la_inputs()
    R = SR.RefPipeline(workdir=str(tmp_path))
    for a in (ad8, ad8w):
        ai = stream_restate.ad8_int32(a)
        for m, y in S.LA_PAR:
            want = R.lengtharea(plen, a) if m is None else R.lengtharea(plen, a, m=m, y=y)
            got = td.lengtharea_grid(plen, ai) if m is None else td.lengtharea_grid(plen, ai, m=m, y=y)
            assert_bits(got, want, f"lengtharea_grid {m} {y}")
            assert_bits(got, stream_restate.lengtharea(plen, a, m, y), f"lengtharea_grid {m} {y} (restatement)")


def test_file_level_and_executables(tmp_path):
    """td_peukerdouglas / td_lengtharea through the binding and the two executables (the ss rasters: int16, nodata -2 and -32768)"""
    import taudem_b200 as td
    dem = S.holes()
    (tmp_path / "r").mkdir()
    want = SR.RefPipeline(workdir=str(tmp_path / "r"), np_ranks=1).peukerdouglas(dem, weights=(0.5, 0.0, 0.2))
    fel = str(tmp_path / "fel.tif")
    td.write_raster(fel, dem, float(S.ND))
    out = _exe("peukerdouglas", "-fel", fel, "-ss", tmp_path / "ss.tif", "-par", 0.5, 0.0, 0.2)
    assert "PeukerDouglas version" in out and "Compute time" in out, out
    assert_bits(td.read_raster(str(tmp_path / "ss.tif"), np.int16), want, "peukerdouglas executable")
    assert td.raster_info(str(tmp_path / "ss.tif"))["nodata"] == -2
    check = td.lib().td_peukerdouglas(fel.encode(), str(tmp_path / "ss2.tif").encode(), np.asarray((0.5, 0.0, 0.2), np.float32).ctypes.data)
    assert check == 0
    assert_bits(td.read_raster(str(tmp_path / "ss2.tif"), np.int16), want, "td_peukerdouglas")

    plen, ad8, ad8w = S.la_inputs()
    want = SR.RefPipeline(workdir=str(tmp_path / "r")).lengtharea(plen, ad8w, m=0.01, y=1.5)
    td.write_raster(str(tmp_path / "plen.tif"), plen, -1.0)
    td.write_raster(str(tmp_path / "ad8.tif"), ad8w, -1.0)
    out = _exe("lengtharea", "-plen", tmp_path / "plen.tif", "-ad8", tmp_path / "ad8.tif", "-ss", tmp_path / "la.tif", "-par", 0.01, 1.5)
    assert "LengthArea version" in out and "Compute time" in out, out
    assert_bits(td.read_raster(str(tmp_path / "la.tif"), np.int16), want, "lengtharea executable")
    assert td.raster_info(str(tmp_path / "la.tif"))["nodata"] == -32768


@pytest.mark.parametrize("name", sorted(S.DEMS))
def test_peukerdouglas_on_1_2_and_3_gpus(tmp_path, name):
    """TAUDEM_B200_GPUS=N: row strips, the smoothed edge rows exchanged between the passes; identical for every N and to the
    reference on 3 ranks."""
    import taudem_b200 as td
    dem = S.DEMS[name]()
    want = SR.RefPipeline(workdir=str(tmp_path), np_ranks=3).peukerdouglas(dem)
    fel = str(tmp_path / "fel.tif")
    td.write_raster(fel, dem, float(S.ND))
    outs = []
    for n in (1, 2, 3):
        out = _exe("peukerdouglas", "-fel", fel, "-ss", tmp_path / f"ss{n}.tif", gpus=n)
        if n > 1:
            assert f"Processors: {n}" in out, out
        outs.append(td.read_raster(str(tmp_path / f"ss{n}.tif"), np.int16))
    for n, o in zip((1, 2, 3), outs):
        assert_bits(o, outs[0], f"{n} GPUs vs 1")
        assert_bits(o, want, f"{n} GPUs vs the reference")


def test_peukerdouglas_workflow_with_the_executables(tmp_path):
    import taudem_b200 as td
    dem = S.workflow_dem()
    (tmp_path / "r").mkdir()
    _, _, ss_r, ssa_r, src_r = S.pd_workflow(SR.RefPipeline(workdir=str(tmp_path / "r")), dem)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("dem.tif"), dem, -9999.0)
    _exe("pitremove", "-z", d("dem.tif"), "-fel", d("fel.tif"))
    _exe("d8flowdir", "-fel", d("fel.tif"), "-p", d("p.tif"), "-sd8", d("sd8.tif"))
    _exe("peukerdouglas", "-fel", d("fel.tif"), "-ss", d("ss.tif"))
    _exe("aread8", "-p", d("p.tif"), "-ad8", d("ssa.tif"), "-wg", d("ss.tif"))
    _exe("threshold", "-ssa", d("ssa.tif"), "-src", d("src.tif"), "-thresh", S.PD_THRESH)
    assert_bits(td.read_raster(d("ss.tif"), np.int16), ss_r, "ss")
    assert_bits(td.read_raster(d("ssa.tif"), np.float32), ssa_r, "aread8 -wg ss")
    src = td.read_raster(d("src.tif"), np.int16)
    assert_bits(src, src_r, "threshold")
    assert (src == 1).sum() > 0


def test_lengtharea_workflow_with_the_executables(tmp_path):
    import taudem_b200 as td
    dem = S.workflow_dem()
    (tmp_path / "r").mkdir()
    _, _, plen_r, ad8_r, ss_r = S.la_workflow(SR.RefPipeline(workdir=str(tmp_path / "r")), dem)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("dem.tif"), dem, -9999.0)
    _exe("pitremove", "-z", d("dem.tif"), "-fel", d("fel.tif"))
    _exe("d8flowdir", "-fel", d("fel.tif"), "-p", d("p.tif"), "-sd8", d("sd8.tif"))
    _exe("gridnet", "-p", d("p.tif"), "-plen", d("plen.tif"), "-tlen", d("tlen.tif"), "-gord", d("gord.tif"))
    _exe("aread8", "-p", d("p.tif"), "-ad8", d("ad8.tif"))
    _exe("lengtharea", "-plen", d("plen.tif"), "-ad8", d("ad8.tif"), "-ss", d("ss.tif"))
    assert_bits(td.read_raster(d("plen.tif"), np.float32), plen_r, "gridnet plen")
    assert_bits(td.read_raster(d("ad8.tif"), np.float32), ad8_r, "aread8")
    ss = td.read_raster(d("ss.tif"), np.int16)
    assert_bits(ss, ss_r, "lengtharea")
    assert (ss == 1).sum() > 0 and (ss == 0).sum() > 0
