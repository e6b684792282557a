"""flowdircond on the GPU against the reference's outputs (tests/golden/conditioning_reference.json, replayed by the C restatement:
tests/conditioning_reference.py) and the restatement itself, bit for bit: the grid level on every recorded case (p of a burned DEM
on the raw DEM, p of another DEM, random codes with cycles and code 0s, nodata holes in z, in p and in both, z nodata -FLT_MAX,
-9999 and a value cells lie within 1e-5 of, +-0 and NaN, rivers leaving every edge, rivers crossing tiles), the file level and the
executable in both usages, TAUDEM_B200_GPUS = 1, 2 and 3 in rounds and (one device per rank) peer mode, the pitremove ->
d8flowdir -> flowdircond workflow with our executables, and a 2000 x 1500 grid."""
import os
import subprocess

import numpy as np
import pytest

import conditioning_port
import conditioning_reference as CR
from util import assert_bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")


def _exe(*args, gpus=None, peer=None):
    env = dict(os.environ)
    env.pop("TAUDEM_B200_PEER", None)
    if gpus is not None:
        env["TAUDEM_B200_GPUS"] = str(gpus)
    if peer is not None:
        env["TAUDEM_B200_PEER"] = peer
    r = subprocess.run([os.path.join(BIN, args[0]), *map(str, args[1:])], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0 and " error" not in r.stdout and "Error" not in r.stdout, r.stdout
    return r.stdout


def test_grid_level_matches_the_reference(tmp_path):
    import taudem_b200 as td
    for case in CR.cases():
        name, p, pnd, z, znd, ranks = case
        want = CR.reference_case(CR.pipeline(tmp_path, case), case)
        got = td.flowdircond_grid(p, z, p_nodata=int(pnd), nodata=float(znd))
        assert_bits(got, want, f"{name} ({ranks} reference ranks)")
        assert_bits(got, conditioning_port.flowdircond(p, z, p_nodata=pnd, nodata=znd), f"{name} (restatement)")


def test_file_level_and_executable(tmp_path):
    """td_flowdircond through the binding, the executable with flags and in simple usage: float32, z's nodata and georeference"""
    import taudem_b200 as td
    case = [c for c in CR.cases() if c[0] == "both holes"][0]
    name, p, pnd, z, znd, _ = case
    (tmp_path / "r").mkdir()
    want = CR.reference_case(CR.pipeline(tmp_path / "r", case), case)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("basez.tif"), z, float(znd), dx=10.0, dy=7.0)
    td.write_raster(d("basep.tif"), p, int(pnd), dx=10.0, dy=7.0)
    out = _exe("flowdircond", "-p", d("basep.tif"), "-z", d("basez.tif"), "-zfdc", d("o1.tif"))
    assert "FlowDirCond version" in out and "Compute time" in out, out
    assert td.lib().td_flowdircond(d("basep.tif").encode(), d("basez.tif").encode(), d("o2.tif").encode()) == 0
    _exe("flowdircond", d("base.tif"))                                # simple usage: basep.tif, basez.tif -> basezfdc.tif
    for f in ("o1.tif", "o2.tif", "basezfdc.tif"):
        assert_bits(td.read_raster(d(f), np.float32), want, f)
        info = td.raster_info(d(f))
        assert info["nodata"] == float(znd) and info["bits"] == 32 and (info["dx"], info["dy"]) == (10.0, 7.0), info
    # the output takes z's nodata value as z's header holds it (a double that is not a float here)
    td.write_raster(d("z3.tif"), z, -3.0e38, dx=10.0, dy=7.0)
    _exe("flowdircond", "-p", d("basep.tif"), "-z", d("z3.tif"), "-zfdc", d("o3.tif"))
    assert td.raster_info(d("o3.tif"))["nodata"] == -3.0e38
    assert_bits(td.read_raster(d("o3.tif"), np.float32), conditioning_port.flowdircond(p, z, p_nodata=pnd, nodata=np.float32(-3.0e38)), "o3")


@pytest.mark.parametrize("which", ["strips", "strips other", "strips random"])
def test_on_1_2_and_3_gpus(tmp_path, which):
    """TAUDEM_B200_GPUS=N in rounds mode, and in peer mode where there is one device per rank: identical for every N and to the
    reference on 3 ranks"""
    import taudem_b200 as td
    case = [c for c in CR.cases() if c[0] == which and c[5] == 3][0]
    name, p, pnd, z, znd, _ = case
    (tmp_path / "r").mkdir()
    want = CR.reference_case(CR.pipeline(tmp_path / "r", case), case)
    td.write_raster(str(tmp_path / "z.tif"), z, float(znd))
    td.write_raster(str(tmp_path / "p.tif"), p, int(pnd))
    runs = [(1, None), (2, "0"), (3, "0")] + [(n, None) for n in (2, 3) if td.device_count() >= n]
    for n, peer in runs:
        f = tmp_path / f"o{n}_{peer}.tif"
        out = _exe("flowdircond", "-p", tmp_path / "p.tif", "-z", tmp_path / "z.tif", "-zfdc", f, gpus=n, peer=peer)
        if n > 1:
            assert f"Processors: {n}" in out, out
        assert_bits(td.read_raster(str(f), np.float32), want, f"{n} GPUs, peer={peer}")


def test_workflow_with_the_executables(tmp_path):
    """pitremove -> d8flowdir -> flowdircond of the raw DEM with our executables, equal to the reference's chain"""
    import taudem_b200 as td
    dem = CR.workflow_dem()
    (tmp_path / "r").mkdir()
    fel_r, p_r, z_r = CR.workflow(CR.RefPipeline(workdir=str(tmp_path / "r")), dem)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("dem.tif"), dem, -9999.0)
    _exe("pitremove", "-z", d("dem.tif"), "-fel", d("fel.tif"))
    _exe("d8flowdir", "-fel", d("fel.tif"), "-p", d("p.tif"), "-sd8", d("sd8.tif"))
    _exe("flowdircond", "-p", d("p.tif"), "-z", d("dem.tif"), "-zfdc", d("zfdc.tif"))
    assert_bits(td.read_raster(d("fel.tif"), np.float32), fel_r, "pitremove")
    assert_bits(td.read_raster(d("p.tif"), np.int16), p_r, "d8flowdir")
    assert_bits(td.read_raster(d("zfdc.tif"), np.float32), z_r, "flowdircond")


def test_large_grid(tmp_path):
    """2000 x 1500: p of a burned DEM on the raw DEM"""
    import taudem_b200 as td
    z, p = CR.large()
    want = CR.RefPipeline(workdir=str(tmp_path)).flowdircond(p, z)
    got = td.flowdircond_grid(p, z)
    assert_bits(got, want, "2000 x 1500")
    assert (got < z).sum() > 1000


# ---------------------------------------------------------------- retlimflow
def _rl_want(case):
    name, ang, andv, wg, wnd, rc, rcnd, dx, dy, ranks = case
    return conditioning_port.retlimflow(ang, wg, rc, dx=dx, dy=dy, ang_nodata=andv, wg_nodata=wnd, rc_nodata=rcnd)


def test_retlimflow_grid_level(tmp_path):
    """every retlimflow case against the restatement, and against the reference's output wherever the reference's one-rank edge
    handling (DESIGN.md §2) changes nothing: every case but the angle torture"""
    import taudem_b200 as td
    for case in CR.rl_cases():
        name, ang, andv, wg, wnd, rc, rcnd, dx, dy, ranks = case
        ref = CR.rl_reference_case(CR.rl_pipeline(tmp_path, case), case)
        got = td.retlimflow_grid(ang, wg, rc, dx=dx, dy=dy, ang_nodata=float(andv), wg_nodata=float(wnd), rc_nodata=float(rcnd))
        assert_bits(got, _rl_want(case), f"{name} (restatement)")
        if name != "rl torture":
            assert_bits(got, ref, f"{name} ({ranks} reference ranks)")


def test_retlimflow_geographic_rows(tmp_path):
    import taudem_b200 as td
    from util import write_geographic_dem
    name, ang, andv, wg, wnd, rc, rcnd, dx, dy, r = [c for c in CR.rl_cases() if c[0] == "rl strips"][0]
    f = str(tmp_path / "geo.tif")
    write_geographic_dem(f, np.zeros(ang.shape, np.float32))
    ny = ang.shape[0]
    xc, yc = np.empty(ny), np.empty(ny)
    assert td.lib().td_raster_cell_sizes(f.encode(), xc.ctypes.data, yc.ctypes.data, ny) == 0
    want = conditioning_port.retlimflow(ang, wg, rc, dxc=xc, dyc=yc)
    assert_bits(td.retlimflow_grid(ang, wg, rc, dxc=xc, dyc=yc), want, "geographic")


def test_retlimflow_refuses_an_angle_nodata_that_is_a_direction():
    import taudem_b200 as td
    name, ang, andv, wg, wnd, rc, rcnd, dx, dy, r = CR.rl_cases()[0]
    for nd in (1.0, 0.0, -0.5):
        with pytest.raises(td.TaudemError) as e:
            td.retlimflow_grid(ang, wg, rc, ang_nodata=nd)
        assert e.value.code == 1
    td.retlimflow_grid(ang, wg, rc, ang_nodata=-9999.0)


def test_retlimflow_file_level_and_executable(tmp_path):
    """td_retlimro, the executable with flags and in simple usage: float32, nodata MISSINGFLOAT, rc's georeference"""
    import taudem_b200 as td
    case = [c for c in CR.rl_cases() if c[0] == "rl all holes"][0]
    name, ang, andv, wg, wnd, rc, rcnd, dx, dy, _ = case
    (tmp_path / "r").mkdir()
    want = CR.rl_reference_case(CR.rl_pipeline(tmp_path / "r", case), case)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("baseang.tif"), ang, float(andv))
    td.write_raster(d("basewg.tif"), wg, float(wnd))
    td.write_raster(d("baserc.tif"), rc, float(rcnd))
    out = _exe("retlimflow", "-ang", d("baseang.tif"), "-wg", d("basewg.tif"), "-rc", d("baserc.tif"), "-qrl", d("q1.tif"))
    assert "Retention limited flow accumulation version" in out, out
    assert td.lib().td_retlimro(d("baseang.tif").encode(), d("basewg.tif").encode(), d("baserc.tif").encode(), d("q2.tif").encode()) == 0
    _exe("retlimflow", d("base.tif"))                                 # simple usage -> baseqrl.tif
    for f in ("q1.tif", "q2.tif", "baseqrl.tif"):
        assert_bits(td.read_raster(d(f), np.float32), want, f)
        info = td.raster_info(d(f))
        assert np.float32(info["nodata"]) == CR.MISSINGFLOAT and info["bits"] == 32, info


@pytest.mark.parametrize("which", ["rl strips", "rl comb"])
def test_retlimflow_on_1_2_and_3_gpus(tmp_path, which):
    import taudem_b200 as td
    case = [c for c in CR.rl_cases() if c[0] == which and c[9] == 3][0]
    name, ang, andv, wg, wnd, rc, rcnd, dx, dy, _ = case
    (tmp_path / "r").mkdir()
    want = CR.rl_reference_case(CR.rl_pipeline(tmp_path / "r", case), case)
    for n_, f in (("ang", ang), ("wg", wg), ("rc", rc)):
        td.write_raster(str(tmp_path / f"{n_}.tif"), f, float({"ang": andv, "wg": wnd, "rc": rcnd}[n_]))
    runs = [(1, None), (2, "0"), (3, "0")] + [(n, None) for n in (2, 3) if td.device_count() >= n]
    for n, peer in runs:
        f = tmp_path / f"q{n}_{peer}.tif"
        out = _exe("retlimflow", "-ang", tmp_path / "ang.tif", "-wg", tmp_path / "wg.tif", "-rc", tmp_path / "rc.tif", "-qrl", f, gpus=n, peer=peer)
        if n > 1:
            assert f"Processors: {n}" in out, out
        assert_bits(td.read_raster(str(f), np.float32), want, f"{n} GPUs, peer={peer}")


def test_retlimflow_workflow_and_large(tmp_path):
    """pitremove -> dinfflowdir -> retlimflow with our executables, and a 2000 x 1500 grid, equal to the reference"""
    import taudem_b200 as td
    dem = CR.workflow_dem()
    wg, rc = CR.rl_inputs(dem, 74)
    (tmp_path / "r").mkdir()
    q_r = CR.rl_workflow(CR.RefPipeline(workdir=str(tmp_path / "r")), dem, wg, rc)
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("dem.tif"), dem, -9999.0)
    td.write_raster(d("wg.tif"), wg, -9999.0)
    td.write_raster(d("rc.tif"), rc, -9999.0)
    _exe("pitremove", "-z", d("dem.tif"), "-fel", d("fel.tif"))
    _exe("dinfflowdir", "-fel", d("fel.tif"), "-ang", d("ang.tif"), "-slp", d("slp.tif"))
    _exe("retlimflow", "-ang", d("ang.tif"), "-wg", d("wg.tif"), "-rc", d("rc.tif"), "-qrl", d("qrl.tif"))
    assert_bits(td.read_raster(d("qrl.tif"), np.float32), q_r, "retlimflow")
    ang, wg, rc = CR.rl_large()
    want = CR.RefPipeline(workdir=str(tmp_path)).retlimflow(ang, wg, rc)
    assert_bits(td.retlimflow_grid(ang, wg, rc), want, "2000 x 1500")
