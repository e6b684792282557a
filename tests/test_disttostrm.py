"""d8hdisttostrm and d8vdisttostrm without a GPU: the C restatement (oracle/port/disttostrm_oracle.c) replays every reference output
the GPU tests compare against (tests/golden/disttostrm_reference.json) and, where oracle/_ref holds the reference's tools, matches the
live executables on random grids at 1 and 3 ranks; the BFS kernels (k_dts_seed, k_dts_level, k_dts_edge) on the CPU emulation of
the thread model (tests/emu/dts_driver.cpp), bit for bit against the restatement on 1, 2 and 3 row strips with the value raster's
edge rows exchanged between rounds, under several schedule seeds and on geographic rows; and the command lines' usage and error
paths."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import disttostrm_port
import disttostrm_reference as DR
import test_emu
from util import assert_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")

pytestmark = pytest.mark.skipif(not disttostrm_port.available(), reason="make -C oracle -f disttostrm.mk port")


def _want(case, vertical, dxc=None, dyc=None):
    name, p, fel, src, thresh, dx, dy, _ = case
    return disttostrm_port.disttostrm(p, src, fel=fel if vertical else None, thresh=thresh, dx=dx, dy=dy, src_nodata=int(DR.SRC_ND), dxc=dxc,
                                      dyc=dyc)


# ---------------------------------------------------------------- the restatement on the stored reference outputs
def test_restatement_replays_every_stored_output(tmp_path):
    """Every reference output of the distance tests, recomputed by the restatements and matched to its stored digest.  The count is
    asserted: a call that is not replayed fails here."""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    before = set(DR.replayed)
    n = 0
    for case in DR.cases():
        DR.reference_case(DR.pipeline(tmp_path, case), case)
        n += 1
    DR.workflow(DR.RefPipeline(workdir=str(tmp_path)), DR.workflow_dem())
    p, fel, src, thresh = DR.large()
    R = DR.RefPipeline(workdir=str(tmp_path))
    R.d8hdisttostrm(p, src, thresh=thresh)
    R.d8vdisttostrm(p, fel, src, thresh=thresh)
    if not DR.reference.RECORD:
        tools = sorted(DR.replayed[k] for k in set(DR.replayed) - before)
        assert tools.count("d8hdisttostrm") == tools.count("d8vdisttostrm") == n + 2 == 16, tools
        assert all(tools.count(t) == 1 for t in ("pitremove", "d8flowdir", "aread8", "threshold")), tools


def test_cases_cover_the_edge_shapes():
    """the recorded cases reach what they are named for: an all-nodata result, stream cells with nodata p, a path of more than one
    batch of levels, values through NaN, and cells left MISSINGFLOAT beside reached ones"""
    by = {c[0]: c for c in DR.cases()}
    assert (_want(by["rough thresh=1000000"], False) == DR.MISSINGFLOAT).all()
    c = by["stream p nodata"]
    assert ((c[3] >= c[4]) & (c[1] == DR.P_ND)).sum() > 5
    assert (_want(c, False)[(c[3] >= c[4]) & (c[1] == DR.P_ND)] == 0).all()
    sp = _want(by["spiral"], False)
    assert (sp != DR.MISSINGFLOAT).all() and sp.max() > 30.0 * 600
    v = _want(by["fel float range"], True)
    assert np.isnan(v).sum() > 10 and (v == DR.MISSINGFLOAT).sum() > 10 and np.isfinite(v).sum() > 100
    j = _want(by["junk codes"], False)
    assert (j == DR.MISSINGFLOAT).sum() > 50 and (j > 0).sum() > 100


def test_restatement_matches_the_live_reference(tmp_path, monkeypatch):
    """With oracle/_ref built: random small grids (random codes in -3..12, cycles, nodata in p and src, fel holes at -FLT_MAX, NaN),
    both reference executables at 1 and 3 ranks against the restatement."""
    import refrun
    if not DR.available():
        pytest.skip("the reference's distance tools are not built (make -C oracle -f disttostrm.mk ref)")
    monkeypatch.setattr(refrun, "INPUTS_ONLY", False)
    for seed in range(6):
        rng = np.random.default_rng(seed)
        fel, p, src = DR.flow(23, 31, 100 + seed)
        if seed % 3 == 0:
            m = rng.random(p.shape) < 0.3
            p[m] = rng.integers(-3, 13, m.sum())
            p[rng.random(p.shape) < 0.05] = DR.P_ND
        if seed % 2:
            src[rng.random(p.shape) < 0.1] = DR.SRC_ND
            fel[rng.random(p.shape) < 0.05] = DR.MISSINGFLOAT
            fel[rng.random(p.shape) < 0.03] = np.nan
        thresh = int(rng.integers(1, 40))
        for dx, dy in ((30.0, 30.0), (10.0, 7.0)):
            case = ("random", p, fel, src, thresh, dx, dy, 1)
            wh, wv = _want(case, False), _want(case, True)
            for ranks in (1, 3):
                F = DR.Files(workdir=str(tmp_path), dx=dx, dy=dy, np_ranks=ranks)
                assert_bits(F.d8hdisttostrm(p, src, thresh=thresh), wh, f"h seed {seed} dx {dx} at {ranks} ranks")
                assert_bits(F.d8vdisttostrm(p, fel, src, thresh=thresh), wv, f"v seed {seed} dx {dx} at {ranks} ranks")


# ---------------------------------------------------------------- the kernels on the CPU emulation
@pytest.fixture(scope="module")
def emu():
    os.makedirs(test_emu.BUILD, exist_ok=True)
    inc = test_emu._transform("disttostrm", 5)
    so = os.path.join(test_emu.BUILD, "libemu_dts.so")
    srcs = [os.path.join(test_emu.EMU, f) for f in ("dts_driver.cpp", "emu.cpp")]
    deps = srcs + [inc, os.path.join(test_emu.EMU, "cuda_runtime.h"), os.path.join(test_emu.CSRC, "common.cuh"), os.path.join(test_emu.CSRC, "kernels.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        # (the default TLS model: another initial-exec emulation library in the process would exhaust the static TLS block the others need)
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ffp-contract=off",
                               "-I", test_emu.EMU, "-I", test_emu.BUILD, "-I", test_emu.CSRC, "-o", so, *srcs])
    lib = C.CDLL(so)
    P = C.c_void_p
    lib.emu_disttostrm.argtypes = [C.c_int, P, P, P, P, C.c_int, C.c_int, C.c_int16, C.c_int32, C.c_int, P, P, C.c_int, P, C.c_uint, C.c_int, P]
    return lib


def _emu(lib, case, vertical, strips=None, seed=1, grid=3, dxc=None, dyc=None):
    name, p, fel, src, thresh, dx, dy, _ = case
    p = np.ascontiguousarray(p, np.int16); src = np.ascontiguousarray(src, np.int32); fel = np.ascontiguousarray(fel, np.float32)
    ny, nx = p.shape
    xc = np.ascontiguousarray(np.full(ny, dx) if dxc is None else dxc, np.float64)
    yc = np.ascontiguousarray(np.full(ny, dy) if dyc is None else dyc, np.float64)
    rows = np.ascontiguousarray([ny] if strips is None else strips, np.int32)
    assert rows.sum() == ny
    out = np.empty((ny, nx), np.float32)
    rounds = C.c_int(0)
    assert lib.emu_disttostrm(int(vertical), p.ctypes.data, fel.ctypes.data, src.ctypes.data, out.ctypes.data, nx, ny, int(DR.P_ND), int(DR.SRC_ND),
                              int(thresh), xc.ctypes.data, yc.ctypes.data, len(rows), rows.ctypes.data, seed, grid, C.byref(rounds)) == 0
    return out, rounds.value


@pytest.mark.parametrize("vertical", [False, True])
def test_emulated_kernels_match_the_restatement(emu, vertical):
    """every one-rank case on one strip, under two schedule seeds and two grid sizes"""
    for case in DR.cases():
        if case[7] != 1:
            continue
        want = _want(case, vertical)
        for seed, grid in ((1, 1), (7, 3)):
            assert_bits(_emu(emu, case, vertical, seed=seed, grid=grid)[0], want, f"{case[0]} seed {seed}")


@pytest.mark.parametrize("strips", [(35, 35), (23, 24, 23), (1, 2, 67), (34, 1, 35)])
def test_emulated_row_strips(emu, strips):
    """2 and 3 strips (and strips of one and two rows), the value raster's edge rows exchanged between rounds until no strip adds a
    cell: identical to the restatement"""
    for case in DR.cases():
        if case[0] == "strips" and case[7] == 1:
            for vertical in (False, True):
                assert_bits(_emu(emu, case, vertical, strips, seed=3)[0], _want(case, vertical), f"{case[0]} {strips} v={vertical}")


def test_emulated_serpentine_crosses_strips_many_times(emu):
    """a path down and up every column: 3 strips need a round per crossing, and the result is the one-strip result"""
    case = [c for c in DR.cases() if c[0] == "serpentine"][0]
    for vertical in (False, True):
        got, rounds = _emu(emu, case, vertical, (10, 10, 10), seed=5)
        assert_bits(got, _want(case, vertical), f"serpentine v={vertical}")
        assert rounds > 2 * 11
        assert_bits(_emu(emu, case, vertical, (1, 28, 1), seed=2)[0], _want(case, vertical), "serpentine one-row strips")


def test_emulated_geographic_rows(emu, tmp_path):
    """per-row cell sizes of a geographic raster for the horizontal distances"""
    import taudem_b200 as td
    from util import write_geographic_dem
    case = [c for c in DR.cases() if c[0] == "strips"][0]
    f = str(tmp_path / "geo.tif")
    write_geographic_dem(f, case[2])
    ny = case[1].shape[0]
    xc, yc = np.empty(ny), np.empty(ny)
    assert td.lib().td_raster_cell_sizes(f.encode(), xc.ctypes.data, yc.ctypes.data, ny) == 0
    want = _want(case, False, xc, yc)
    assert len(np.unique(xc)) > 10 and (want != DR.MISSINGFLOAT).sum() > 1000
    for strips in (None, (30, 40)):
        assert_bits(_emu(emu, case, False, strips, dxc=xc, dyc=yc)[0], want, f"geographic {strips}")


# ---------------------------------------------------------------- command line and arguments
def _run(tool, *args):
    exe = os.path.join(BIN, tool)
    if not os.access(exe, os.X_OK):
        pytest.skip("executables not built")
    r = subprocess.run([exe, *args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    return r.returncode, r.stdout


@pytest.mark.parametrize("tool,line,usage", [("d8hdisttostrm", "D8 distance error 1", "-src <srcfile> -dist <distfile> [-thresh <thresh>]"),
                                             ("d8vdisttostrm", "D8 distance down error 1", "-fel <felfile> -src <srcfile> -dist <distfile> [-thresh <thresh>]")])
def test_cli_usage_and_errors(tmp_path, tool, line, usage):
    """Usage on missing or bad arguments (exit 0, the reference's text); a missing input ends in the reference's error line (which
    always shows 1: `err=distgrid(...) != 0`); rasters of different sizes end in "File sizes do not match" and exit status 5, as the
    reference's MPI_Abort(MCW, 5), before any device is needed."""
    import taudem_b200 as td
    rc, out = _run(tool)
    assert rc == 0 and out.startswith("Error: To run this program") and usage in out, out
    bad = [("-bogus", "x"), ("-p", "a.tif", "-src"), ("-p", "a.tif", "-src", "b.tif", "-dist", "c.tif", "-thresh")]
    if tool == "d8hdisttostrm":
        bad.append(("-p", "a.tif", "-fel", "b.tif"))           # d8hdisttostrm has no -fel
    for args in bad:
        rc, out = _run(tool, *args)
        assert rc == 0 and out.startswith("Simple Usage:") and "version" not in out, out
    rc, out = _run(tool, str(tmp_path / "missing.tif"))                  # simple use: missingp.tif
    assert rc == 0 and "missingp.tif" in out and line in out, out
    td.write_raster(str(tmp_path / "p.tif"), np.ones((5, 7), np.int16), -32768)
    td.write_raster(str(tmp_path / "fel.tif"), np.zeros((5, 7), np.float32), -1.0)
    td.write_raster(str(tmp_path / "src.tif"), np.ones((5, 8), np.int32), -1)
    td.write_raster(str(tmp_path / "fel8.tif"), np.zeros((5, 8), np.float32), -1.0)
    td.write_raster(str(tmp_path / "src7.tif"), np.ones((5, 7), np.int32), -1)
    runs = [("-p", str(tmp_path / "p.tif"), "-src", str(tmp_path / "src.tif"), "-dist", str(tmp_path / "d.tif"))]
    if tool == "d8vdisttostrm":
        runs = [r + ("-fel", str(tmp_path / "fel.tif")) for r in runs]
        runs.append(("-p", str(tmp_path / "p.tif"), "-fel", str(tmp_path / "fel8.tif"), "-src", str(tmp_path / "src7.tif"), "-dist", str(tmp_path / "d.tif")))
    for args in runs:
        rc, out = _run(tool, *args)
        assert rc == 5 and "File sizes do not match" in out and line not in out, out
        assert not (tmp_path / "d.tif").exists()


def test_grid_level_shape_checks():
    import taudem_b200 as td
    with pytest.raises(ValueError):
        td.d8hdisttostrm_grid(np.zeros((3, 3), np.int16), np.zeros((3, 4), np.int32))
    with pytest.raises(ValueError):
        td.d8vdisttostrm_grid(np.zeros((3, 3), np.int16), np.zeros((3, 4), np.float32), np.zeros((3, 3), np.int32))
