"""GPU parity: the CUDA path (through the C ABI, host-grid level) against
(a) the committed golden outputs of the reference's own tools and
(b) the recorded outputs of the reference tools on larger seeded inputs (tests/golden/reference.json, tests/reference.py)
Bar: every raster bit for bit, ang and sca included (DESIGN.md §2).  The 1e-5 relative figure that the project states towards
its users is not used here: it cannot see a D-infinity contribution lost or counted twice where a river crosses a tile.
"""
import numpy as np
import pytest

import flat_cases
import pointwise_cases as P
import port
import sibling_cases
import taudem_b200 as td
from taudem_b200 import synth
from util import ANG_ND, FEL_ND, assert_bits, golden_cases, load_golden, write_geographic_dem

pytestmark = pytest.mark.gpu
MISSINGFLOAT = np.float32(-3.4028234663852886e38)


@pytest.mark.parametrize("name", golden_cases())
def test_golden(name):
    g = load_golden(name)
    dx, dy = float(g["dx"]), float(g["dy"])
    assert_bits(td.pitremove_grid(g["dem"]), g["fel"], "fel")
    assert_bits(td.pitremove_grid(g["dem"], is_4Point=True), g["fel4"], "fel -4way")
    p, sd8 = td.d8flowdir_grid(g["fel"], dx=dx, dy=dy)
    assert_bits(sd8, g["sd8"], "sd8")
    assert_bits(p, g["p"], "p")
    ang, slp = td.dinfflowdir_grid(g["fel"], dx=dx, dy=dy)
    assert_bits(slp, g["slp"], "slp")
    assert_bits(ang, g["ang"], "ang")
    assert_bits(td.aread8_grid(g["p"]), g["ad8"], "ad8")
    assert_bits(td.aread8_grid(g["p"], weights=g["w"]), g["ad8_w"], "ad8 -wg")
    assert_bits(td.aread8_grid(g["p"], contcheck=False), g["ad8_nc"], "ad8 -nc")
    assert_bits(td.areadinf_grid(g["ang"], dx=dx, dy=dy), g["sca"], "sca")
    assert_bits(td.areadinf_grid(g["ang"], weights=g["w"], dx=dx, dy=dy), g["sca_w"], "sca -wg")
    assert_bits(td.areadinf_grid(g["ang"], dx=dx, dy=dy, contcheck=False), g["sca_nc"], "sca -nc")


CASES = [
    ("rough768", lambda: synth.gen_dem(768, family="rough", seed=11), 30.0, 30.0),
    ("hills_holes_1000x700", lambda: synth.punch_holes(synth.gen_dem(700, 1000, hurst=0.8, tilt=1.0, seed=5)), 25.0, 40.0),
    ("tilted_odd", lambda: synth.gen_dem(333, 517, family="tilted", seed=2), 30.0, 30.0),
]


@pytest.mark.parametrize("name,make,dx,dy", CASES, ids=[c[0] for c in CASES])
def test_recorded_reference(refrun, name, make, dx, dy):
    dem = make()
    w = synth.gen_weights(*dem.shape)
    R = refrun.RefPipeline(dx=dx, dy=dy, np_ranks=4)
    fel_r = R.pitremove(dem)
    p_r, sd8_r = R.d8flowdir(fel_r)
    ang_r, slp_r = R.dinfflowdir(fel_r)
    # every stage on the reference's input for that stage ...
    assert_bits(td.pitremove_grid(dem), fel_r, "fel")
    p, sd8 = td.d8flowdir_grid(fel_r, dx=dx, dy=dy)
    assert_bits(sd8, sd8_r, "sd8"); assert_bits(p, p_r, "p")
    ang, slp = td.dinfflowdir_grid(fel_r, dx=dx, dy=dy)
    assert_bits(slp, slp_r, "slp"); assert_bits(ang, ang_r, "ang")
    assert_bits(td.aread8_grid(p_r), R.aread8(p_r), "ad8")
    assert_bits(td.aread8_grid(p_r, weights=w, contcheck=False), R.aread8(p_r, weights=w, contcheck=False), "ad8 -wg -nc")
    assert_bits(td.areadinf_grid(ang_r, dx=dx, dy=dy), R.areadinf(ang_r), "sca")
    assert_bits(td.areadinf_grid(ang_r, weights=w, dx=dx, dy=dy), R.areadinf(ang_r, weights=w), "sca -wg")
    # ... and end to end: D8 chain is bit-exact from the raw DEM
    p2, _ = td.d8flowdir_grid(td.pitremove_grid(dem), dx=dx, dy=dy)
    assert_bits(td.aread8_grid(p2), R.aread8(p_r), "ad8 end-to-end")


def test_file_level_cli(refrun, tmp_path):
    """The five executables on files, against the reference executables on the same files."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    bindir = os.path.join(root, "taudem_b200", "bin")
    dem = synth.punch_holes(synth.gen_dem(200, 260, hurst=0.8, tilt=1.0, seed=21))
    R = refrun.RefPipeline(workdir=str(tmp_path / "ref"), dx=30.0, dy=30.0) if os.makedirs(tmp_path / "ref", exist_ok=True) is None else None
    fel_r = R.pitremove(dem); p_r, sd8_r = R.d8flowdir(fel_r); ad8_r = R.aread8(p_r); ang_r, slp_r = R.dinfflowdir(fel_r); sca_r = R.areadinf(ang_r)
    d = tmp_path
    td.write_raster(str(d / "dem.tif"), dem, -9999.0, dx=30.0, dy=30.0)

    def run(tool, *args):
        r = subprocess.run([os.path.join(bindir, tool)] + [str(a) for a in args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0 and "error" not in r.stdout.lower(), r.stdout
        return r.stdout

    out = run("pitremove", "-z", d / "dem.tif", "-fel", d / "demfel.tif")
    assert "PitRemove version" in out and "Compute time" in out
    run("d8flowdir", d / "dem.tif")            # simple usage: demfel.tif -> demp.tif, demsd8.tif
    run("aread8", d / "dem.tif")               # demp.tif -> demad8.tif
    run("dinfflowdir", "-fel", d / "demfel.tif", "-ang", d / "demang.tif", "-slp", d / "demslp.tif")
    run("areadinf", "-ang", d / "demang.tif", "-sca", d / "demsca.tif")
    assert_bits(td.read_raster(str(d / "demfel.tif")), fel_r, "fel file")
    assert_bits(td.read_raster(str(d / "demp.tif"), np.int16), p_r, "p file")
    assert_bits(td.read_raster(str(d / "demsd8.tif")), sd8_r, "sd8 file")
    assert_bits(td.read_raster(str(d / "demad8.tif")), ad8_r, "ad8 file")
    assert_bits(td.read_raster(str(d / "demslp.tif")), slp_r, "slp file")
    assert_bits(td.read_raster(str(d / "demang.tif")), ang_r, "ang file")
    assert_bits(td.read_raster(str(d / "demsca.tif")), sca_r, "sca file")
    # nodata tags round-trip like the reference's (SURVEY.md 8(b) file contract)
    for f, nd in (("demfel.tif", -3.0e38), ("demp.tif", -32768), ("demad8.tif", -1.0), ("demang.tif", ANG_ND)):
        assert np.float32(td.raster_info(str(d / f))["nodata"]) == np.float32(nd)


def test_file_level_cli_multi_gpu(tmp_path):
    """TAUDEM_B200_GPUS=N aread8 / areadinf (the reference's `mpiexec -n N`, src/aread8.cpp:57-100): one forked process per
    GPU with its row strip; the files are bit-identical to the single-GPU run.  With fewer devices than ranks the ranks share
    devices and exchange in rounds (the reference's scheme); with one device per rank the kernels deliver over NVLink."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    bindir = os.path.join(root, "taudem_b200", "bin")
    dem = synth.punch_holes(synth.gen_dem(520, 700, hurst=0.7, tilt=0.6, seed=33))
    fel = td.pitremove_grid(dem, nodata=-9999.0)
    p, _ = td.d8flowdir_grid(fel, dx=30.0, dy=30.0)
    ang, _ = td.dinfflowdir_grid(fel, dx=30.0, dy=30.0)
    rng = np.random.default_rng(5)
    w = rng.uniform(0.0, 3.0, dem.shape).astype(np.float32)
    d = tmp_path
    td.write_raster(str(d / "p.tif"), p, -32768, dx=30.0, dy=30.0)
    td.write_raster(str(d / "ang.tif"), ang, ANG_ND, dx=30.0, dy=30.0)
    td.write_raster(str(d / "w.tif"), w, -9999.0, dx=30.0, dy=30.0)

    def run(gpus, tool, *args):
        env = dict(os.environ, TAUDEM_B200_GPUS=str(gpus))
        r = subprocess.run([os.path.join(bindir, tool)] + [str(a) for a in args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                           timeout=300)
        assert r.returncode == 0 and "error" not in r.stdout.lower(), r.stdout
        return r.stdout

    cases = [("aread8", "ad8", ("-p", d / "p.tif")), ("aread8", "ad8w", ("-p", d / "p.tif", "-wg", d / "w.tif", "-nc")),
             ("areadinf", "sca", ("-ang", d / "ang.tif")), ("areadinf", "scaw", ("-ang", d / "ang.tif", "-wg", d / "w.tif"))]
    for tool, name, args in cases:
        outflag = "-ad8" if tool == "aread8" else "-sca"
        run(1, tool, *args, outflag, d / f"{name}_1.tif")
        one = td.read_raster(str(d / f"{name}_1.tif"))
        for n in (2, 3):
            out = run(n, tool, *args, outflag, d / f"{name}_{n}.tif")
            assert (f"Number of Processes: {n}" if tool == "aread8" else f"Processors: {n}") in out, out
            assert_bits(td.read_raster(str(d / f"{name}_{n}.tif")), one, f"{tool} {name} on {n} ranks")
    assert_bits(td.read_raster(str(d / "ad8_1.tif")), td.aread8_grid(p), "ad8 file vs grid call")


def test_file_level_cli_multi_gpu_flow_directions(tmp_path):
    """TAUDEM_B200_GPUS=N pitremove / d8flowdir / dinfflowdir (the reference's `mpiexec -n N`: src/flood.cpp:344-479 relax + share +
    ringTerm, src/d8.cpp:459-680 resolveflats with share() / MPI_Allreduce per pass): forked ranks with one row strip each, the
    row exchanges and sums staged through a shared mapping; every file bit-identical to the single-GPU run (flats included:
    a rough DEM with a third of its cells flat, lakes crossing the strip boundaries)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    bindir = os.path.join(root, "taudem_b200", "bin")
    dem = synth.punch_holes(synth.gen_dem(410, 530, hurst=0.6, tilt=0.1, seed=35))
    rng = np.random.default_rng(6)
    mask = (rng.random(dem.shape) < 0.01).astype(np.int16)
    d = tmp_path
    td.write_raster(str(d / "dem.tif"), dem, -9999.0, dx=30.0, dy=25.0)
    td.write_raster(str(d / "mask.tif"), mask, -32768, dx=30.0, dy=25.0)

    def run(gpus, tool, *args):
        env = dict(os.environ, TAUDEM_B200_GPUS=str(gpus))
        r = subprocess.run([os.path.join(bindir, tool)] + [str(a) for a in args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                           timeout=600)
        assert r.returncode == 0 and "error" not in r.stdout.lower(), r.stdout
        return r.stdout

    for n in (1, 2, 3):
        run(n, "pitremove", "-z", d / "dem.tif", "-fel", d / f"fel_{n}.tif")
        run(n, "pitremove", "-z", d / "dem.tif", "-fel", d / f"fel4m_{n}.tif", "-4way", "-depmask", d / "mask.tif")
        out = run(n, "d8flowdir", "-fel", d / "fel_1.tif", "-p", d / f"p_{n}.tif", "-sd8", d / f"sd8_{n}.tif")
        assert f"Processors: {n}" in out, out
        run(n, "dinfflowdir", "-fel", d / "fel_1.tif", "-ang", d / f"ang_{n}.tif", "-slp", d / f"slp_{n}.tif")
    for name, dt in (("fel", np.float32), ("fel4m", np.float32), ("p", np.int16), ("sd8", np.float32), ("ang", np.float32), ("slp", np.float32)):
        one = td.read_raster(str(d / f"{name}_1.tif"), dt)
        for n in (2, 3):
            assert_bits(td.read_raster(str(d / f"{name}_{n}.tif"), dt), one, f"{name} on {n} ranks")
    p = td.read_raster(str(d / "p_1.tif"), np.int16)
    assert (p == 0).sum() == 0 and (td.read_raster(str(d / "sd8_1.tif")) == 0).mean() > 0.05      # flats existed and were all resolved
    assert_bits(td.read_raster(str(d / "fel_1.tif")), td.pitremove_grid(dem), "fel file vs grid call")


def test_properties_large():
    """Size-independent properties at a size the CPU reference cannot reach quickly (4096^2):
    fill is idempotent and never lowers a cell; every resolved D8 direction points to a cell that
    is not higher; D8 area (no contamination check) is conserved: the area leaving the grid equals
    the number of cells."""
    n = 4096
    dem = synth.gen_dem(n, hurst=0.8, tilt=1.0, seed=77)
    fel = td.pitremove_grid(dem)
    assert (fel >= dem).all()
    assert_bits(td.pitremove_grid(fel, nodata=-9999.0), fel, "fill idempotence")
    p, sd8 = td.d8flowdir_grid(fel)
    d1 = np.array([0, 1, 1, 0, -1, -1, -1, 0, 1]); d2 = np.array([0, 0, -1, -1, -1, 0, 1, 1, 1])
    yy, xx = np.nonzero((p >= 1) & (p <= 8))
    k = p[yy, xx]
    assert (fel[yy + d2[k], xx + d1[k]] <= fel[yy, xx]).all()
    assert (sd8[(p >= 1) & (p <= 8)] >= 0).all()
    ad8 = td.aread8_grid(p, contcheck=False)
    valid = (p >= 1) & (p <= 8)
    ty, tx = yy + d2[k], xx + d1[k]
    leaves = ~valid[ty, tx]                     # cells whose downslope neighbour is an edge/nodata cell
    total = ad8[yy[leaves], xx[leaves]].astype(np.float64).sum()
    assert abs(total - valid.sum()) <= 1e-3 * valid.sum(), (total, valid.sum())
    assert ad8[valid].min() >= 1.0


@pytest.fixture(scope="module")
def crossings():
    """the 2100 x 3000 DEM of the tile-crossing tests: (fel, p, sd8, ang) of the C restatement"""
    dem = synth.punch_holes(synth.gen_dem(2100, 3000, hurst=0.8, tilt=1.0, seed=9))
    fel = port.pitremove(dem)
    p, sd8 = port.d8flowdir(fel)
    ang, _ = port.dinfflowdir(fel)
    return fel, p, sd8, ang


def test_sweep_with_many_tile_crossings_matches_the_reference(refrun, crossings):
    """2100 x 3000 cells (6 200 tiles of the dataflow sweep, rivers that cross hundreds of tiles, thousands of tile
    re-activations): ad8 and sca bit for bit, with and without weights, against the reference tools."""
    fel, p, _, ang = crossings
    w = synth.gen_weights(*p.shape)
    R = refrun.RefPipeline(np_ranks=8)
    ad8 = td.aread8_grid(p)
    assert_bits(ad8, R.aread8(p), "ad8")
    assert_bits(td.aread8_grid(p, weights=w, contcheck=False), R.aread8(p, weights=w, contcheck=False), "ad8 -wg -nc")
    assert_bits(td.areadinf_grid(ang), R.areadinf(ang), "sca")
    assert_bits(td.areadinf_grid(ang, weights=w, contcheck=False), R.areadinf(ang, weights=w, contcheck=False), "sca -wg -nc")
    assert ad8.max() > 1e5


@pytest.mark.parametrize("world", [2, 3])
def test_row_strip_partition_matches_single_strip(world):
    """Rank-count invariance of the row-strip partition (SURVEY.md A.6): `world` processes, each owning
    one strip (uneven last strip, partial tiles at the strip edge), reproduce the single-strip rasters
    bit for bit.  On a one-GPU box the ranks share cuda:0 and exchange halos through gloo; on the
    multi-GPU box scripts/dist_check.py runs the same check over NCCL."""
    import os
    import socket
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
    env = dict(os.environ, TD_BACKEND="gloo")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(root, "scripts", "dist_check.py"), "1001", "1300"],
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "DIFFERENT" not in r.stdout and r.stdout.count("identical") == 9, r.stdout[-3000:]


def test_edge_shapes_against_c_restatement():
    """Degenerate and awkward shapes, checked against the pinned C restatement (oracle/port): a single
    row / column (everything is edge), 2-row and 3-row grids, widths that are not multiples of the
    vector width or of the tile size, an all-nodata grid, a grid whose border is nodata, a constant grid."""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    rng = np.random.default_rng(4)
    shapes = [(1, 9), (9, 1), (2, 5), (3, 3), (3, 70), (33, 65), (64, 129), (31, 257)]
    grids = [(rng.random(s) * 50).astype(np.float32) for s in shapes]
    ring = (rng.random((40, 37)) * 30).astype(np.float32); ring[0, :] = ring[-1, :] = ring[:, 0] = ring[:, -1] = -9999.0
    grids += [np.full((12, 19), -9999.0, np.float32), ring, np.full((20, 21), 7.0, np.float32)]
    for dem in grids:
        w = rng.random(dem.shape).astype(np.float32)
        fel = td.pitremove_grid(dem)
        assert_bits(fel, port.pitremove(dem), f"fel {dem.shape}")
        p, sd8 = td.d8flowdir_grid(fel, dx=10.0, dy=12.0)
        p_o, sd8_o = port.d8flowdir(fel, dx=10.0, dy=12.0)
        assert_bits(p, p_o, f"p {dem.shape}"); assert_bits(sd8, sd8_o, f"sd8 {dem.shape}")
        ang, slp = td.dinfflowdir_grid(fel, dx=10.0, dy=12.0)
        ang_o, slp_o = port.dinfflowdir(fel, dx=10.0, dy=12.0)
        assert_bits(slp, slp_o, f"slp {dem.shape}"); assert_bits(ang, ang_o, f"ang {dem.shape}")
        assert_bits(td.aread8_grid(p_o, weights=w), port.aread8(p_o, weights=w), f"ad8 {dem.shape}")
        assert_bits(td.areadinf_grid(ang_o, dx=10.0, dy=12.0), port.areadinf(ang_o, dx=10.0, dy=12.0), f"sca {dem.shape}")


def test_odd_direction_codes_and_nodata_weights():
    """aread8 quirks of the reference that a real p raster can contain (SURVEY.md A.6/A.7): unresolved
    flats (0), out-of-range codes, a nodata value other than -32768, nodata weights."""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    rng = np.random.default_rng(8)
    p = rng.integers(-3, 13, size=(70, 90)).astype(np.int16)
    p[rng.random(p.shape) < 0.05] = -1
    w = rng.random(p.shape).astype(np.float32); w[rng.random(p.shape) < 0.1] = -5.0
    for cont in (True, False):
        assert_bits(td.aread8_grid(p, nodata=-1, weights=w, w_nodata=-5.0, contcheck=cont),
                    port.aread8(p, nodata=-1, weights=w, w_nodata=-5.0, contcheck=cont), f"ad8 contcheck={cont}")


def test_large_vs_c_restatement():
    """1500 x 1100 hills DEM end to end against the C restatement (seconds on one CPU core)."""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    dem = synth.punch_holes(synth.gen_dem(1100, 1500, hurst=0.8, tilt=1.0, seed=31))
    fel = td.pitremove_grid(dem); assert_bits(fel, port.pitremove(dem), "fel")
    p, sd8 = td.d8flowdir_grid(fel); p_o, sd8_o = port.d8flowdir(fel)
    assert_bits(p, p_o, "p"); assert_bits(sd8, sd8_o, "sd8")
    assert_bits(td.aread8_grid(p), port.aread8(p_o), "ad8")
    ang, slp = td.dinfflowdir_grid(fel); ang_o, slp_o = port.dinfflowdir(fel)
    assert_bits(slp, slp_o, "slp"); assert_bits(ang, ang_o, "ang")
    assert_bits(td.areadinf_grid(ang_o), port.areadinf(ang_o), "sca")


def test_depression_mask():
    """pitremove -depmask (src/flood.cpp:75-85, 250-251): masked cells are seeds and keep their elevation."""
    g = load_golden("lake")
    assert_bits(td.pitremove_grid(g["dem"], depmask=g["depmask"]), g["fel_mask"], "fel -depmask")
    assert_bits(td.pitremove_grid(g["dem"], depmask=g["depmask"], is_4Point=True), g["fel_mask4"], "fel -depmask -4way")
    # and a partial mask on a larger grid against the C restatement
    import port
    if port.available():
        dem = synth.gen_dem(300, 420, family="rough", seed=3)
        mask = (synth.gen_weights(300, 420, seed=17) > 0.97).astype(np.int16)
        assert_bits(td.pitremove_grid(dem, depmask=mask), port.pitremove(dem, depmask=mask), "fel -depmask rough")


def test_geographic_dem_file_level(refrun, tmp_path):
    """A DEM in geographic coordinates through the file-level entry points: per-row cell sizes on the
    ellipsoid (src/tiffIO.cpp:118-151) reach every kernel; rasters against the reference tools'."""
    import os
    dem = synth.punch_holes(synth.gen_dem(150, 210, hurst=0.8, tilt=1.0, seed=12))
    d = str(tmp_path)
    write_geographic_dem(os.path.join(d, "geo.tif"), dem)
    q = lambda n: os.path.join(d, n)
    # the reference tools' chain on the file, pinned bit for bit on the C restatement with the file's per-row cell sizes
    import ctypes
    ny = dem.shape[0]
    dxc, dyc = np.zeros(ny), np.zeros(ny)
    assert td.lib().td_raster_cell_sizes(q("geo.tif").encode(), dxc.ctypes.data_as(ctypes.c_void_p), dyc.ctypes.data_as(ctypes.c_void_p), ny) == 0
    x = {"dem": dem, "fel": port.pitremove(dem)}
    x["p"], x["sd8"] = port.d8flowdir(x["fel"], dx=dxc, dy=dyc)
    x["ang"], x["slp"] = port.dinfflowdir(x["fel"], dx=dxc, dy=dyc)
    x["ad8"], x["sca"] = port.aread8(x["p"]), port.areadinf(x["ang"], dx=dxc, dy=dyc)
    os.makedirs(q("ref"))
    for tool, args, ins, outs in (("pitremove", ["-z", "geo.tif", "-fel", "{o}fel.tif"], ["dem"], ["fel"]),
                                  ("d8flowdir", ["-fel", "{o}fel.tif", "-p", "{o}p.tif", "-sd8", "{o}sd8.tif"], ["fel"], ["p", "sd8"]),
                                  ("dinfflowdir", ["-fel", "{o}fel.tif", "-ang", "{o}ang.tif", "-slp", "{o}slp.tif"], ["fel"], ["ang", "slp"]),
                                  ("aread8", ["-p", "{o}p.tif", "-ad8", "{o}ad8.tif"], ["p"], ["ad8"]), ("areadinf", ["-ang", "{o}ang.tif", "-sca", "{o}sca.tif"], ["ang"], ["sca"])):
        got = refrun.run_tool_outputs(tool, [q(a.format(o="ref/")) if a.endswith(".tif") else a for a in args], [q(f"ref/{n}.tif") for n in outs],
                                      [np.int16 if n == "p" else np.float32 for n in outs], [x[i] for i in ins])
        for n, r in zip(outs, got):
            assert_bits(x[n], r, n + " (geographic, reference tools)")
    assert td.flood(q("geo.tif"), q("fel.tif")) == 0
    assert td.setdird8(q("fel.tif"), q("p.tif"), q("sd8.tif")) == 0
    assert td.setdir(q("fel.tif"), q("ang.tif"), q("slp.tif")) == 0
    assert td.aread8(q("p.tif"), q("ad8.tif")) == 0
    assert td.area(q("ang.tif"), q("sca.tif")) == 0
    for n, dt in (("fel", np.float32), ("p", np.int16), ("sd8", np.float32), ("slp", np.float32), ("ad8", np.float32), ("ang", np.float32),
                  ("sca", np.float32)):
        assert_bits(td.read_raster(q(n + ".tif"), dt), x[n], n + " (geographic)")
    assert td.raster_info(q("sca.tif"))["is_geographic"]        # GeoTIFF keys pass through to the outputs
    # the same on row strips (TAUDEM_B200_GPUS=N behind the executables): rows of different cell sizes on both sides of a strip
    # boundary — the halo row of a strip is evaluated with the neighbour row's cell sizes like the reference does (getdxdyc(jn))
    import subprocess
    bindir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "taudem_b200", "bin")
    for n in (2, 3):
        env = dict(os.environ, TAUDEM_B200_GPUS=str(n))
        for tool, args in (("pitremove", ["-z", q("geo.tif"), "-fel", q(f"fel_{n}.tif")]),
                           ("d8flowdir", ["-fel", q("fel.tif"), "-p", q(f"p_{n}.tif"), "-sd8", q(f"sd8_{n}.tif")]),
                           ("dinfflowdir", ["-fel", q("fel.tif"), "-ang", q(f"ang_{n}.tif"), "-slp", q(f"slp_{n}.tif")]),
                           ("aread8", ["-p", q("p.tif"), "-ad8", q(f"ad8_{n}.tif")]), ("areadinf", ["-ang", q("ang.tif"), "-sca", q(f"sca_{n}.tif")])):
            r = subprocess.run([os.path.join(bindir, tool)] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=300)
            assert r.returncode == 0 and "error" not in r.stdout.lower(), r.stdout
        for name, dt in (("fel", np.float32), ("p", np.int16), ("sd8", np.float32), ("ang", np.float32), ("slp", np.float32), ("ad8", np.float32), ("sca", np.float32)):
            assert_bits(td.read_raster(q(f"{name}_{n}.tif"), dt), td.read_raster(q(name + ".tif"), dt), f"{name} (geographic) on {n} ranks")


def test_d8_stencil_ties_and_near_ties():
    """Exact ties and drops that are adjacent floats whose slopes round to the same float32 (the literal fallback of
    d8_cell): p and sd8 of the positive-slope pass + flats against the C restatement.  Same grids as
    tests/test_emu.py::test_emulated_d8_stencil_ties_and_near_ties."""
    from oracle import port
    rng = np.random.default_rng(5)
    ny, nx = 96, 128
    base = (1000.0 + rng.integers(0, 4, (ny, nx)) * 2.5).astype(np.float32)
    grids = [(base.view(np.int32) + rng.integers(-3, 4, (ny, nx)).astype(np.int32)).view(np.float32)]
    rng = np.random.default_rng(7)
    ny, nx = 192, 256
    g = (10.0 + rng.integers(0, 2, (ny, nx)) * 16.0 + rng.integers(-4, 5, (ny, nx)) * 3.0e-5).astype(np.float32)
    g[1::3, 1::3] = (np.float32(1000.0).view(np.int32) + rng.integers(-2, 3, g[1::3, 1::3].shape).astype(np.int32)).view(np.float32)
    grids.append(g)
    for fel in grids:
        for dx, dy in ((30.0, 30.0), (12.5, 40.0), (7.0, 7.1)):
            p, sd8 = td.d8flowdir_grid(fel, dx=dx, dy=dy)
            p_ref, sd8_ref = port.d8flowdir(fel, dx=dx, dy=dy)
            assert_bits(p, p_ref, f"p ties {dx}x{dy}"); assert_bits(sd8, sd8_ref, f"sd8 ties {dx}x{dy}")


def test_overlapped_two_tool_call_equals_the_two_calls():
    """td_contributing_areas_host (aread8 + areadinf of one DEM, copies overlapped with the kernels on three streams) returns
    exactly what td_aread8_host and td_area_host return."""
    dem = synth.punch_holes(synth.gen_dem(700, 900, hurst=0.8, tilt=1.0, seed=23))
    fel = td.pitremove_grid(dem); p, _ = td.d8flowdir_grid(fel, dx=25.0, dy=35.0); ang, _ = td.dinfflowdir_grid(fel, dx=25.0, dy=35.0)
    ad8, sca = td.contributing_areas_grid(p, ang, dx=25.0, dy=35.0)
    assert_bits(ad8, td.aread8_grid(p), "ad8 (overlapped call)")
    assert_bits(sca, td.areadinf_grid(ang, dx=25.0, dy=35.0), "sca (overlapped call)")
    ad8, sca = td.contributing_areas_grid(p, ang, dx=25.0, dy=35.0, contcheck=False)
    assert_bits(ad8, td.aread8_grid(p, contcheck=False), "ad8 -nc (overlapped call)")
    assert_bits(sca, td.areadinf_grid(ang, dx=25.0, dy=35.0, contcheck=False), "sca -nc (overlapped call)")


def _bin(tool):
    import os
    return os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "taudem_b200", "bin", tool)


def _run(tool, *args):
    import subprocess
    r = subprocess.run([_bin(tool)] + [str(a) for a in args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "rror" not in r.stdout, r.stdout


def _reference(refrun, calls, workdir):
    """the reference outputs of a sibling case's calls (tests/sibling_cases.py), by label"""
    R = refrun.RefPipeline(workdir=str(workdir))
    return {label: getattr(R, tool)(*args, **kw) for label, tool, args, kw in calls}


def test_d8_flow_path_extreme_up(refrun, tmp_path):
    """d8flowpathextremeup (SURVEY.md 8(f) rank 3: a sibling of aread8 on the same sweep) against the reference's outputs (replayed by
    the C restatement, tests/reference.py): max, min, -nc, outlets; grid level and our executable, bit for bit."""
    x, calls = sibling_cases.flowpathextremeup(tmp_path)
    ref = _reference(refrun, calls, tmp_path)
    p, sa, outs = x["p"], x["sa"], (x["cols"], x["rows"])
    assert_bits(td.d8flowpathextremeup_grid(p, sa), ref["ssa max"], "ssa max")
    assert_bits(td.d8flowpathextremeup_grid(p, x["fel"], usemax=False, contcheck=False), ref["ssa min -nc"], "ssa min -nc")
    assert_bits(td.d8flowpathextremeup_grid(p, sa, outlets=outs), ref["ssa max -o"], "ssa max -o")
    out = str(tmp_path / "ours_ssa.tif")
    _run("d8flowpathextremeup", "-p", tmp_path / "pin.tif", "-sa", tmp_path / "sa.tif", "-ssa", out, "-o", x["shp"])
    assert_bits(td.read_raster(out), ref["ssa max -o"], "d8flowpathextremeup -o (files)")


def test_gridnet(refrun, tmp_path):
    """gridnet (SURVEY.md 8(f) rank 3: a sibling of aread8 on the same sweep) against the reference's outputs: plain, mask + threshold,
    outlets, outlets + mask; grid level and our executable, bit for bit."""
    x, calls = sibling_cases.gridnet(tmp_path)
    ref = _reference(refrun, calls, tmp_path)
    p, mask, outs = x["p"], x["mask"], (x["cols"], x["rows"])

    def same(ours, want, what):
        for a, b, n in zip(ours, want, ("plen", "tlen", "gord")):
            assert_bits(a, b, f"{n} {what}")

    same(td.gridnet_grid(p), ref[""], "")
    same(td.gridnet_grid(p, mask=mask, thresh=20), ref["-mask -thresh 20"], "-mask -thresh 20")
    same(td.gridnet_grid(p, outlets=outs), ref["-o"], "-o")
    same(td.gridnet_grid(p, mask=mask, thresh=20, outlets=outs), ref["-o -mask"], "-o -mask")
    o = {n: str(tmp_path / f"ours_{n}.tif") for n in ("plen", "tlen", "gord")}
    _run("gridnet", "-p", tmp_path / "pin.tif", "-plen", o["plen"], "-tlen", o["tlen"], "-gord", o["gord"], "-o", x["shp"], "-mask", tmp_path / "mask.tif",
         "-thresh", "20")
    same((td.read_raster(o["plen"]), td.read_raster(o["tlen"]), td.read_raster(o["gord"], np.int16)), ref["-o -mask"], "-o -mask (files)")


def test_dinf_decay_accumulation(refrun, tmp_path):
    """dinfdecayaccum (SURVEY.md 8(f) rank 3: a sibling of areadinf on the same sweep) against the reference's outputs: plain,
    weights + -nc, nodata multipliers, outlets; grid level and our executable, bit for bit."""
    x, calls = sibling_cases.dinfdecayaccum(tmp_path)
    ref = _reference(refrun, calls, tmp_path)
    ang, dm = x["ang"], x["dm"]
    assert_bits(td.dinfdecayaccum_grid(ang, dm), ref["dsca"], "dsca")
    assert_bits(td.dinfdecayaccum_grid(ang, dm, weights=x["w"], contcheck=False), ref["dsca -wg -nc"], "dsca -wg -nc")
    assert_bits(td.dinfdecayaccum_grid(ang, dm, outlets=(x["cols"], x["rows"])), ref["dsca -o"], "dsca -o")
    out = str(tmp_path / "ours_dsca.tif")
    _run("dinfdecayaccum", "-ang", tmp_path / "angin.tif", "-dm", tmp_path / "dm.tif", "-dsca", out, "-o", x["shp"])
    assert_bits(td.read_raster(out), ref["dsca -o"], "dinfdecayaccum -o (files)")


def test_dinf_conc_lim_and_trans_lim_accumulation(refrun, tmp_path):
    """DinfConcLimAccum and DinfTransLimAccum (SURVEY.md 8(f) rank 3: the last two siblings of areadinf on the same sweep) against the
    reference's outputs: with and without contamination checking, with and without the concentration that travels with the transport,
    outlets; grid level and our executables, bit for bit."""
    x, calls = sibling_cases.conc_and_trans_lim(tmp_path)
    ref = _reference(refrun, calls, tmp_path)
    ang, q, dm, dg, tc, cs, outs = x["ang"], x["q"], x["dm"], x["dg"], x["tc"], x["cs"], (x["cols"], x["rows"])
    # concentration limited
    assert_bits(td.dinfconclimaccum_grid(ang, dm, q, dg, csol=2.5), ref["ctpt"], "ctpt")
    assert_bits(td.dinfconclimaccum_grid(ang, dm, q, dg, contcheck=False), ref["ctpt -nc"], "ctpt -nc")
    assert_bits(td.dinfconclimaccum_grid(ang, dm, q, dg, csol=0.75, contcheck=False, outlets=outs), ref["ctpt -o"], "ctpt -o")
    out = str(tmp_path / "ours_ctpt.tif")
    _run("dinfconclimaccum", "-ang", tmp_path / "angin.tif", "-dm", tmp_path / "dm.tif", "-q", tmp_path / "q.tif", "-dg", tmp_path / "dg.tif", "-ctpt", out,
         "-csol", "0.75", "-nc", "-o", x["shp"])
    assert_bits(td.read_raster(out), ref["ctpt -o"], "dinfconclimaccum -o (files)")
    assert (td.read_raster(out) != MISSINGFLOAT).mean() > 0.02
    # transport limited
    tsup = q
    for kw in ({}, {"contcheck": False}, {"cs": cs}, {"cs": cs, "contcheck": False}):
        ours = td.dinftranslimaccum_grid(ang, tsup, tc, **kw)
        for o, f, name in zip(ours, ref[f"translim {sorted(kw)}"], ("tla", "tdep", "ctpt")):
            if f is not None:
                assert_bits(o, f, f"{name} {kw.keys()}")
    assert (ours[0] != MISSINGFLOAT).mean() > 0.5 and (ours[1] > 0).mean() > 0.1
    refs = ref["translim -cs -nc -o"]
    ours = td.dinftranslimaccum_grid(ang, tsup, tc, cs=cs, contcheck=False, outlets=outs)
    for o, f, name in zip(ours, refs, ("tla", "tdep", "ctpt")):
        assert_bits(o, f, name + " -o")
    outs = [str(tmp_path / f"ours_{n}.tif") for n in ("tla", "tdep", "ctptout")]
    _run("dinftranslimaccum", "-ang", tmp_path / "angin.tif", "-tsup", tmp_path / "tsup.tif", "-tc", tmp_path / "tc.tif", "-cs", tmp_path / "cs.tif",
         "-ctpt", outs[2], "-tla", outs[0], "-tdep", outs[1], "-nc", "-o", x["shp"])
    for o, f, name in zip(outs, refs, ("tla", "tdep", "ctpt")):
        assert_bits(td.read_raster(o), f, name + " -o (files)")


def test_pointwise_consumers_threshold_and_twi(refrun, tmp_path):
    """threshold and twi (SURVEY.md 8(f) rank 4) on the rasters of the path: grid level and our executables against the
    reference executables (oracle/_ref/threshold, oracle/_ref/twi: Threshold.cpp / TWI.cpp compiled unchanged).  src is
    bit-exact; twi = ln(sca / slp) is correctly rounded, so it differs from glibc's logf exactly where logf is not correctly
    rounded (tests/pointwise_cases.py)."""
    import os
    import subprocess
    dem = synth.punch_holes(synth.gen_dem(300, 380, hurst=0.8, tilt=1.0, seed=31))
    fel = port.pitremove(dem); p, _ = port.d8flowdir(fel); ang, slp = port.dinfflowdir(fel)
    ad8 = port.aread8(p); sca = port.areadinf(ang)
    mask = (synth.gen_weights(*dem.shape) - 0.3).astype(np.float32)          # negative on ~30 % of the cells
    R = refrun.RefPipeline(workdir=str(tmp_path))
    assert_bits(td.threshold_grid(ad8, 50.0), R.threshold(ad8, 50.0), "src")
    src_ref = R.threshold(ad8, 7.5, mask=mask)
    assert_bits(td.threshold_grid(ad8, 7.5, mask=mask), src_ref, "src -mask")
    twi, ref = td.twi_grid(slp, sca), R.twi(slp, sca)
    assert_bits(P.twi(slp, sca), ref, "twi restatement with libm's logf")
    P.assert_log_pow_contract(twi, P.twi(slp, sca), P.twi(slp, sca, libm=False), "twi")
    # executables on the files the reference run left in tmp_path
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "ours_src.tif")
    r = subprocess.run([os.path.join(root, "taudem_b200", "bin", "threshold"), "-ssa", str(tmp_path / "ssa.tif"), "-src", out, "-thresh", "7.5",
                        "-mask", str(tmp_path / "mask.tif")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert_bits(td.read_raster(out, np.int16), src_ref, "threshold (files)")
    out = str(tmp_path / "ours_twi.tif")
    r = subprocess.run([os.path.join(root, "taudem_b200", "bin", "twi"), "-slp", str(tmp_path / "slpin.tif"), "-sca", str(tmp_path / "scain.tif"), "-twi", out],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    assert_bits(td.read_raster(out), twi, "twi (files)")


def test_pointwise_consumers_slopearea_and_slopearearatio(refrun, tmp_path):
    """slopearea and slopearearatio (the other two tools of SURVEY.md 8(f) rank 4): grid level and our executables against the
    reference executables (SlopeArea.cpp / SlopeAreaRatio.cpp compiled unchanged).  sar = slp / sca is bit-exact; sa = slp^m * sca^n
    is a product of two powf results in the reference; ours of two correctly rounded powers, so it differs exactly where a powf is
    not correctly rounded (tests/pointwise_cases.py)."""
    import os
    import subprocess
    dem = synth.punch_holes(synth.gen_dem(260, 420, hurst=0.8, tilt=1.0, seed=37))
    fel = port.pitremove(dem); ang, slp = port.dinfflowdir(fel); sca = port.areadinf(ang)
    R = refrun.RefPipeline(workdir=str(tmp_path))
    with np.errstate(all="ignore"):
        sar_ref = R.slopearearatio(slp, sca)
        assert_bits(td.slopearearatio_grid(slp, sca), sar_ref, "sar")
    for m, n in ((None, None), (0.5, 1.75)):
        ours = td.slopearea_grid(slp, sca) if m is None else td.slopearea_grid(slp, sca, m, n)
        ref = R.slopearea(slp, sca, m, n)
        mm, nn = (2.0, 1.0) if m is None else (m, n)
        assert_bits(P.slopearea(slp, sca, mm, nn), ref, "slopearea restatement with libm's powf")
        P.assert_log_pow_contract(ours, P.slopearea(slp, sca, mm, nn), P.slopearea(slp, sca, mm, nn, libm=False), f"slopearea {m} {n}")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "ours_sa.tif")
    r = subprocess.run([os.path.join(root, "taudem_b200", "bin", "slopearea"), "-slp", str(tmp_path / "slpin.tif"), "-sca", str(tmp_path / "scain.tif"), "-sa", out,
                        "-par", "0.5", "1.75"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "rror" not in r.stdout, r.stdout
    assert_bits(td.read_raster(out), ours, "slopearea (files)")
    out = str(tmp_path / "ours_sar.tif")
    r = subprocess.run([os.path.join(root, "taudem_b200", "bin", "slopearearatio"), "-slp", str(tmp_path / "slpin.tif"), "-sca", str(tmp_path / "scain.tif"), "-sar", out],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "rror" not in r.stdout, r.stdout
    assert_bits(td.read_raster(out), sar_ref, "slopearearatio (files)")


def test_dinf_angle_torture():
    """areadinf on angles at and next to every place where prop() changes its mind (sector edges, the 1e-5 share threshold, the
    wrap sector, angles beyond 2 PI), bit for bit against the C restatement (pinned on the reference tools by the CPU suite)."""
    from oracle import port
    from util import angle_torture
    for dx, dy in ((30.0, 30.0), (12.5, 40.0)):
        ang = angle_torture(ny=200, nx=330, dx=dx, dy=dy)
        assert_bits(td.areadinf_grid(ang, dx=dx, dy=dy), port.areadinf(ang, dx=dx, dy=dy), f"sca angle torture {dx}x{dy}")
        assert_bits(td.areadinf_grid(ang, dx=dx, dy=dy, contcheck=False), port.areadinf(ang, dx=dx, dy=dy, contcheck=False), f"sca angle torture -nc {dx}x{dy}")


def test_outlets_grid_and_file_level(refrun, tmp_path):
    """aread8 / areadinf -o: the cells upstream of the outlets only.  Grid level against the C restatement (which the
    CPU suite pins on the reference tools), file level (our executables with a point shapefile) against the reference
    executables on the same files."""
    import os
    import subprocess
    from oracle import port
    from util import write_point_shapefile
    dem = synth.punch_holes(synth.gen_dem(300, 420, hurst=0.8, tilt=1.0, seed=15))
    fel = port.pitremove(dem); p, _ = port.d8flowdir(fel); ang, _ = port.dinfflowdir(fel)
    w = synth.gen_weights(*dem.shape)
    ny, nx = p.shape
    order = np.argsort(port.aread8(p).ravel())
    cells = [int(order[-1]), int(order[-60]), int(order[-900]), int(order[len(order) // 2])]
    cols = [c % nx for c in cells] + [-4]; rows = [c // nx for c in cells] + [7]
    outs = (cols, rows)
    assert_bits(td.aread8_grid(p, outlets=outs), port.aread8(p, outlets=outs), "ad8 -o")
    assert_bits(td.aread8_grid(p, weights=w, contcheck=False, outlets=outs), port.aread8(p, weights=w, contcheck=False, outlets=outs), "ad8 -o -wg -nc")
    assert_bits(td.areadinf_grid(ang, outlets=outs), port.areadinf(ang, outlets=outs), "sca -o")
    assert_bits(td.aread8_grid(p, outlets=([], [])), np.full(p.shape, -1.0, np.float32), "ad8 -o, no points")
    # file level
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    dx = dy = 30.0
    xs = [(c + 0.5) * dx for c in cols]; ys = [dy * ny - (r + 0.5) * dy for r in rows]
    shp = str(tmp_path / "outlets.shp")
    write_point_shapefile(shp, xs, ys)
    R = refrun.RefPipeline(workdir=str(tmp_path), dx=dx, dy=dy)
    ad8_ref = R.aread8(p, outlets=shp); sca_ref = R.areadinf(ang, outlets=shp)
    for tool, inflag, infile, outflag, ref in (("aread8", "-p", "pin.tif", "-ad8", ad8_ref), ("areadinf", "-ang", "angin.tif", "-sca", sca_ref)):
        out = str(tmp_path / f"ours_{tool}.tif")
        r = subprocess.run([os.path.join(root, "taudem_b200", "bin", tool), inflag, str(tmp_path / infile), outflag, out, "-o", shp],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
        assert_bits(td.read_raster(out), ref, f"{tool} -o (files)")


# ---- the sibling sweep tools (algebras 1-9 of k_sweep_warp, sweep_warp.cu) against the C restatement (oracle/port), which the CPU suite
#      pins on the reference's outputs: cell-level diffs at the shapes, sizes and values where the kernels could go wrong.
def _sibling_values(rng, shape):
    """value grids with nodata (-9999), zero and negative values"""
    def vals(lo, hi, zero=0.03, nd=0.02):
        v = rng.uniform(lo, hi, shape).astype(np.float32)
        v[rng.random(shape) < zero] = 0.0
        v[rng.random(shape) < nd] = -9999.0
        return v
    return dict(sa=vals(-50.0, 50.0), dm=vals(-0.2, 1.2), w=vals(-0.5, 2.0), q=vals(-0.5, 3.0), tc=vals(-0.5, 6.0), cs=vals(-0.2, 2.0),
                dg=(rng.random(shape) < 0.05).astype(np.int16), mask=rng.integers(-1, 4, shape).astype(np.int32))


def _check_siblings(p, ang, v, what, dx=30.0, dy=30.0, dxc=None, dyc=None, contchecks=(True, False), outlets=None, algs=range(1, 10), thresh=1):
    """the nine algebras on (p, ang) with the value grids v, GPU against the restatement, bit for bit"""
    sz = dict(dx=dx, dy=dy, dxc=dxc, dyc=dyc)
    for cont in contchecks:
        tag = f"{what} contcheck={cont}"
        for alg, usemax in ((1, True), (2, False)):
            if alg in algs:
                assert_bits(td.d8flowpathextremeup_grid(p, v["sa"], usemax=usemax, contcheck=cont, outlets=outlets),
                            port.d8flowpathextremeup(p, v["sa"], usemax=usemax, contcheck=cont, outlets=outlets), f"ssa usemax={usemax} {tag}")
        if 3 in algs:
            assert_bits(td.dinfdecayaccum_grid(ang, v["dm"], contcheck=cont, outlets=outlets, **sz),
                        port.dinfdecayaccum(ang, v["dm"], contcheck=cont, outlets=outlets, **sz), f"dsca {tag}")
            assert_bits(td.dinfdecayaccum_grid(ang, v["dm"], weights=v["w"], contcheck=cont, outlets=outlets, **sz),
                        port.dinfdecayaccum(ang, v["dm"], weights=v["w"], contcheck=cont, outlets=outlets, **sz), f"dsca -wg {tag}")
        if 7 in algs:
            assert_bits(td.dinfconclimaccum_grid(ang, v["dm"], v["q"], v["dg"], csol=1.5, contcheck=cont, outlets=outlets, **sz),
                        port.dinfconclimaccum(ang, v["dm"], v["q"], v["dg"], csol=1.5, contcheck=cont, outlets=outlets, **sz), f"ctpt {tag}")
        for alg, cs in ((8, None), (9, v["cs"])):
            if alg in algs:
                for o, r, n in zip(td.dinftranslimaccum_grid(ang, v["q"], v["tc"], cs=cs, contcheck=cont, outlets=outlets, **sz),
                                   port.dinftranslimaccum(ang, v["q"], v["tc"], cs=cs, contcheck=cont, outlets=outlets, **sz), ("tla", "tdep", "ctpt")):
                    if r is not None:
                        assert_bits(o, r, f"{n} (algebra {alg}) {tag}")
    if {4, 5, 6} & set(algs):
        for kw in ({}, {"mask": v["mask"], "thresh": thresh}):
            for o, r, n in zip(td.gridnet_grid(p, outlets=outlets, **kw, **sz), port.gridnet(p, outlets=outlets, **kw, **sz), ("plen", "tlen", "gord")):
                assert_bits(o, r, f"{n} {sorted(kw)} {what}")


def _flow(dem, dx, dy):
    fel = port.pitremove(dem)
    return port.d8flowdir(fel, dx=dx, dy=dy)[0], port.dinfflowdir(fel, dx=dx, dy=dy)[0]


def test_sibling_edge_shapes_against_c_restatement():
    """The nine algebras on the degenerate shapes of test_edge_shapes_against_c_restatement (a single row / column, 2 and 3 rows,
    widths that are not multiples of the tile, all nodata, a nodata ring, a constant grid), dx != dy, with and without -nc."""
    rng = np.random.default_rng(14)
    shapes = [(1, 9), (9, 1), (2, 5), (3, 3), (3, 70), (33, 65), (64, 129), (31, 257)]
    grids = [(rng.random(s) * 50).astype(np.float32) for s in shapes]
    ring = (rng.random((40, 37)) * 30).astype(np.float32); ring[0, :] = ring[-1, :] = ring[:, 0] = ring[:, -1] = -9999.0
    grids += [np.full((12, 19), -9999.0, np.float32), ring, np.full((20, 21), 7.0, np.float32)]
    for dem in grids:
        p, ang = _flow(dem, 10.0, 12.0)
        _check_siblings(p, ang, _sibling_values(rng, dem.shape), f"{dem.shape}", dx=10.0, dy=12.0)


def test_siblings_with_many_tile_crossings(crossings):
    """The nine algebras on the 2100 x 3000 DEM of test_sweep_with_many_tile_crossings_matches_the_reference (6 200 tiles, rivers across
    hundreds of them: the warp-cooperative tail of algebras 1-6, algebra 9's second travelling value in global memory), with weights,
    mask + threshold and the supply concentration; the case is checked to reach long rivers and mostly data cells."""
    fel, p, sd8, ang = crossings
    rng = np.random.default_rng(19)
    shape = p.shape
    sa = np.where(sd8 < 0, np.float32(0.0), sd8).astype(np.float32)
    dm = rng.uniform(0.995, 1.0, shape).astype(np.float32); dm[rng.random(shape) < 1e-5] = -9999.0
    w = rng.uniform(0.0, 2.0, shape).astype(np.float32)
    q = rng.uniform(0.5, 3.0, shape).astype(np.float32)
    tc = rng.uniform(0.0, 400.0, shape).astype(np.float32)
    cs = rng.uniform(0.0, 2.0, shape).astype(np.float32)
    dg = (rng.random(shape) < 0.001).astype(np.int16)
    assert_bits(td.d8flowpathextremeup_grid(p, sa), port.d8flowpathextremeup(p, sa), "ssa max")
    assert_bits(td.d8flowpathextremeup_grid(p, fel, usemax=False, contcheck=False), port.d8flowpathextremeup(p, fel, usemax=False, contcheck=False), "ssa min -nc")
    gn = td.gridnet_grid(p)
    for o, r, n in zip(gn, port.gridnet(p), ("plen", "tlen", "gord")):
        assert_bits(o, r, n)
    mask = np.minimum(gn[2].astype(np.int32), 3)              # Strahler order as the mask: the threshold cuts the first-order cells off
    for o, r, n in zip(td.gridnet_grid(p, mask=mask, thresh=2), port.gridnet(p, mask=mask, thresh=2), ("plen", "tlen", "gord")):
        assert_bits(o, r, n + " -mask -thresh 2")
    dsca = td.dinfdecayaccum_grid(ang, dm)
    assert_bits(dsca, port.dinfdecayaccum(ang, dm), "dsca")
    assert_bits(td.dinfdecayaccum_grid(ang, dm, weights=w, contcheck=False), port.dinfdecayaccum(ang, dm, weights=w, contcheck=False), "dsca -wg -nc")
    assert_bits(td.dinfconclimaccum_grid(ang, dm, q, dg, csol=2.0), port.dinfconclimaccum(ang, dm, q, dg, csol=2.0), "ctpt")
    for cs_, cont in ((None, True), (cs, False)):
        ours, ref = td.dinftranslimaccum_grid(ang, q, tc, cs=cs_, contcheck=cont), port.dinftranslimaccum(ang, q, tc, cs=cs_, contcheck=cont)
        for o, r, n in zip(ours, ref, ("tla", "tdep", "ctpt")):
            if r is not None:
                assert_bits(o, r, f"{n} cs={cs_ is not None} contcheck={cont}")
    assert gn[0].max() > 3e4 and gn[1].max() > 1e6 and gn[2].max() >= 5        # rivers of more than 1000 cells, thousands of tiles
    assert dsca.max() > 1e6
    assert (ours[0] != MISSINGFLOAT).mean() > 0.5 and (ours[1] > 0).mean() > 0.02 and (ours[2] > 0).mean() > 0.5


def test_sibling_dinf_angle_torture():
    """Algebras 3, 7, 8 and 9 on angles at and next to every place where prop() changes its mind (util.angle_torture), square and oblong
    cells, with and without -nc."""
    from util import angle_torture
    rng = np.random.default_rng(21)
    for dx, dy in ((30.0, 30.0), (12.5, 40.0)):
        ang = angle_torture(ny=200, nx=330, dx=dx, dy=dy)
        _check_siblings(None, ang, _sibling_values(rng, ang.shape), f"angle torture {dx}x{dy}", dx=dx, dy=dy, algs=(3, 7, 8, 9))


def test_sibling_per_row_cell_sizes(tmp_path):
    """Per-row (geographic) cell sizes: the non-uniform prop() branch of the D-infinity algebras and gridnet's per-row distances.  Grid
    level with dxc / dyc of a geographic file; file level: each sibling executable on geographic files against the restatement with the
    file's cell sizes."""
    import ctypes
    import os
    dem = synth.punch_holes(synth.gen_dem(150, 210, hurst=0.8, tilt=1.0, seed=12))
    geo = str(tmp_path / "geo.tif")
    write_geographic_dem(geo, dem)
    ny = dem.shape[0]
    dxc, dyc = np.zeros(ny), np.zeros(ny)
    assert td.lib().td_raster_cell_sizes(geo.encode(), dxc.ctypes.data_as(ctypes.c_void_p), dyc.ctypes.data_as(ctypes.c_void_p), ny) == 0
    assert np.unique(dxc).size > 100 and np.unique(dyc).size > 1
    fel = port.pitremove(dem)
    p, _ = port.d8flowdir(fel, dx=dxc, dy=dyc)
    ang, _ = port.dinfflowdir(fel, dx=dxc, dy=dyc)
    rng = np.random.default_rng(22)
    v = _sibling_values(rng, dem.shape)
    v["dm"] = rng.uniform(0.2, 1.0, dem.shape).astype(np.float32)
    _check_siblings(p, ang, v, "geographic", dxc=dxc, dyc=dyc, algs=(3, 4, 5, 6, 7, 8, 9))
    # file level
    q = lambda n: str(tmp_path / n)
    for name, a, nd in (("p", p, -32768), ("ang", ang, ANG_ND), ("sa", v["sa"], -9999.0), ("dm", v["dm"], -9999.0), ("w", v["w"], -9999.0),
                        ("q", v["q"], -9999.0), ("dg", v["dg"], -32768), ("tc", v["tc"], -9999.0), ("cs", v["cs"], -9999.0)):
        td.write_raster(q(name + ".tif"), a, nd, like=geo)
    assert td.raster_info(q("ang.tif"))["is_geographic"]
    _run("d8flowpathextremeup", "-p", q("p.tif"), "-sa", q("sa.tif"), "-ssa", q("ssa.tif"), "-min")
    assert_bits(td.read_raster(q("ssa.tif")), port.d8flowpathextremeup(p, v["sa"], usemax=False), "ssa -min (geographic file)")
    _run("gridnet", "-p", q("p.tif"), "-plen", q("plen.tif"), "-tlen", q("tlen.tif"), "-gord", q("gord.tif"))
    for n, r in zip(("plen", "tlen", "gord"), port.gridnet(p, dxc=dxc, dyc=dyc)):
        assert_bits(td.read_raster(q(n + ".tif"), r.dtype), r, n + " (geographic file)")
    _run("dinfdecayaccum", "-ang", q("ang.tif"), "-dm", q("dm.tif"), "-dsca", q("dsca.tif"))
    assert_bits(td.read_raster(q("dsca.tif")), port.dinfdecayaccum(ang, v["dm"], dxc=dxc, dyc=dyc), "dsca (geographic file)")
    _run("dinfdecayaccum", "-ang", q("ang.tif"), "-dm", q("dm.tif"), "-wg", q("w.tif"), "-nc", "-dsca", q("dscaw.tif"))
    assert_bits(td.read_raster(q("dscaw.tif")), port.dinfdecayaccum(ang, v["dm"], weights=v["w"], contcheck=False, dxc=dxc, dyc=dyc), "dsca -wg -nc (geographic file)")
    _run("dinfconclimaccum", "-ang", q("ang.tif"), "-dm", q("dm.tif"), "-q", q("q.tif"), "-dg", q("dg.tif"), "-ctpt", q("ctpt.tif"), "-csol", "1.5")
    assert_bits(td.read_raster(q("ctpt.tif")), port.dinfconclimaccum(ang, v["dm"], v["q"], v["dg"], csol=1.5, dxc=dxc, dyc=dyc), "ctpt (geographic file)")
    _run("dinftranslimaccum", "-ang", q("ang.tif"), "-tsup", q("q.tif"), "-tc", q("tc.tif"), "-cs", q("cs.tif"), "-tla", q("tla.tif"), "-tdep", q("tdep.tif"),
         "-ctpt", q("ctptout.tif"))
    for n, r in zip(("tla", "tdep", "ctptout"), port.dinftranslimaccum(ang, v["q"], v["tc"], cs=v["cs"], dxc=dxc, dyc=dyc)):
        assert_bits(td.read_raster(q(n + ".tif")), r, n + " (geographic file)")


def test_sibling_algebra_edges():
    """The values where each algebra could take a wrong branch: sa ties and negative values (max and min), Strahler ties (three
    tributaries of equal order), mask cells exactly at the threshold and masked-out cells in the middle of rivers, unresolved flats
    (p = 0, angle -1: dependencies only), odd direction codes, dm = 0 / nodata, q <= 0 / nodata, dg on cells that receive flow, tc = 0,
    cs nodata, and outlets: nested and disjoint basins, one off the grid, one on a nodata cell, none at all."""
    rng = np.random.default_rng(31)
    dem = synth.punch_holes(synth.gen_dem(130, 170, hurst=0.8, tilt=1.0, seed=33))
    fel = port.pitremove(dem)
    p, _ = port.d8flowdir(fel, dx=20.0, dy=25.0)
    ang, _ = port.dinfflowdir(fel, dx=20.0, dy=25.0)
    v = _sibling_values(rng, p.shape)
    v["sa"] = rng.integers(-3, 3, p.shape).astype(np.float32)                 # ties everywhere, negative values
    for k in ("dm", "q", "tc"):
        v[k][rng.random(p.shape) < 0.05] = 0.0
    v["q"][rng.random(p.shape) < 0.03] = -2.0
    ad8 = port.aread8(p, contcheck=False)
    mask = np.where(ad8 >= 0, ad8, 0).astype(np.int32)
    river = (ad8 > 30) & (rng.random(p.shape) < 0.2)
    mask[river] = 0                                                            # masked-out cells in the middle of rivers
    v["mask"] = mask
    assert (mask == 12).any()
    _check_siblings(p, ang, v, "edge values", dx=20.0, dy=25.0, thresh=12)
    # unresolved flats: direction 0 / angle -1
    pf, _ = port.d8flowdir(fel, dx=20.0, dy=25.0, flats=False)
    af, _ = port.dinfflowdir(fel, dx=20.0, dy=25.0, flats=False)
    assert (pf == 0).sum() > 100 and (af == -1).sum() > 100
    _check_siblings(pf, af, v, "flats", dx=20.0, dy=25.0, thresh=12)
    # odd direction codes and another nodata value (algebras 1 and 2 follow the reference's aread8 quirks; gridnet the same graph)
    po = rng.integers(-3, 13, size=p.shape).astype(np.int16)
    po[rng.random(p.shape) < 0.05] = -1
    for cont in (True, False):
        for usemax in (True, False):
            assert_bits(td.d8flowpathextremeup_grid(po, v["sa"], usemax=usemax, nodata=-1, contcheck=cont),
                        port.d8flowpathextremeup(po, v["sa"], usemax=usemax, nodata=-1, contcheck=cont), f"ssa odd codes {usemax} {cont}")
    for o, r, n in zip(td.gridnet_grid(po, nodata=-1, dx=20.0, dy=25.0), port.gridnet(po, nodata=-1, dx=20.0, dy=25.0), ("plen", "tlen", "gord")):
        assert_bits(o, r, n + " odd codes")
    # Strahler ties: three order-2 tributaries meet at (4, 4) (order 3), which drains south out of the grid
    s = np.full((9, 9), -32768, np.int16)
    for (r, c), d in {(2, 3): 8, (2, 5): 6, (3, 4): 7, (3, 2): 8, (5, 2): 2, (4, 3): 1, (3, 6): 6, (5, 6): 4, (4, 5): 5, (4, 4): 7, (5, 4): 7, (6, 4): 7,
                      (7, 4): 7}.items():
        s[r, c] = d
    gord = td.gridnet_grid(s)[2]
    assert gord[4, 4] == 3 and gord[3, 4] == gord[4, 3] == gord[4, 5] == 2
    for o, r, n in zip(td.gridnet_grid(s), port.gridnet(s), ("plen", "tlen", "gord")):
        assert_bits(o, r, n + " Strahler ties")
    # outlets: nested (the 2nd lies upstream of the 1st), disjoint, off the grid, on a nodata cell; and none
    ny, nx = p.shape
    order = np.argsort(ad8.ravel())
    top = int(order[-1])
    up = next(int(c) for c in order[::-1][1:] if ad8.flat[c] < ad8.flat[top] and ad8.flat[c] > 20 and abs(c % nx - top % nx) + abs(c // nx - top // nx) < 40)
    nodata_cell = int(np.flatnonzero(p.ravel() == -32768)[len(np.flatnonzero(p.ravel() == -32768)) // 2])
    cells = [top, up, int(order[-300]), int(order[len(order) // 2]), nodata_cell]
    outs = ([c % nx for c in cells] + [-4, nx + 3], [c // nx for c in cells] + [7, 2])
    _check_siblings(p, ang, v, "outlets", dx=20.0, dy=25.0, outlets=outs, thresh=12)
    _check_siblings(p, ang, v, "no outlets", dx=20.0, dy=25.0, outlets=([], []), contchecks=(True,), thresh=12)


# ---------------------------------------------------------------- flat resolution (taudem_b200/csrc/flats.cu) at deep, crowded and multi-pass flats
def _bfs_grid_threads():
    """threads of one pass of k_bfs_level's fixed grid: SMs x 4 blocks x 256"""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 4 * 256


@pytest.mark.parametrize("name", list(flat_cases.CASES))
def test_flat_cases_against_the_reference(refrun, tmp_path, name):
    """Each flat case (tests/flat_cases.py) through d8flowdir_grid / dinfflowdir_grid against the reference (its stored outputs,
    recomputed by the restatement), square cells and dx != dy: p, sd8, slp and ang bit for bit.  port.flat_stats()
    of every reference call shows that the case reaches what it claims; for the pockets, a BFS level larger than one pass of the
    fixed BFS grid on this device."""
    dem, fel = flat_cases.CASES[name]()
    for dx, dy, tool, arg in flat_cases.calls(name):
        R = refrun.RefPipeline(workdir=str(tmp_path), dx=dx, dy=dy, np_ranks=1)
        if tool == "pitremove":
            assert_bits(td.pitremove_grid(dem), R.pitremove(dem), "fel")
            continue
        ref = getattr(R, tool)(fel)
        stats = port.flat_stats()
        assert not flat_cases.reach(name, stats), stats
        if name == "pockets":
            assert stats["rise_level"] > _bfs_grid_threads(), stats
        what = f"{name} {dx}x{dy}"
        if tool == "d8flowdir":
            p, sd8 = td.d8flowdir_grid(fel, dx=dx, dy=dy)
            assert_bits(sd8, ref[1], f"sd8 {what}"); assert_bits(p, ref[0], f"p {what}")
        else:
            ang, slp = td.dinfflowdir_grid(fel, dx=dx, dy=dy)
            assert_bits(slp, ref[1], f"slp {what}"); assert_bits(ang, ref[0], f"ang {what}")


@pytest.mark.parametrize("name", ["deep_lake", "pockets"])
def test_flat_resolution_level_batches(name, monkeypatch):
    """TAUDEM_B200_FLATS_BATCH = 0 (one launch and read-back per BFS level), 1, 3, 64 (the default) and 4096 levels per host read-back
    on the deep lake (508 fall levels: 8 batches of 64) and the pockets (a level larger than one pass of the fixed grid): every
    result bit-identical to the restatement.  The variable is read on every call."""
    _, fel = flat_cases.CASES[name]()
    dx, dy = flat_cases.SIZES[1]
    p_o, sd8_o = port.d8flowdir(fel, dx=dx, dy=dy)
    ang_o, slp_o = port.dinfflowdir(fel, dx=dx, dy=dy)
    for batch in (0, 1, 3, 64, 4096):
        monkeypatch.setenv("TAUDEM_B200_FLATS_BATCH", str(batch))
        p, sd8 = td.d8flowdir_grid(fel, dx=dx, dy=dy)
        assert_bits(p, p_o, f"p, batch {batch}"); assert_bits(sd8, sd8_o, f"sd8, batch {batch}")
        ang, slp = td.dinfflowdir_grid(fel, dx=dx, dy=dy)
        assert_bits(ang, ang_o, f"ang, batch {batch}"); assert_bits(slp, slp_o, f"slp, batch {batch}")


@pytest.mark.parametrize("name", ["deep_lake", "pockets"])
def test_flat_resolution_on_row_strips(name, tmp_path):
    """TAUDEM_B200_GPUS=2 and 3 pitremove -> d8flowdir / dinfflowdir on files (k_merge: BFS levels that cross the strip boundaries,
    which run through the lake and through rows of pockets): every file bit-identical to the one-GPU run, and p / ang to the
    restatement."""
    import os
    import subprocess
    dem, _ = flat_cases.CASES[name]()
    dx, dy = flat_cases.SIZES[1]
    d = tmp_path
    td.write_raster(str(d / "dem.tif"), dem, -9999.0, dx=dx, dy=dy)

    def run(gpus, tool, *args):
        env = dict(os.environ, TAUDEM_B200_GPUS=str(gpus))
        r = subprocess.run([_bin(tool)] + [str(a) for a in args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=600)
        assert r.returncode == 0 and "error" not in r.stdout.lower(), r.stdout

    for n in (1, 2, 3):
        run(n, "pitremove", "-z", d / "dem.tif", "-fel", d / f"fel_{n}.tif")
        run(n, "d8flowdir", "-fel", d / f"fel_{n}.tif", "-p", d / f"p_{n}.tif", "-sd8", d / f"sd8_{n}.tif")
        run(n, "dinfflowdir", "-fel", d / f"fel_{n}.tif", "-ang", d / f"ang_{n}.tif", "-slp", d / f"slp_{n}.tif")
    for nm, dt in (("fel", np.float32), ("p", np.int16), ("sd8", np.float32), ("ang", np.float32), ("slp", np.float32)):
        one = td.read_raster(str(d / f"{nm}_1.tif"), dt)
        for n in (2, 3):
            assert_bits(td.read_raster(str(d / f"{nm}_{n}.tif"), dt), one, f"{nm} on {n} ranks")
    fel = td.read_raster(str(d / "fel_1.tif"))
    assert_bits(fel, port.pitremove(dem), "fel")
    p_o, sd8_o = port.d8flowdir(fel, dx=dx, dy=dy)
    assert_bits(td.read_raster(str(d / "p_1.tif"), np.int16), p_o, "p"); assert_bits(td.read_raster(str(d / "sd8_1.tif")), sd8_o, "sd8")
    ang_o, slp_o = port.dinfflowdir(fel, dx=dx, dy=dy)
    assert_bits(td.read_raster(str(d / "ang_1.tif")), ang_o, "ang"); assert_bits(td.read_raster(str(d / "slp_1.tif")), slp_o, "slp")


def test_flat_needing_32767_passes_is_an_error(tmp_path):
    """A corridor of 32 768 cells needs 32 768 fall passes; the reference's 16-bit pass counter wraps at 32767, so there is no
    result to reproduce: d8flowdir_grid / dinfflowdir_grid fail with TD_ERR_FLAT_PASSES and the executable prints its error line.
    A corridor of 32 766 cells (32 766 fall passes, the most there can be) still resolves."""
    import subprocess
    _, fel = flat_cases.corridor(32768)
    for f in (td.d8flowdir_grid, td.dinfflowdir_grid):
        with pytest.raises(td.TaudemError) as e:
            f(fel)
        assert e.value.code == 92 and "32768 fall passes" in str(e.value), str(e.value)
    td.write_raster(str(tmp_path / "c.tif"), fel, -9999.0)
    r = subprocess.run([_bin("d8flowdir"), "-fel", tmp_path / "c.tif", "-p", tmp_path / "p.tif", "-sd8", tmp_path / "sd8.tif"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert "D8FlowDir device error" in r.stdout and "16-bit pass counter" in r.stdout, r.stdout
    _, ok = flat_cases.corridor(32766)
    p, _ = td.d8flowdir_grid(ok)
    assert (p[2, 1:-1] == 1).all()
