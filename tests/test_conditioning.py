"""flowdircond and retlimflow without a GPU: the C restatement (oracle/port/conditioning_oracle.c) replays every reference output the GPU tests
compare against (tests/golden/conditioning_reference.json) and, where oracle/_ref holds the reference's flowdircond, matches the live
executables on random grids at 1 and 3 ranks; algebras 11 and 12 of the contributing-area sweep on the CPU emulation of the thread
model (tests/emu/cond_driver.cpp), bit for bit against the restatements on 1, 2 and 3 row strips and several schedule seeds; the
sweep table's entries for algebras 11 and 12; the command lines' usage and error paths."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import conditioning_port
import conditioning_reference as CR
import test_emu
from test_slopeavedown import processed
from util import assert_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")

pytestmark = pytest.mark.skipif(not conditioning_port.available(), reason="make -C oracle -f conditioning.mk port")


# ---------------------------------------------------------------- the restatement on the stored reference outputs
def test_restatement_replays_every_stored_output(tmp_path):
    """Every reference output of the flowdircond tests, recomputed by the restatement and matched to its stored digest.  The count
    is asserted: a call that is not replayed fails here."""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    before = set(CR.replayed)
    n = 0
    for case in CR.cases():
        CR.reference_case(CR.pipeline(tmp_path, case), case)
        n += 1
    CR.workflow(CR.RefPipeline(workdir=str(tmp_path)), CR.workflow_dem())
    z, p = CR.large()
    CR.RefPipeline(workdir=str(tmp_path)).flowdircond(p, z)
    if not CR.reference.RECORD:
        tools = sorted(CR.replayed[k] for k in set(CR.replayed) - before)
        assert tools.count("flowdircond") == n + 2 == 18, tools
        assert tools.count("pitremove") == tools.count("d8flowdir") == 1, tools


def test_retlimflow_restatement_replays_every_stored_output(tmp_path):
    """Every reference output of the retlimflow tests, recomputed by the restatement and matched to its stored digest"""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    before = set(CR.replayed)
    n = 0
    for case in CR.rl_cases():
        CR.rl_reference_case(CR.rl_pipeline(tmp_path, case), case)
        n += 1
    dem = CR.workflow_dem()
    wg, rc = CR.rl_inputs(dem, 74)
    CR.rl_workflow(CR.RefPipeline(workdir=str(tmp_path)), dem, wg, rc)
    ang, wg, rc = CR.rl_large()
    CR.RefPipeline(workdir=str(tmp_path)).retlimflow(ang, wg, rc)
    if not CR.reference.RECORD:
        tools = sorted(CR.replayed[k] for k in set(CR.replayed) - before)
        assert tools.count("retlimflow") == n + 2 == 13, tools
        assert tools.count("dinfflowdir") == 1, tools


def test_restatement_matches_the_live_reference(tmp_path, monkeypatch):
    """With oracle/_ref built: random small grids (random codes in -2..10 with cycles and code 0s, p of another DEM, nodata in z and
    p, z nodata -9999 and -FLT_MAX, +-0 and NaN), the reference executable at 1 and 3 ranks against the restatement."""
    import refrun
    if not CR.available():
        pytest.skip("the reference's flowdircond is not built (make -C oracle -f conditioning.mk ref)")
    monkeypatch.setattr(refrun, "INPUTS_ONLY", False)
    for seed in range(8):
        rng = np.random.default_rng(seed)
        z, p = CR.burned(23, 31, 200 + seed)
        znd = np.float32(-9999.0) if seed % 2 else CR.MISSINGFLOAT
        if seed % 3 == 0:
            p = CR.other_p(23, 31, seed)
            m = rng.random(p.shape) < 0.3
            p[m] = rng.integers(-2, 11, m.sum())
        elif seed % 3 == 1:
            p = CR.random_p(23, 31, seed)
        p[rng.random(p.shape) < 0.05] = CR.P_ND
        z[rng.random(z.shape) < 0.06] = znd
        if seed >= 4:
            z = CR.signed_zeros_nan(z, seed)
        want = conditioning_port.flowdircond(p, z, nodata=znd)
        for ranks in (1, 3):
            got = CR.Files(workdir=str(tmp_path), np_ranks=ranks).flowdircond(p, z, z_nodata=float(znd))
            assert_bits(got, want, f"seed {seed} at {ranks} ranks")


def test_restatement_processes_the_aread8_cells():
    """the cells the restatement's queue dequeues are the cells aread8's queue reaches (tests/test_slopeavedown.processed): the same
    cells the D8 sweep evaluates"""
    for case in CR.cases():
        name, p, pnd, z, znd, ranks = case
        _, n = conditioning_port.flowdircond(p, z, p_nodata=pnd, nodata=znd, processed=True)
        assert n == int(processed(p, pnd).sum()), name


def test_cases_condition_something():
    """most cases lower cells (the directions disagree with z), and the NaN / signed-zero case keeps NaN where z was NaN"""
    lowered = 0
    for name, p, pnd, z, znd, ranks in CR.cases():
        got = conditioning_port.flowdircond(p, z, p_nodata=pnd, nodata=znd)
        ok = ~np.isnan(z)
        assert (got[ok] <= z[ok]).all(), name
        lowered += int((got[ok] < z[ok]).sum() > 0)
        assert np.isnan(got[~ok]).all(), name
    assert lowered >= len(CR.cases()) - 1


# ---------------------------------------------------------------- algebra 11 on the CPU emulation
@pytest.fixture(scope="module")
def emu():
    test_emu._build()                                  # the transformed kernel sources
    so = os.path.join(test_emu.BUILD, "libemu_cond.so")
    srcs = [os.path.join(test_emu.EMU, f) for f in ("cond_driver.cpp", "emu.cpp")]
    deps = srcs + [os.path.join(test_emu.EMU, "sibling_strips_driver.cpp"), os.path.join(test_emu.EMU, "driver.cpp"),
                   os.path.join(test_emu.BUILD, "sweep_warp_emu.inc"), os.path.join(test_emu.BUILD, "outlets_emu.inc"),
                   os.path.join(test_emu.EMU, "cuda_runtime.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ftls-model=initial-exec", "-ffp-contract=off",
                               "-I", test_emu.EMU, "-I", test_emu.BUILD, "-I", test_emu.CSRC, "-o", so, *srcs])
    lib = C.CDLL(so)
    P = C.c_void_p
    lib.emu_flowdircond_strips.argtypes = [P, P, C.c_int, C.c_int, C.c_int, P, C.c_float, C.c_ulonglong, P, P]
    lib.emu_retlimflow_strips.argtypes = [P, P, P, C.c_int, C.c_int, C.c_int, P, C.c_float, C.c_float, P, P, C.c_ulonglong, P, P]
    return lib


def _emu(lib, p, z, znd, strips=None, seed=1):
    p = np.ascontiguousarray(p, np.int16); z = np.ascontiguousarray(z, np.float32)
    ny, nx = z.shape
    rows = np.ascontiguousarray([ny] if strips is None else strips, np.int32)
    assert rows.sum() == ny
    out = np.empty((ny, nx), np.float32)
    st = np.zeros(3, np.int64)
    rc = lib.emu_flowdircond_strips(p.ctypes.data, z.ctypes.data, nx, ny, len(rows), rows.ctypes.data, np.float32(znd), seed, out.ctypes.data,
                                    st.ctypes.data)
    assert rc == 0, rc
    return out, int(st[0]), int(st[1]), int(st[2])


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_emulated_sweep_matches_the_restatement(emu, seed):
    """every case on one strip, three schedule seeds: bit for bit, and the sweep evaluates exactly the cells the queue dequeues"""
    for name, p, pnd, z, znd, ranks in CR.cases():
        if ranks != 1:
            continue
        want, n = conditioning_port.flowdircond(p, z, p_nodata=pnd, nodata=znd, processed=True)
        got, _, _, evaluated = _emu(emu, p, z, znd, seed=seed)
        assert_bits(got, want, name)
        assert evaluated == n, name


@pytest.mark.parametrize("strips", [(35, 35), (23, 24, 23), (1, 2, 67), (34, 1, 35)])
def test_emulated_row_strips(emu, strips):
    """2 and 3 strips (and strips of one and two rows), the conditioned elevation's edge rows exchanged every round: identical to the
    restatement, and flow really crosses the strip boundaries"""
    for seed, (name, p, pnd, z, znd, ranks) in enumerate(c for c in CR.cases() if c[0].startswith("strips") and c[5] == 1):
        got, rounds, handed, _ = _emu(emu, p, z, znd, strips, seed=seed + 5)
        assert_bits(got, conditioning_port.flowdircond(p, z, p_nodata=pnd, nodata=znd), f"{name} {strips}")
        assert rounds > 1 and handed > 0, (name, strips, rounds, handed)


def test_retlimflow_restatement_matches_the_live_reference(tmp_path, monkeypatch):
    """With oracle/_ref built: random small grids (angles of a DEM or the angle torture, wg / rc holes, NaN wg, rc above the inflow,
    oblong cells), the reference executable at 1 rank against the restatement with the reference's edge handling, and at 3 ranks
    where that handling changes nothing (on 3 ranks the reference reads an uninitialised top border, src/linearpart.h:263-278)"""
    import refrun
    from util import angle_torture
    if not os.access(os.path.join(refrun.REF, "retlimflow"), os.X_OK):
        pytest.skip("the reference's retlimflow is not built (make -C oracle -f conditioning.mk ref)")
    monkeypatch.setattr(refrun, "INPUTS_ONLY", False)
    for seed in range(6):
        rng = np.random.default_rng(seed)
        dx, dy = (10.0, 7.0) if seed % 3 == 2 else (30.0, 30.0)
        ang = angle_torture(23, 31, dx, dy, seed) if seed % 2 else CR.dinf_angles(23, 31, 300 + seed, dx, dy)
        wg, rc = CR.rl_inputs(ang, seed, 1.0, 0.3 + seed)
        wg[rng.random(ang.shape) < 0.05] = CR.Z_ND
        rc[rng.random(ang.shape) < 0.05] = CR.Z_ND
        wg[rng.random(ang.shape) < 0.02] = np.nan
        want = conditioning_port.retlimflow(ang, wg, rc, dx=dx, dy=dy, edge_quirk=True)
        plain = conditioning_port.retlimflow(ang, wg, rc, dx=dx, dy=dy)
        for ranks in (1, 3):
            if ranks == 3 and not np.array_equal(want.view(np.uint32), plain.view(np.uint32)):
                continue
            got = CR.Files(workdir=str(tmp_path), dx=dx, dy=dy, np_ranks=ranks).retlimflow(ang, wg, rc)
            assert_bits(got, want, f"seed {seed} at {ranks} ranks")


def _emu_rl(lib, ang, wg, rc, wnd, rcnd, dxr, dyr, strips=None, seed=1):
    ang, wg, rc = (np.ascontiguousarray(a, np.float32) for a in (ang, wg, rc))
    ny, nx = ang.shape
    rows = np.ascontiguousarray([ny] if strips is None else strips, np.int32)
    dxr, dyr = (np.ascontiguousarray(np.broadcast_to(np.asarray(v, np.float64), (ny,))) for v in (dxr, dyr))
    out = np.empty((ny, nx), np.float32)
    st = np.zeros(3, np.int64)
    rc_ = lib.emu_retlimflow_strips(ang.ctypes.data, wg.ctypes.data, rc.ctypes.data, nx, ny, len(rows), rows.ctypes.data, np.float32(wnd),
                                    np.float32(rcnd), dxr.ctypes.data, dyr.ctypes.data, seed, out.ctypes.data, st.ctypes.data)
    assert rc_ == 0, rc_
    return out, int(st[0]), int(st[1]), int(st[2])


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_emulated_retlimflow_matches_the_restatement(emu, seed):
    """every retlimflow case on one strip, three schedule seeds: bit for bit; the sweep evaluates exactly the cells the queue dequeues
    (blocked cells included)"""
    for name, ang, andv, wg, wnd, rc, rcnd, dx, dy, ranks in CR.rl_cases():
        if ranks != 1:
            continue
        want, n = conditioning_port.retlimflow(ang, wg, rc, dx=dx, dy=dy, wg_nodata=wnd, rc_nodata=rcnd, processed=True)
        got, _, _, evaluated = _emu_rl(emu, ang, wg, rc, wnd, rcnd, dx, dy, seed=seed)
        assert_bits(got, want, name)
        assert evaluated == n, (name, evaluated, n)


@pytest.mark.parametrize("strips", [(35, 35), (23, 24, 23), (1, 2, 67), (34, 1, 35)])
def test_emulated_retlimflow_row_strips(emu, strips):
    """2 and 3 strips (and strips of one and two rows): identical to the restatement, with flow and blocked closures crossing the
    strip boundaries"""
    for seed, (name, ang, andv, wg, wnd, rc, rcnd, dx, dy, ranks) in enumerate(c for c in CR.rl_cases() if c[9] == 1 and c[1].shape[0] == 70):
        got, rounds, handed, _ = _emu_rl(emu, ang, wg, rc, wnd, rcnd, dx, dy, strips, seed=seed + 5)
        assert_bits(got, conditioning_port.retlimflow(ang, wg, rc, dx=dx, dy=dy, wg_nodata=wnd, rc_nodata=rcnd), f"{name} {strips}")
        assert rounds > 1 and handed > 0, (name, strips, rounds, handed)


def test_emulated_retlimflow_geographic_rows(emu, tmp_path):
    """per-row cell sizes of a geographic raster: each contributor's share with its own row's sizes, on one and two strips"""
    import taudem_b200 as td
    from util import write_geographic_dem
    name, ang, andv, wg, wnd, rc, rcnd, dx, dy, r = [c for c in CR.rl_cases() if c[0] == "rl strips"][0]
    f = str(tmp_path / "geo.tif")
    write_geographic_dem(f, np.zeros(ang.shape, np.float32))
    ny = ang.shape[0]
    xc, yc = np.empty(ny), np.empty(ny)
    assert td.lib().td_raster_cell_sizes(f.encode(), xc.ctypes.data, yc.ctypes.data, ny) == 0
    want = conditioning_port.retlimflow(ang, wg, rc, dxc=xc, dyc=yc, wg_nodata=wnd, rc_nodata=rcnd)
    assert (want > 0).sum() > 1000
    for strips in (None, (30, 40)):
        assert_bits(_emu_rl(emu, ang, wg, rc, wnd, rcnd, xc, yc, strips)[0], want, f"geographic {strips}")


def test_retlimflow_cases_block_and_clip():
    """the cases exercise what they are meant to: blocked closures (cells the queue reaches that stay nodata), clipped cells (0) and
    NaN"""
    blocked = clipped = nan = 0
    for name, ang, andv, wg, wnd, rc, rcnd, dx, dy, ranks in CR.rl_cases():
        q = conditioning_port.retlimflow(ang, wg, rc, dx=dx, dy=dy, wg_nodata=wnd, rc_nodata=rcnd)
        blocked += int(((q == CR.MISSINGFLOAT) & (np.abs(wg - wnd) >= 1e-5) & (np.abs(rc - rcnd) >= 1e-5) & (ang != CR.MISSINGFLOAT)).sum())
        clipped += int((q == 0).sum())
        nan += int(np.isnan(q).sum())
    assert blocked > 100 and clipped > 100 and nan > 10, (blocked, clipped, nan)


def test_retlimflow_edge_quirk_is_confined():
    """The reference's one-rank handling of shares that leave the grid through the top / bottom edge (DESIGN.md §2) starts at cells of
    the first and last row (and reaches what drains from them); of the recorded cases it changes only the angle torture"""
    for name, ang, andv, wg, wnd, rc, rcnd, dx, dy, ranks in CR.rl_cases():
        a = conditioning_port.retlimflow(ang, wg, rc, dx=dx, dy=dy, wg_nodata=wnd, rc_nodata=rcnd, edge_quirk=True)
        b = conditioning_port.retlimflow(ang, wg, rc, dx=dx, dy=dy, wg_nodata=wnd, rc_nodata=rcnd)
        d = a.view(np.uint32) != b.view(np.uint32)
        assert d.any() == (name == "rl torture"), name
        if d.any():
            assert d[0].any() or d[-1].any(), name


# ---------------------------------------------------------------- the sweep table
@pytest.mark.parametrize("alg,combo,required", [(11, (0, 1), 1), (12, (1, 1), 1 | 2)])
def test_sweep_table_algebras_11_and_12(alg, combo, required):
    """the sweep accepts algebra 11 only as (D8, weights) with `w`, and algebra 12 only as (D-infinity, weights) with `w` and `dm`;
    every other flow model / weights combination, and a call without a required grid, is rejected with TD_ERR_ARG; the other grids
    are not required.  Algebra 13 is not a sweep."""
    lib = test_emu._build()
    lib.emu_wsweep_call.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint]
    for dinf, usew in itertools.product((0, 1), (0, 1)):
        assert lib.emu_wsweep_call(dinf, usew, alg, 0) == (0 if (dinf, usew) == combo else 1), (alg, dinf, usew)
        assert lib.emu_wsweep_call(dinf, usew, 13, 0) == 1, (dinf, usew)
    for bit in (1, 2, 4, 8, 16, 32, 64, 128):
        assert lib.emu_wsweep_call(*combo, alg, bit) == (1 if required & bit else 0), (alg, bit)


# ---------------------------------------------------------------- command line
def _run(*args):
    exe = os.path.join(BIN, "flowdircond")
    if not os.access(exe, os.X_OK):
        pytest.skip("executables not built")
    r = subprocess.run([exe, *args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    return r.returncode, r.stdout


def test_cli_usage_and_errors(tmp_path):
    """Usage on missing or bad arguments (exit 0 and the reference's text, which has no "Simple Usage" line); a missing input ends in
    "flowdiircond error 21" (the reference's spelling); p and z of different sizes end in "File sizes do not match" and
    "flowdiircond error 5", before any device is needed."""
    import taudem_b200 as td
    rc, out = _run()
    assert rc == 0 and out.startswith("Error: To run this program") and "-z <zfile> -zfdc <zfdcfile> \n" in out, out
    for args in (("-bogus", "x"), ("-p", "a.tif", "-z"), ("-p", "a.tif", "-z", "b.tif", "-zfdc")):
        rc, out = _run(*args)
        assert rc == 0 and out.startswith("Use with specific file names:") and "FlowDirCond version" not in out, out
    rc, out = _run(str(tmp_path / "missing.tif"))                     # simple use: missingp.tif first
    assert rc == 0 and "missingp.tif" in out and "flowdiircond error 21" in out, out
    td.write_raster(str(tmp_path / "z.tif"), np.zeros((5, 7), np.float32), -9999.0)
    td.write_raster(str(tmp_path / "p.tif"), np.ones((5, 8), np.int16), -32768)
    rc, out = _run("-p", str(tmp_path / "p.tif"), "-z", str(tmp_path / "z.tif"), "-zfdc", str(tmp_path / "o.tif"))
    assert rc == 0 and "File sizes do not match" in out and "flowdiircond error 5" in out, out
    assert not (tmp_path / "o.tif").exists()


def _run_rl(*args):
    exe = os.path.join(BIN, "retlimflow")
    if not os.access(exe, os.X_OK):
        pytest.skip("executables not built")
    r = subprocess.run([exe, *args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    return r.returncode, r.stdout


def test_retlimflow_cli_usage_and_errors(tmp_path):
    """Usage on missing or bad arguments (exit 0, the reference's text); every failure prints "RetlimFlow error 1" (the reference
    assigns `retlimro(...) != 0` to err); a grid of another size ends in "File sizes do not match" before any device is needed."""
    import taudem_b200 as td
    rc, out = _run_rl()
    assert rc == 0 and out.startswith("Error: To run this program") and "-rc <rcfile> -wg <wgfile> -qrl <qrlfile>" in out, out
    for args in (("-bogus", "x"), ("-ang", "a.tif", "-wg"), ("-ang", "a.tif", "-wg", "b.tif", "-rc", "c.tif", "-qrl")):
        rc, out = _run_rl(*args)
        assert rc == 0 and out.startswith("Simple Usage:") and "version" not in out, out
    rc, out = _run_rl(str(tmp_path / "missing.tif"))                  # simple use: missingang.tif first
    assert rc == 0 and "missingang.tif" in out and "RetlimFlow error 1" in out, out
    td.write_raster(str(tmp_path / "ang.tif"), np.zeros((5, 7), np.float32), -3.4028234663852886e38)
    td.write_raster(str(tmp_path / "wg.tif"), np.zeros((5, 7), np.float32), -9999.0)
    td.write_raster(str(tmp_path / "rc.tif"), np.zeros((6, 7), np.float32), -9999.0)
    rc, out = _run_rl("-ang", str(tmp_path / "ang.tif"), "-wg", str(tmp_path / "wg.tif"), "-rc", str(tmp_path / "rc.tif"), "-qrl", str(tmp_path / "q.tif"))
    assert rc == 0 and "File sizes do not match" in out and "RetlimFlow error 1" in out, out
    assert not (tmp_path / "q.tif").exists()
