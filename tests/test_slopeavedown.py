"""slopeavedown without a GPU: the C restatement (oracle/port/slopeavedown_oracle.c) replays every reference output the GPU tests
compare against (tests/golden/slopeavedown_reference.json) and, where oracle/_ref holds the reference's slopeavedown, matches the
live executable on random grids at 1 and 3 ranks; the Jacobi kernels (k_sad_init, k_sad_pass) on the CPU emulation of the thread
model (tests/emu/sad_driver.cpp), bit for bit against the restatement on 1, 2 and 3 row strips with the state's edge rows exchanged
after every pass; the command line's usage and error paths; and the argument checks."""
import ctypes as C
import os
import subprocess
from collections import deque

import numpy as np
import pytest

import downslope_port
import slopeavedown_reference as SR
import test_emu
from util import assert_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")
D1 = (0, 1, 1, 0, -1, -1, -1, 0, 1)
D2 = (0, 0, -1, -1, -1, 0, 1, 1, 1)

pytestmark = pytest.mark.skipif(not downslope_port.available(), reason="make -C oracle -f downslope.mk port")


# ---------------------------------------------------------------- the restatement on the stored reference outputs
def test_restatement_replays_every_stored_output(tmp_path):
    """Every reference output of the slopeavedown tests, recomputed by the restatement and matched to its stored digest.  The count
    is asserted: a call that is not replayed fails here."""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    before = set(SR.replayed)
    n = 0
    for case in SR.cases():
        SR.reference_case(SR.pipeline(tmp_path, case), case)
        n += 1
    SR.workflow(SR.RefPipeline(workdir=str(tmp_path)), SR.workflow_dem())
    fel, p, dn = SR.large()
    SR.RefPipeline(workdir=str(tmp_path)).slopeavedown(fel, p, dn=dn)
    if not SR.reference.RECORD:
        tools = sorted(SR.replayed[k] for k in set(SR.replayed) - before)
        assert tools.count("slopeavedown") == n + 2 == 21, tools
        assert tools.count("pitremove") == tools.count("d8flowdir") == 1, tools


def test_restatement_matches_the_live_reference(tmp_path, monkeypatch):
    """With oracle/_ref built: random small grids (random codes in -2..10, cycles, code 0s, nodata in fel and p, DEM nodata -9999 and
    -FLT_MAX, five cell-size / dn settings), the reference executable at 1 and 3 ranks against the restatement."""
    import refrun
    if not SR.available():
        pytest.skip("the reference's slopeavedown is not built (make -C oracle -f downslope.mk ref)")
    monkeypatch.setattr(refrun, "INPUTS_ONLY", False)
    for seed in range(6):
        rng = np.random.default_rng(seed)
        fel, p = SR.flow(23, 31, 100 + seed)
        znd = np.float32(-9999.0) if seed % 2 else SR.MISSINGFLOAT
        if seed % 3 == 0:
            m = rng.random(p.shape) < 0.3
            p[m] = rng.integers(-2, 11, m.sum())
            p[rng.random(p.shape) < 0.05] = SR.P_ND
        if seed % 3 != 2:
            fel[rng.random(p.shape) < 0.06] = znd
        for dx, dy, dn in ((30.0, 30.0, 50.0), (10.0, 7.0, 45.0), (1.0, 1.0, 6.0), (30.0, 30.0, 2000.0), (30.0, 30.0, 0.0)):
            want = downslope_port.slopeavedown(fel, p, dn=dn, dx=dx, dy=dy, nodata=znd)
            for ranks in (1, 3):
                got = SR.Files(workdir=str(tmp_path), dx=dx, dy=dy, np_ranks=ranks).slopeavedown(fel, p, dn=dn, fel_nodata=float(znd))
                assert_bits(got, want, f"seed {seed} dx {dx} dy {dy} dn {dn} at {ranks} ranks")


def test_restatement_niter():
    assert downslope_port.niter(50.0, 30.0, 30.0) == 2
    assert downslope_port.niter(50.0, 10.0, 7.0) == 8
    assert downslope_port.niter(-10.0, 30.0, 30.0) == 0
    assert downslope_port.niter(-100.0, 30.0, 30.0) == -2
    assert downslope_port.niter(float("nan"), 30.0, 30.0) is None
    assert downslope_port.niter(float("inf"), 30.0, 30.0) is None
    assert downslope_port.niter(1e300, 30.0, 30.0) is None
    assert downslope_port.niter(50.0, 0.0, 30.0) is None


# ---------------------------------------------------------------- the kernels on the CPU emulation
def processed(p, pnd):
    """the cells the aread8 queue of initNeighborD8up reaches (src/commonLib.cpp:250-281, src/SlopeAveDown.cpp:251-260)"""
    ny, nx = p.shape
    node = (p != pnd) & (p >= 0) & (p <= 8)
    cnt = np.zeros(p.shape, np.int64)
    q = deque()
    for j in range(ny):
        for i in range(nx):
            if not node[j, i]:
                continue
            for k in range(1, 9):
                a, b = i + D1[k], j + D2[k]
                if 0 <= a < nx and 0 <= b < ny and node[b, a] and p[b, a] - k in (4, -4):
                    cnt[j, i] += 1
            if cnt[j, i] == 0:
                q.append((i, j))
    done = np.zeros(p.shape, np.uint8)
    while q:
        i, j = q.popleft()
        done[j, i] = 1
        k = int(p[j, i])
        a, b = i + D1[k], j + D2[k]
        if 1 <= k <= 8 and 0 <= a < nx and 0 <= b < ny and node[b, a]:
            cnt[b, a] -= 1
            if cnt[b, a] == 0:
                q.append((a, b))
    return done


@pytest.fixture(scope="module")
def emu():
    os.makedirs(test_emu.BUILD, exist_ok=True)
    inc = test_emu._transform("slopeavedown", 2)
    so = os.path.join(test_emu.BUILD, "libemu_sad.so")
    srcs = [os.path.join(test_emu.EMU, f) for f in ("sad_driver.cpp", "emu.cpp")]
    deps = srcs + [inc, os.path.join(test_emu.EMU, "cuda_runtime.h"), os.path.join(test_emu.CSRC, "common.cuh"), os.path.join(test_emu.CSRC, "kernels.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ftls-model=initial-exec", "-ffp-contract=off",
                               "-I", test_emu.EMU, "-I", test_emu.BUILD, "-I", test_emu.CSRC, "-o", so, *srcs])
    lib = C.CDLL(so)
    P = C.c_void_p
    lib.emu_slopeavedown.argtypes = [P, P, P, P, C.c_int, C.c_int, C.c_float, C.c_int16, P, P, C.c_double, C.c_int, C.c_int, P, P]
    return lib


def _emu(lib, case, strips=None, dxc=None, dyc=None):
    name, fel, fnd, p, pnd, dx, dy, dn, _ = case
    fel = np.ascontiguousarray(fel, np.float32); p = np.ascontiguousarray(p, np.int16)
    ny, nx = fel.shape
    xc = np.ascontiguousarray(np.full(ny, dx) if dxc is None else dxc, np.float64)
    yc = np.ascontiguousarray(np.full(ny, dy) if dyc is None else dyc, np.float64)
    rows = np.ascontiguousarray([ny] if strips is None else strips, np.int32)
    assert rows.sum() == ny
    mask = processed(p, pnd)
    sd = np.empty((ny, nx), np.float32)
    passes = C.c_int(0)
    niter = downslope_port.niter(dn, dx, dy)
    assert lib.emu_slopeavedown(fel.ctypes.data, p.ctypes.data, mask.ctypes.data, sd.ctypes.data, nx, ny, float(fnd), int(pnd), xc.ctypes.data,
                                yc.ctypes.data, float(dn), niter, len(rows), rows.ctypes.data, C.byref(passes)) == 0
    return sd, passes.value


def _want(case, dxc=None, dyc=None):
    name, fel, fnd, p, pnd, dx, dy, dn, _ = case
    return downslope_port.slopeavedown(fel, p, dn=dn, dx=dx, dy=dy, nodata=fnd, p_nodata=pnd, dxc=dxc, dyc=dyc, passes=True)


def test_emulated_kernels_match_the_restatement(emu):
    """every recorded case on one strip; the early stop fires where a pass changes nothing, and the result is the full run's"""
    stopped = 0
    for case in SR.cases():
        if case[8] != 1:
            continue
        want, last = _want(case)
        got, passes = _emu(emu, case)
        assert_bits(got, want, case[0])
        niter = downslope_port.niter(case[7], case[5], case[6])
        assert passes == min(niter, last + 1) if niter > 0 else passes == 0, (case[0], passes, last, niter)
        stopped += passes < niter
    assert stopped >= 1


@pytest.mark.parametrize("strips", [(35, 35), (23, 24, 23), (1, 2, 67), (34, 1, 35)])
def test_emulated_row_strips(emu, strips):
    """2 and 3 strips (and strips of one and two rows), the state's edge rows exchanged after every pass: identical to the
    restatement"""
    for case in SR.cases():
        if case[0].startswith("strips") and case[8] == 1:
            assert_bits(_emu(emu, case, strips)[0], _want(case)[0], f"{case[0]} {strips}")


def test_emulated_geographic_rows(emu, tmp_path):
    """per-row cell sizes of a geographic raster for the distances (the header's sizes for niter)"""
    import taudem_b200 as td
    from util import write_geographic_dem
    name, fel, fnd, p, pnd, dx, dy, dn, r = [c for c in SR.cases() if c[0] == "strips junk"][0]
    f = str(tmp_path / "geo.tif")
    write_geographic_dem(f, fel)
    ny = fel.shape[0]
    xc, yc = np.empty(ny), np.empty(ny)
    assert td.lib().td_raster_cell_sizes(f.encode(), xc.ctypes.data, yc.ctypes.data, ny) == 0
    case = (name, fel, fnd, p, pnd, abs(xc[ny // 2]), abs(yc[ny // 2]), 700.0, 1)
    want, _ = _want(case, xc, yc)
    assert (want != SR.MISSINGFLOAT).sum() > 100
    for strips in (None, (30, 40)):
        assert_bits(_emu(emu, case, strips, xc, yc)[0], want, f"geographic {strips}")


# ---------------------------------------------------------------- command line and arguments
def _run(*args):
    exe = os.path.join(BIN, "slopeavedown")
    if not os.access(exe, os.X_OK):
        pytest.skip("executables not built")
    r = subprocess.run([exe, *args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    return r.returncode, r.stdout


def test_cli_usage_and_errors(tmp_path):
    """Usage on missing or bad arguments (exit 0, like the reference's main); a missing input ends in "sloped error 21"; fel and p
    of different sizes end in "File sizes do not match" and "sloped error 5", before any device is needed."""
    import taudem_b200 as td
    rc, out = _run()
    assert rc == 0 and out.startswith("Error: To run this program") and "-slpd <slpdfile> -dn <dn>" in out, out
    for args in (("-bogus", "x"), ("-fel", "a.tif", "-p"), ("-fel", "a.tif", "-p", "b.tif", "-slpd", "c.tif", "-dn")):
        rc, out = _run(*args)
        assert rc == 0 and out.startswith("Simple Usage:") and "SlopeAveDown version" not in out, out
    rc, out = _run(str(tmp_path / "missing.tif"))                     # simple use: missingfel.tif
    assert rc == 0 and "missingfel.tif" in out and "sloped error 21" in out, out
    td.write_raster(str(tmp_path / "fel.tif"), np.zeros((5, 7), np.float32), -1.0)
    td.write_raster(str(tmp_path / "p.tif"), np.ones((5, 8), np.int16), -32768)
    rc, out = _run("-fel", str(tmp_path / "fel.tif"), "-p", str(tmp_path / "p.tif"), "-slpd", str(tmp_path / "s.tif"))
    assert rc == 0 and "File sizes do not match" in out and "sloped error 5" in out, out
    assert not (tmp_path / "s.tif").exists()


def test_niter_and_shape_checks():
    import taudem_b200 as td
    n = C.c_int(0)
    assert td.lib().td_slopeavedown_niter(50.0, 10.0, 7.0, C.byref(n)) == 0 and n.value == 8
    for dn, dx in ((float("nan"), 30.0), (float("inf"), 30.0), (1e300, 30.0), (50.0, 0.0)):
        assert td.lib().td_slopeavedown_niter(dn, dx, 30.0, C.byref(n)) == 1, (dn, dx)
    with pytest.raises(ValueError):
        td.slopeavedown_grid(np.zeros((3, 3), np.float32), np.zeros((3, 4), np.int16))
