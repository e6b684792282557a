"""peukerdouglas and lengtharea without a GPU: the numpy restatements (tests/stream_restate.py; lengtharea with libm's powf) replay
every reference output the GPU tests compare against (tests/golden/stream_reference.json) and, where oracle/_ref holds the two
reference tools (oracle/stream.mk), match the live reference executables; the command lines' usage and error paths; and the three kernels (k_pd_smooth, k_pd_mark,
k_lengtharea) on the CPU emulation of the thread model (tests/emu), bit for bit against the restatements, on edge shapes, tile
crossings, nodata at the edges and in quad origins, plateaus, a zero side weight, and 2 and 3 row strips with the smoothed rows
exchanged between the passes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import stream_cases as S
import stream_reference as SR
import stream_restate as restate
import test_emu
from util import assert_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")


# ---------------------------------------------------------------- the restatements on the stored reference outputs
def _all_calls(tmp_path):
    """every recorded call; returns the number of calls"""
    n = 0
    for name, dem, w, ranks in S.pd_calls():
        R = SR.RefPipeline(workdir=str(tmp_path), np_ranks=ranks)
        ss = R.peukerdouglas(dem) if w is None else R.peukerdouglas(dem, weights=w)
        assert set(np.unique(np.asarray(ss))) <= {0, 1}, name
        n += 1
    plen, ad8, ad8w = S.la_inputs()
    R = SR.RefPipeline(workdir=str(tmp_path))
    for a in (ad8, ad8w):
        for m, y in S.LA_PAR:
            R.lengtharea(plen, a) if m is None else R.lengtharea(plen, a, m=m, y=y)
            n += 1
    dem = S.workflow_dem()
    S.pd_workflow(SR.RefPipeline(workdir=str(tmp_path)), dem)
    S.la_workflow(SR.RefPipeline(workdir=str(tmp_path)), dem)
    return n + 5 + 5 - 2            # the two chains share pitremove and d8flowdir


def test_restatements_replay_every_stored_stream_definition_output(tmp_path):
    """Every reference output of the stream-definition tests, recomputed by the restatements and matched to its stored digest.
    The count is asserted: a call that is not replayed fails here."""
    import port
    import reference
    if not port.available():
        pytest.skip("oracle/port not built")              # (the workflows' other tools are replayed by oracle/port)
    before = set(reference.replayed)
    n = _all_calls(tmp_path)
    if not reference.RECORD:
        new = set(reference.replayed) - before
        tools = sorted(reference.replayed[k] for k in new)
        assert tools.count("peukerdouglas") == len(S.pd_calls()) + 1 == 13, tools
        assert tools.count("lengtharea") == 2 * len(S.LA_PAR) + 1 == 7, tools
        assert len(new) <= n


def test_restatements_match_the_live_reference(tmp_path, monkeypatch):
    """With oracle/_ref built: peukerdouglas at 1 and 3 ranks and lengtharea at 1 rank, the executables themselves."""
    import refrun
    if not SR.available():
        pytest.skip("the reference's peukerdouglas / lengtharea are not built (make -C oracle -f stream.mk)")
    monkeypatch.setattr(refrun, "INPUTS_ONLY", False)
    for name, dem, w, ranks in S.pd_calls():
        R = SR.Files(workdir=str(tmp_path), np_ranks=ranks)
        got = R.peukerdouglas(dem) if w is None else R.peukerdouglas(dem, weights=w)
        want = restate.peukerdouglas(dem) if w is None else restate.peukerdouglas(dem, weights=w)
        assert_bits(got, want, f"peukerdouglas {name} {w} {ranks} ranks")
    plen, ad8, ad8w = S.la_inputs()
    R = SR.Files(workdir=str(tmp_path))
    for a in (ad8, ad8w):
        for m, y in S.LA_PAR:
            got = R.lengtharea(plen, a) if m is None else R.lengtharea(plen, a, m=m, y=y)
            assert_bits(got, restate.lengtharea(plen, a, m, y), f"lengtharea {m} {y}")


# ---------------------------------------------------------------- command lines
def _run(tool, *args, cwd=None):
    exe = os.path.join(BIN, tool)
    if not os.access(exe, os.X_OK):
        pytest.skip("executables not built")
    r = subprocess.run([exe, *args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120, cwd=cwd)
    return r.returncode, r.stdout


def test_cli_usage_and_errors(tmp_path):
    """Usage on missing or bad arguments (exit 0, like the reference mains); -par needs all its values; a missing input file and
    lengtharea's grids that do not match end in the reference's error lines before any device is needed."""
    import taudem_b200 as td
    for tool, flag in (("peukerdouglas", "-fel"), ("lengtharea", "-plen")):
        rc, out = _run(tool)
        assert rc == 0 and "Simple Use:" in out and flag in out, out
        rc, out = _run(tool, "-bogus", "x")
        assert rc == 0 and "Simple Use:" in out, out
    rc, out = _run("peukerdouglas", "-fel", "a.tif", "-ss", "b.tif", "-par", "0.4", "0.1")
    assert rc == 0 and "Simple Use:" in out and "PeukerDouglas version" not in out, out
    rc, out = _run("lengtharea", "-plen", "a.tif", "-ad8", "b.tif", "-ss", "c.tif", "-par", "0.03")
    assert rc == 0 and "Simple Use:" in out, out
    rc, out = _run("peukerdouglas", "-fel", str(tmp_path / "missing.tif"), "-ss", str(tmp_path / "ss.tif"), "-par", "0.4", "0.1", "0.05")
    assert rc == 0 and "PeukerDouglas version" in out and "Peuker Douglas Error 21" in out, out
    rc, out = _run("peukerdouglas", str(tmp_path / "missing.tif"))                    # simple use: missingfel.tif
    assert rc == 0 and "missingfel.tif" in out and "Peuker Douglas Error 21" in out, out
    td.write_raster(str(tmp_path / "plen.tif"), np.zeros((5, 7), np.float32), -1.0)
    td.write_raster(str(tmp_path / "ad8.tif"), np.ones((5, 8), np.float32), -1.0)
    rc, out = _run("lengtharea", "-plen", str(tmp_path / "plen.tif"), "-ad8", str(tmp_path / "ad8.tif"), "-ss", str(tmp_path / "ss.tif"))
    assert rc == 0 and "LengthArea version" in out and "Length Area Error 1" in out, out
    assert not (tmp_path / "ss.tif").exists()


def test_lengtharea_grid_refuses_a_non_int32_area():
    import taudem_b200 as td
    with pytest.raises(TypeError):
        td.lengtharea_grid(np.zeros((3, 3), np.float32), np.zeros((3, 3), np.float32))
    with pytest.raises(ValueError):
        td.peukerdouglas_grid(np.zeros((3, 3), np.float32), weights=(0.4, 0.1))


# ---------------------------------------------------------------- the kernels on the CPU emulation
def build_pd_emu():
    """tests/emu/pd_driver.cpp with peuker.cu and pointwise.cu on the CPU emulation (also the point-wise kernels' tests)"""
    os.makedirs(test_emu.BUILD, exist_ok=True)
    incs = [test_emu._transform("peuker", 2), test_emu._transform("pointwise", 7)]
    so = os.path.join(test_emu.BUILD, "libemu_pd.so")
    srcs = [os.path.join(test_emu.EMU, f) for f in ("pd_driver.cpp", "emu.cpp")]
    deps = srcs + incs + [os.path.join(test_emu.EMU, "cuda_runtime.h"), os.path.join(test_emu.CSRC, "tile_pipe.cuh"), os.path.join(test_emu.CSRC, "common.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ftls-model=initial-exec", "-ffp-contract=off",
                               "-I", test_emu.EMU, "-I", test_emu.BUILD, "-I", test_emu.CSRC, "-o", so, *srcs])
    lib = C.CDLL(so)
    P = C.c_void_p
    lib.emu_peukerdouglas.argtypes = [P, P, C.c_int, C.c_int, C.c_float, P, C.c_int, P]
    lib.emu_lengtharea.argtypes = [P, P, P, C.c_int, C.c_int, C.c_float, C.c_float, P]
    lib.emu_threshold.argtypes = [P, P, P, C.c_int, C.c_int, C.c_float, C.c_float]
    lib.emu_slp_sca.argtypes = [C.c_int, P, P, P, C.c_int, C.c_int, C.c_float, C.c_float]
    return lib


@pytest.fixture(scope="module")
def emu():
    return build_pd_emu()


def _emu_pd(lib, fel, weights=(0.4, 0.1, 0.05), strips=None):
    fel = np.ascontiguousarray(fel, np.float32)
    ny, nx = fel.shape
    rows = np.ascontiguousarray([ny] if strips is None else strips, np.int32)
    assert rows.sum() == ny
    w = np.ascontiguousarray(weights, np.float32)
    ss = np.empty((ny, nx), np.int16)
    assert lib.emu_peukerdouglas(fel.ctypes.data, ss.ctypes.data, nx, ny, float(S.ND), w.ctypes.data, len(rows), rows.ctypes.data) == 0
    return ss


def _edge_dems():
    """small and thin shapes: nx or ny in {1, 2, 3}, odd widths, one tile and a few tiles (32 x 128 cells)"""
    rng = np.random.default_rng(5)
    out = []
    for ny, nx in ((1, 1), (1, 6), (2, 2), (2, 9), (3, 3), (3, 40), (7, 1), (9, 2), (11, 3), (33, 129), (40, 3), (70, 261)):
        d = np.round(rng.normal(size=(ny, nx)).astype(np.float32) * 2.0) / 2.0          # half units: plateaus and ties
        d = d.astype(np.float32)
        if ny > 4 and nx > 4:
            m = rng.random((ny, nx)) < 0.06
            d[m] = S.ND
            d[0, 1] = d[-1, -2] = d[2, 0] = d[3, -1] = S.ND                              # nodata on every edge
        out.append(d)
    return out


@pytest.mark.parametrize("weights", [(0.4, 0.1, 0.05), (0.5, 0.0, 0.2), (1.0, 0.3, 0.0)])
def test_emulated_pd_kernels_match_the_restatement(emu, weights):
    dems = _edge_dems() + [S.rough(), S.holes()]
    for d in dems:
        assert_bits(_emu_pd(emu, d, weights), restate.peukerdouglas(d, weights=weights), f"{d.shape} {weights}")


def test_emulated_pd_quad_origins_on_nodata(emu):
    """A quad's origin is not tested for nodata: a nodata origin with a large positive nodata value is the quad's maximum and its
    other cells stay flagged; with the usual very negative nodata value they compete among themselves."""
    d = S.rough()[:20, :30].copy()
    d[5, 5] = d[9, 12] = d[14, 20] = S.ND
    assert_bits(_emu_pd(emu, d), restate.peukerdouglas(d), "nodata origins")
    big = np.float32(1.0e30)
    e = S.rough()[:20, :30].copy()
    e[5, 5] = e[9, 12] = big
    ss = np.empty(e.shape, np.int16)
    w = np.asarray((0.4, 0.1, 0.05), np.float32)
    assert emu.emu_peukerdouglas(e.ctypes.data, ss.ctypes.data, 30, 20, float(big), w.ctypes.data, 1, np.asarray([20], np.int32).ctypes.data) == 0
    assert_bits(ss, restate.peukerdouglas(e, nodata=float(big)), "positive nodata origins")


@pytest.mark.parametrize("strips", [(26, 27), (17, 18, 18), (1, 2, 50), (25, 1, 27)])
def test_emulated_pd_row_strips(emu, strips):
    """2 and 3 strips (and strips of one and two rows): the first pass on raw halo rows, the smoothed edge rows exchanged, the
    second pass; identical to one strip and to the restatement."""
    d = S.holes()
    for w in ((0.4, 0.1, 0.05), (0.5, 0.0, 0.2)):
        want = restate.peukerdouglas(d, weights=w)
        assert_bits(_emu_pd(emu, d, w, strips), want, f"{strips} {w}")


def test_emulated_lengtharea_matches_the_restatement(emu):
    plen, ad8, ad8w = S.la_inputs()
    rng = np.random.default_rng(9)
    odd = rng.random((3, 37)).astype(np.float32) * 500 - 50                          # negative plen: nodata; an odd width
    for pl, a in ((plen, ad8), (plen, ad8w), (odd, np.abs(odd) * 3)):
        ai = restate.ad8_int32(a)
        for m, y in S.LA_PAR + ((0.5, 0.5), (1.0, 2.0)):
            mm, yy = (0.03, 1.3) if m is None else (m, y)
            ss = np.empty(pl.shape, np.int16)
            p = np.ascontiguousarray(pl, np.float32)
            assert emu.emu_lengtharea(p.ctypes.data, ai.ctypes.data, ss.ctypes.data, pl.shape[1], pl.shape[0], mm, yy, None) == 0
            assert_bits(ss, restate.lengtharea(pl, a, m, y), f"{pl.shape} {m} {y}")
