"""dinfdistdown without a GPU: the C restatement (oracle/port/dinfdistdown_oracle.c) replays every reference output the GPU tests
compare against (tests/golden/dinfdistdown_reference.json) and, where oracle/_ref holds the reference's executable, matches it on
random grids (junk angles, cycles, nodata in every input, NaN fel) through the 12 method / statistic pairs with and without -nc; the
level kernels (k_ddd_seed, k_ddd_level, k_ddd_pyth) on the CPU emulation of the thread model (tests/emu/ddd_driver.cpp), bit for bit
against the restatement under several schedule seeds and on geographic rows; and the command line's usage, -m parsing and error
paths."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import dinfdistdown_cases as DC
import dinfdistdown_port
import dinfdistdown_reference as DR
import test_emu
from util import assert_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")

pytestmark = pytest.mark.skipif(not dinfdistdown_port.available(), reason="make -C oracle -f dinfdistdown.mk port")


def _restated(ang, fel, src, w, method, stat, cc=True, dx=30.0, dy=30.0, dxc=None, dyc=None):
    return dinfdistdown_port.dinfdistdown(ang, src, fel, w, method, stat, cc, dx=dx, dy=dy, dxc=dxc, dyc=dyc, fel_nodata=DC.FEL_ND,
                                          w_nodata=DC.W_ND)


def test_restatement_replays_every_stored_output():
    """every stored digest is reproduced by the restatement, and every one is replayed"""
    n = 0
    for key, args in DR.runs():
        assert_bits(_restated(*args[:-2], dx=args[-2], dy=args[-1]), DR.want(key), key)
        n += 1
    assert n == len(DR.stored()) == DR.EXPECTED


def test_cases_reach_the_edge_shapes():
    """the random cases hold what each branch of the algebra needs: nodata results from contamination, NaN values from NaN fel,
    MISSINGFLOAT on cycles, negative results from negative weights, and h max clamped at 0"""
    ang, fel, src, w = DC.random_case(0)
    v = _restated(ang, fel, src, None, "v", "ave", cc=False)
    data = np.isfinite(v) & (v != DC.MISSINGFLOAT)
    assert np.isnan(v).sum() > 5 and (v == DC.MISSINGFLOAT).sum() > 20 and data.sum() > 100
    assert (_restated(ang, fel, src, None, "v", "ave") != DC.MISSINGFLOAT).sum() < (v != DC.MISSINGFLOAT).sum()
    h = _restated(ang, fel, src, w, "h", "min", cc=False)
    assert (h[h != DC.MISSINGFLOAT] < 0).sum() > 0
    hm = _restated(ang, fel, src, w, "h", "max", cc=False)
    assert (hm == 0).sum() > ((src >= 1) & (ang != DC.ANG_ND)).sum()
    c = _restated(*DC.cycles(), "h", "ave")
    assert (c == DC.MISSINGFLOAT).sum() > 10 and (c > 0).sum() > 5


def test_restatement_matches_the_live_reference(monkeypatch):
    """With oracle/_ref built: random small grids through every method and statistic, with and without weights and -nc, square and
    oblong cells, at 1 and 3 ranks."""
    import refrun
    if not DC.available():
        pytest.skip("the reference's dinfdistdown is not built (make -C oracle -f dinfdistdown.mk ref)")
    monkeypatch.setattr(refrun, "INPUTS_ONLY", False)
    for seed in range(3):
        ang, fel, src, w = DC.random_case(seed)
        for dx, dy in ((30.0, 30.0), (10.0, 7.0)):
            for m in DC.METHODS:
                for st in DC.STATS:
                    for cc, ww in ((True, None), (False, w if m != "v" else None), (True, w if m != "v" else None)):
                        want = _restated(ang, fel, src, ww, m, st, cc, dx=dx, dy=dy)
                        for ranks in (1, 3):
                            F = DC.Files(dx=dx, dy=dy, np_ranks=ranks)
                            assert_bits(F.dinfdistdown(ang, fel, src, ww, m, st, cc), want, f"seed {seed} {dx} -m {st} {m} nc {not cc} at {ranks} ranks")


# ---------------------------------------------------------------- the kernels on the CPU emulation
@pytest.fixture(scope="module")
def emu():
    os.makedirs(test_emu.BUILD, exist_ok=True)
    inc = test_emu._transform("dinfdistdown", 3)
    so = os.path.join(test_emu.BUILD, "libemu_ddd.so")
    srcs = [os.path.join(test_emu.EMU, f) for f in ("ddd_driver.cpp", "emu.cpp")]
    deps = srcs + [inc] + [os.path.join(test_emu.CSRC, f) for f in ("common.cuh", "dinf_common.cuh", "flood.cuh", "kernels.h")] + \
        [os.path.join(test_emu.EMU, "cuda_runtime.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ffp-contract=off",
                               "-I", test_emu.EMU, "-I", test_emu.BUILD, "-I", test_emu.CSRC, "-o", so, *srcs])
    lib = C.CDLL(so)
    P = C.c_void_p
    lib.emu_dinfdistdown.argtypes = [P, P, P, P, P, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, P, P, C.c_int, C.c_int, C.c_int,
                                     C.c_int, P, C.c_uint, C.c_int, P, P]
    return lib


def _emu(lib, ang, fel, src, w, method, stat, cc=True, dx=30.0, dy=30.0, dxc=None, dyc=None, seed=1, grid=3, strips=None):
    """(dd, levels, rounds) of the kernels on the CPU emulation, on one strip or on row strips of the given heights"""
    ang = np.ascontiguousarray(ang, np.float32)
    ny, nx = ang.shape
    s = np.asarray(src)
    src = np.ascontiguousarray(np.clip(s, -32768, 32767), np.int16)
    fel = None if method == "h" else np.ascontiguousarray(fel, np.float32)
    w = None if method == "v" or w is None else np.ascontiguousarray(w, np.float32)
    xc = np.ascontiguousarray(np.full(ny, dx) if dxc is None else dxc, np.float64)
    yc = np.ascontiguousarray(np.full(ny, dy) if dyc is None else dyc, np.float64)
    rows = np.ascontiguousarray([ny] if strips is None else strips, np.int32)
    assert rows.sum() == ny
    out = np.empty((ny, nx), np.float32)
    levels, rounds = C.c_longlong(0), C.c_int(0)
    ptr = lambda a: None if a is None else a.ctypes.data
    assert lib.emu_dinfdistdown(ang.ctypes.data, ptr(fel), ptr(w), src.ctypes.data, out.ctypes.data, nx, ny, float(DC.ANG_ND), float(DC.FEL_ND),
                                float(DC.W_ND), xc.ctypes.data, yc.ctypes.data, DC.STATS.index(stat), DC.METHODS.index(method), int(cc), len(rows),
                                rows.ctypes.data, seed, grid, C.byref(levels), C.byref(rounds)) == 0
    return out, levels.value, rounds.value


def test_emulated_kernels_match_the_restatement(emu):
    """random grids, cycles and the serpentine through every method and statistic, under two schedule seeds and two grid sizes"""
    cases = [DC.random_case(s, ny=13, nx=17) for s in range(2)] + [DC.cycles(), DC.serpentine(12, 6)]
    for i, (ang, fel, src, w) in enumerate(cases):
        for m in DC.METHODS:
            for st in DC.STATS:
                for cc in (True, False):
                    want = _restated(ang, fel, src, w, m, st, cc)
                    for seed, grid in ((1, 3), (7, 1)):
                        assert_bits(_emu(emu, ang, fel, src, w, m, st, cc, seed=seed, grid=grid)[0], want, f"case {i} -m {st} {m} nc {not cc} seed {seed}")


def test_emulated_long_path(emu):
    """a path of 720 cells: more than 10 batches of levels, one cell per level"""
    ang, fel, src, w = DC.long_path()
    got, levels, _ = _emu(emu, ang, fel, src, w, "v", "ave")
    assert_bits(got, _restated(ang, fel, src, w, "v", "ave"), "long path")
    assert levels > 10 * 64 and (got != DC.MISSINGFLOAT).all()


@pytest.mark.parametrize("strips", [[1, 1, 11], [3, 2, 1, 7], [4, 5, 4]])
def test_emulated_row_strips(emu, strips):
    """row strips of 1 to 7 rows: the decrements of the halo-row donors and the value rows exchanged between rounds (both value rows
    in the p mode)"""
    ang, fel, src, w = DC.random_case(2, ny=13, nx=17)
    for m in DC.METHODS:
        for st, cc in (("ave", True), ("max", False), ("min", False)):
            got, _, rounds = _emu(emu, ang, fel, src, w, m, st, cc, strips=strips, seed=len(strips))
            assert_bits(got, _restated(ang, fel, src, w, m, st, cc), f"{strips} -m {st} {m} nc {not cc}")


def test_emulated_serpentine_crosses_strips_many_times(emu):
    """a path that crosses every strip boundary once per column: a round per crossing"""
    ang, fel, src, w = DC.serpentine(12, 8)
    for m in ("h", "p"):
        got, _, rounds = _emu(emu, ang, fel, src, w, m, "ave", False, strips=[4, 4, 4])
        assert_bits(got, _restated(ang, fel, src, w, m, "ave", False), f"serpentine {m}")
        assert rounds > 8 and (got != DC.MISSINGFLOAT).sum() > got.size * 3 // 4


def test_emulated_geographic_rows(emu):
    """per-row cell sizes: the shares and distances of every row from its own sizes, the halo rows' from theirs"""
    ang, fel, src, w = DC.random_case(5, ny=15, nx=11)
    xc = 30.0 * np.cos(np.deg2rad(np.linspace(40, 60, 15)))
    yc = np.full(15, 30.0)
    for m in ("h", "s", "p"):
        want = _restated(ang, fel, src, w, m, "ave", cc=False, dxc=xc, dyc=yc)
        for strips in (None, [5, 6, 4]):
            assert_bits(_emu(emu, ang, fel, src, w, m, "ave", cc=False, dxc=xc, dyc=yc, strips=strips)[0], want, f"geographic {m} {strips}")


def test_grid_level_argument_checks():
    import taudem_b200 as td
    z = np.zeros((3, 3), np.float32)
    with pytest.raises(ValueError):
        td.dinfdistdown_grid(z, np.zeros((3, 4), np.int16))
    with pytest.raises(ValueError):
        td.dinfdistdown_grid(z, np.zeros((3, 3), np.int16), method="v")      # v needs fel
    with pytest.raises(ValueError):
        td.dinfdistdown_grid(z, np.zeros((3, 3), np.int16), stat="median")


# ---------------------------------------------------------------- command line and arguments
def _run(*args):
    exe = os.path.join(BIN, "dinfdistdown")
    if not os.access(exe, os.X_OK):
        pytest.skip("executables not built")
    r = subprocess.run([exe, *map(str, args)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=120)
    return r.returncode, r.stdout


USAGE = "-fel <felfile> -slp <slpfile> -src <srcfile> [-wg <wfile>] -dd <dtsfile>\n[-m ave h] [-nc]\n"


def test_cli_usage_and_errors(tmp_path):
    """Usage on missing or bad arguments (exit 0, the reference's text), `-m` with one token left; a missing input ends in the
    reference's error line; rasters of different sizes end in "File sizes do not match" and exit status 5, as the reference's
    MPI_Abort(MCW, 5), before any device is needed, in the order the reference opens its files."""
    import taudem_b200 as td
    rc, out = _run()
    assert rc == 0 and out.startswith("Error: To run this program") and USAGE in out, out
    for args in [("-bogus", "x"), ("-ang", "a.tif", "-src"), ("-ang", "a.tif", "-m"), ("-ang", "a.tif", "-m", "ave"), ("-ang", "a.tif", "-thresh", "3")]:
        rc, out = _run(*args)
        assert rc == 0 and out.startswith("Simple Usage:") and USAGE in out and "version" not in out, (args, out)
    rc, out = _run(tmp_path / "missing.tif")                  # simple use: missingang.tif
    assert rc == 0 and "Error opening file" in out and "missingang.tif" in out and "area error 21" in out, out
    t = lambda n: str(tmp_path / n)
    td.write_raster(t("ang.tif"), np.zeros((5, 7), np.float32), -1.0)
    for name, shape, dtype in (("fel", (5, 7), np.float32), ("fel8", (5, 8), np.float32), ("w8", (5, 8), np.float32), ("w", (5, 7), np.float32),
                               ("src8", (5, 8), np.int32), ("src", (5, 7), np.int16)):
        td.write_raster(t(name + ".tif"), np.ones(shape, dtype), -1)
    runs = [  # (method, fel, w, src, the file that does not match)
        ("h", "fel8", None, "src8", "src8"),          # h never opens fel
        ("h", "fel", "w8", "src8", "w8"),             # h: ang, wg, src
        ("v", "fel8", "w8", "src", "fel8"),           # v: ang, fel, src (no weights)
        ("v", "fel", "w8", "src8", "src8"),
        ("p", "fel", "w8", "src8", "w8"),             # p and s: ang, fel, wg, src
        ("s", "fel8", "w", "src", "fel8"),
    ]
    for m, fel, w, src, bad in runs:
        args = ["-ang", t("ang.tif"), "-fel", t(fel + ".tif"), "-slp", t("none.tif"), "-src", t(src + ".tif"), "-dd", t("dd.tif"), "-m", m, "min"]
        if w:
            args += ["-wg", t(w + ".tif")]
        rc, out = _run(*args)
        assert rc == 5 and f"DinfDistDown -{m} version" in out and f"File sizes do not match\n{t(bad + '.tif')}\n" in out, (m, out)
        assert "area error" not in out and not (tmp_path / "dd.tif").exists()
    # -m in either order, unknown tokens leave the defaults
    for mm, banner in ((("min", "s"), "-s"), (("p", "max"), "-p"), (("x", "y"), "-h"), (("v", "median"), "-v")):
        rc, out = _run("-ang", t("ang.tif"), "-fel", t("fel8.tif"), "-src", t("src.tif"), "-dd", t("dd.tif"), "-m", *mm)
        assert out.startswith(f"DinfDistDown {banner} version"), (mm, out)
