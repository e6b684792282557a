"""dinfdistdown on the GPU against the reference's outputs (tests/golden/dinfdistdown_reference.json, replayed by the C restatement:
tests/dinfdistdown_reference.py) and the restatement itself, bit for bit: the grid level on every recorded call (the 12 method /
statistic pairs with and without weights and -nc on rough DEMs, junk angles, nodata in every input, sector boundaries and the wrap
sector, cycles, NaN and -FLT_MAX fel, src beyond int16, oblong cells, a path of more than 10 batches of levels, a serpentine, the HAND
chain and a 2000 x 1500 grid), geographic per-row cell sizes, the file level and both usages of the executable, TAUDEM_B200_GPUS = 1,
2 and 3, and the pitremove -> dinfflowdir -> d8flowdir -> aread8 -> threshold -> dinfdistdown -m ave v workflow with our
executables."""
import os
import subprocess

import numpy as np
import pytest

import dinfdistdown_cases as DC
import dinfdistdown_port
import dinfdistdown_reference as DR
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


def _grid(ang, fel, src, w, method, stat, cc, dx=30.0, dy=30.0, dxc=None, dyc=None):
    import taudem_b200 as td
    return td.dinfdistdown_grid(ang, src, fel=fel, weights=w, method=method, stat=stat, contcheck=cc, dx=dx, dy=dy, dxc=dxc, dyc=dyc,
                                fel_nodata=float(DC.FEL_ND), w_nodata=float(DC.W_ND))


def _restated(ang, fel, src, w, method, stat, cc, dx=30.0, dy=30.0, dxc=None, dyc=None):
    return dinfdistdown_port.dinfdistdown(ang, src, fel, w, method, stat, cc, dx=dx, dy=dy, dxc=dxc, dyc=dyc, fel_nodata=DC.FEL_ND,
                                          w_nodata=DC.W_ND)


def test_grid_level_matches_the_reference():
    """every recorded call (393, the 2000 x 1500 grid's included) against the reference's digest and the restatement"""
    import taudem_b200 as td
    n = 0
    for key, args in DR.runs():
        got = _grid(*args)
        assert_bits(got, DR.want(key), key)
        assert_bits(got, _restated(*args), key + " (restatement)")
        if key.startswith("long path -m ave h 30x30"):
            assert td.lib().td_dinfdistdown_last_levels() > 10 * 64
        n += 1
    assert n == DR.EXPECTED


def test_grid_level_geographic_rows(tmp_path):
    """per-row cell sizes of a geographic raster: every row's shares and distances from its own sizes"""
    import taudem_b200 as td
    ang, fel, src = DR.rough(61, 47, 3, 10.0)
    f = str(tmp_path / "geo.tif")
    write_geographic_dem(f, fel)
    ny = fel.shape[0]
    xc, yc = np.empty(ny), np.empty(ny)
    assert td.lib().td_raster_cell_sizes(f.encode(), xc.ctypes.data, yc.ctypes.data, ny) == 0
    w = np.random.default_rng(4).random(ang.shape).astype(np.float32)
    for m in DC.METHODS:
        want = _restated(ang, fel, src, w, m, "ave", True, dxc=xc, dyc=yc)
        assert (want != DC.MISSINGFLOAT).sum() > 500
        assert_bits(_grid(ang, fel, src, w, m, "ave", True, dxc=xc, dyc=yc), want, f"geographic {m}")


def _files(tmp_path, ang, fel, src, w, dx=30.0, dy=30.0):
    import taudem_b200 as td
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("baseang.tif"), ang, float(DC.ANG_ND), dx=dx, dy=dy)
    td.write_raster(d("basefel.tif"), fel, float(DC.FEL_ND), dx=dx, dy=dy)
    td.write_raster(d("basesrc.tif"), np.asarray(src, np.int32), int(DC.SRC_ND), dx=dx, dy=dy)
    td.write_raster(d("basewg.tif"), w, float(DC.W_ND), dx=dx, dy=dy)
    return d


def test_file_level_and_executable(tmp_path):
    """td_dinfdistdown through the binding and the executable with flags (every method, -wg, -nc, -m in either order) and in simple
    usage (ave h, no weights): float32, nodata MISSINGFLOAT, ang's georeference"""
    import taudem_b200 as td
    ang, fel, src, w = DC.random_case(0)
    d = _files(tmp_path, ang, fel, src, w, 10.0, 7.0)
    outs = []
    for i, (m, st, cc) in enumerate((("h", "ave", True), ("v", "min", False), ("p", "max", True), ("s", "ave", False))):
        args = ["-ang", d("baseang.tif"), "-fel", d("basefel.tif"), "-slp", d("noslp.tif"), "-src", d("basesrc.tif"), "-wg", d("basewg.tif"),
                "-dd", d(f"x{i}.tif"), "-m", *((st, m) if i % 2 else (m, st))]
        if not cc:
            args.append("-nc")
        out = _exe("dinfdistdown", *args)
        assert f"DinfDistDown -{m} version" in out and "Compute time" in out, out
        outs.append((f"x{i}.tif", _restated(ang, fel, src, w if m != "v" else None, m, st, cc, 10.0, 7.0)))
    assert td.lib().td_dinfdistdown(d("baseang.tif").encode(), d("basefel.tif").encode(), b"", d("basewg.tif").encode(), d("basesrc.tif").encode(),
                                    d("y.tif").encode(), 1, 3, 1, 1) == 0
    outs.append(("y.tif", _restated(ang, fel, src, w, "s", "max", True, 10.0, 7.0)))
    _exe("dinfdistdown", d("base.tif"))                              # simple usage: ave h, basewg.tif named but not used
    outs.append(("basedd.tif", _restated(ang, fel, src, None, "h", "ave", True, 10.0, 7.0)))
    for f, want in outs:
        assert_bits(td.read_raster(d(f), np.float32), want, f)
        info = td.raster_info(d(f))
        assert np.float32(info["nodata"]) == DC.MISSINGFLOAT and info["bits"] == 32 and (info["dx"], info["dy"]) == (10.0, 7.0), info
    td.write_raster(d("small.tif"), np.asarray(src, np.int32)[:, :-1].copy(), int(DC.SRC_ND))
    r = subprocess.run([os.path.join(BIN, "dinfdistdown"), "-ang", d("baseang.tif"), "-src", d("small.tif"), "-dd", d("z.tif")], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=120)
    assert r.returncode == 5 and "File sizes do not match" in r.stdout, r.stdout
    assert not os.path.exists(d("z.tif"))


@pytest.mark.parametrize("which", ["rough", "serpentine"])
def test_on_1_2_and_3_gpus(tmp_path, which):
    """TAUDEM_B200_GPUS=N: levels per strip, the halo-row donors' decrements and the value rows (two in the p mode) exchanged, the
    received decrements starting the next levels; identical for every N and to the restatement's one-rank result"""
    import taudem_b200 as td
    if which == "rough":
        ang, fel, src = DR.rough(157, 211, 5, 8.0)
        w = np.random.default_rng(6).random(ang.shape).astype(np.float32) + 0.5
    else:
        ang, fel, src, w = DC.serpentine(45, 20)
        w = np.ones_like(ang)
    d = _files(tmp_path, ang, fel, src, w)
    for m, st, cc in (("h", "ave", True), ("v", "ave", True), ("p", "max", False), ("s", "min", False)):
        cc = cc and which == "rough"               # (the serpentine's last column leans off the grid: -nc keeps its cells)
        want = _restated(ang, fel, src, None if m == "v" else w, m, st, cc)
        assert (want != DC.MISSINGFLOAT).sum() > want.size // 2
        for n in (1, 2, 3):
            args = ["-ang", d("baseang.tif"), "-fel", d("basefel.tif"), "-src", d("basesrc.tif"), "-wg", d("basewg.tif"), "-dd", d(f"{m}{n}.tif"), "-m", m, st]
            out = _exe("dinfdistdown", *args, *([] if cc else ["-nc"]), gpus=n)
            if n > 1:
                assert f"Processors: {n}" in out, out
                rounds = int(out.split("Exchange rounds:")[1].split()[0])
                if which == "serpentine":
                    assert rounds > 10, out                 # a round per crossing of the path
            assert_bits(td.read_raster(d(f"{m}{n}.tif"), np.float32), want, f"{which} -m {st} {m} at {n} GPUs")


def test_hand_workflow_with_the_executables(tmp_path):
    """pitremove -> dinfflowdir -> d8flowdir -> aread8 -> threshold -> dinfdistdown -m ave v (the height above the nearest drainage)
    with our executables, equal to the reference's output on the same chain"""
    import taudem_b200 as td
    dem = DR.hand_dem()
    d = lambda n: str(tmp_path / n)     # noqa: E731
    td.write_raster(d("dem.tif"), dem, -9999.0)
    _exe("pitremove", "-z", d("dem.tif"), "-fel", d("fel.tif"))
    _exe("dinfflowdir", "-fel", d("fel.tif"), "-ang", d("ang.tif"), "-slp", d("slp.tif"))
    _exe("d8flowdir", "-fel", d("fel.tif"), "-p", d("p.tif"), "-sd8", d("sd8.tif"))
    _exe("aread8", "-p", d("p.tif"), "-ad8", d("ad8.tif"))
    _exe("threshold", "-ssa", d("ad8.tif"), "-src", d("src.tif"), "-thresh", "20")
    _exe("dinfdistdown", "-ang", d("ang.tif"), "-fel", d("fel.tif"), "-slp", d("slp.tif"), "-src", d("src.tif"), "-dd", d("hand.tif"), "-m", "ave", "v")
    ang, fel, src = DR.hand_chain(dem)
    assert_bits(td.read_raster(d("ang.tif"), np.float32), ang, "dinfflowdir")
    assert_bits(td.read_raster(d("src.tif"), np.int16), src, "threshold")
    hand = td.read_raster(d("hand.tif"), np.float32)
    assert_bits(hand, DR.want("hand -m ave v 30x30"), "HAND")
    assert (hand != DC.MISSINGFLOAT).sum() > hand.size // 4
