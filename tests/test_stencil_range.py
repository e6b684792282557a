"""The flow-direction stencils (k_d8_stencil, k_dinf_stencil) outside natural relief.  Both rank the neighbours with a float
pre-screen and run the reference's arithmetic only on the winner or a short list; the pre-screens are exact only while the
drops, slopes and squared slopes they work with are normal floats.  These tests take one terrain with nodata holes and flats
through every power-of-two scale from 2^-149 (drops of a few subnormal ulps, squared slopes that underflow) to 2^127 and to
neighbour differences that overflow float, and build D-infinity grids whose cells sit on exact facet ties, on the drop rules
and on the 1e-9 clip band of VSLOPE.  The same cases run on the CPU emulation of the kernels (positive-slope pass against
the C restatement, bit for bit) and on the GPU (pitremove -> d8flowdir / dinfflowdir against the restatement's pipeline, every
raster bit for bit, ang included); the restatement itself is pinned on the reference tools at a few of the scales."""
import ctypes as C
import os

import numpy as np
import pytest

from taudem_b200 import synth
from util import assert_bits, write_geographic_dem

NY, NX = 45, 150                    # crosses a 32-row and a 128-column tile edge
FEL_ND = -3.0e38
DEM_ND = np.float32(-9999.0)
SIZES = [(30.0, 30.0), (12.5, 40.0), (0.5, 0.5), (1000.0, 1000.0), (float(np.nextafter(32.0, 0.0)), 30.0)]   # the last: RowFact::safe = 0
SCALES = list(range(-149, -39)) + [-20, 0, 10, 60, 100, 126, 127]


def _terrain():
    """the base terrain on [0, 1] (data cells), with its nodata holes"""
    dem = synth.punch_holes(synth.gen_dem(NY, NX, hurst=0.8, tilt=1.0, seed=3))
    ok = dem != DEM_ND
    lo, hi = float(dem[ok].min()), float(dem[ok].max())
    u = np.where(ok, (dem.astype(np.float64) - lo) / (hi - lo), 0.0)
    return u, ok


def scaled_dem(k, signed):
    """the terrain shifted to [0, 1] or [-1, 1] and multiplied by 2^k in float (subnormal results round), holes kept"""
    u, ok = _terrain()
    v = (2.0 * u - 1.0) if signed else u
    out = np.ldexp(v.astype(np.float32), k).astype(np.float32)
    out[~ok] = DEM_ND
    return out


def overflow_dem():
    """values up to +-2.9e38: neighbour differences overflow float to +-inf; the lowest value stays far from the fel nodata -3e38"""
    u, ok = _terrain()
    out = ((2.0 * u - 1.0) * 2.9e38).astype(np.float32)
    out[1::4, 2::5] = np.abs(out[1::4, 2::5])           # peaks next to cells near -2.9e38
    out[~ok] = DEM_ND
    return out


def ulp_dem(seed=4):
    """a high base (8000 m) plus 0..6 ulps: ties, one-ulp drops and wide flats"""
    u, ok = _terrain()
    rng = np.random.default_rng(seed)
    steps = np.round(u * 4).astype(np.int32) + rng.integers(0, 3, u.shape).astype(np.int32)
    out = (np.float32(8000.0).view(np.int32) + steps).view(np.float32)
    out[~ok] = DEM_ND
    return np.ascontiguousarray(out)


def dem_cases():
    cases = [(f"2^{k}{' signed' if s else ''}", scaled_dem(k, s)) for k in SCALES for s in (False, True)]
    return cases + [("overflow", overflow_dem()), ("8000 m + ulps", ulp_dem())]


def test_terrain_has_holes_flats_and_every_regime():
    from oracle import port
    u, ok = _terrain()
    assert (~ok).sum() > 50
    p0, _ = port.d8flowdir(port.pitremove(scaled_dem(0, False)), flats=False)
    assert (p0 == 0).sum() > 20, "the terrain must have flats after filling"
    d = np.abs(np.diff(scaled_dem(-140, False)[ok.all(axis=1)], axis=1))
    assert ((d > 0) & (d < 2.0 ** -126)).any(), "at 2^-140 the drops are subnormal"
    with np.errstate(over="ignore"):
        o = overflow_dem()
        assert np.isinf(np.diff(np.where(ok, o, 0.0).astype(np.float32), axis=1)).any()


# ---------------------------------------------------------------- the D-infinity pre-screen, restated
def _facets(fel, dx, dy):
    """the float ranking of k_dinf_stencil (squared slopes, its drop-rule bits) and the double VSLOPE quantities of every interior
    cell: st (8, n) float32, s2neg / clipsafe (8, n) bool, band (8, n) bool: the facet's |S2 D1 - S1 D2| lies inside VSLOPE's 1e-9 band"""
    f = np.asarray(fel, np.float32)
    z = f[1:-1, 1:-1]
    dxf, dyf = np.float32(dx), np.float32(dy)
    rdxf, rdyf, rddf = np.float32(1) / dxf, np.float32(1) / dyf, np.float32(1) / np.float32(np.sqrt(dx * dx + dy * dy))
    I1, J1 = (0, -1, -1, 0, 0, 1, 1, 0), (1, 0, 0, -1, -1, 0, 0, 1)         # row / column offsets of E1 and E2 (row 0 = north)
    I2, J2 = (-1, -1, -1, -1, 1, 1, 1, 1), (1, 1, -1, -1, -1, -1, 1, 1)
    ny, nx = f.shape
    sh = lambda i, j: f[1 + i:ny - 1 + i, 1 + j:nx - 1 + j]
    st, neg, csafe, band = [], [], [], []
    with np.errstate(all="ignore"):
        for K in range(8):
            d1x = K in (0, 3, 4, 7)
            e1, e2 = sh(I1[K], J1[K]), sh(I2[K], J2[K])
            r1, r2 = (rdxf, rdyf) if d1x else (rdyf, rdxf)
            d1f, d2f = (dxf, dyf) if d1x else (dyf, dxf)
            s1, s2 = (z - e1) * r1, (e1 - e2) * r2
            ng = e1 < e2
            x, y = s2 * d1f, s1 * d2f
            clip = np.where(z <= e1, ~((z == e1) & (e1 == e2)), x > y)
            cs = ~ng & np.where(z <= e1, ~((z == e1) & (e1 == e2)), x > y * np.float32(1.0001))
            lin = np.where(ng, s1, (z - e2) * rddf)
            q = np.where(ng | clip, np.where(lin > 0, lin * lin, np.float32(0)), s1 * s1 + s2 * s2)
            st.append(q.astype(np.float32)); neg.append(ng); csafe.append(cs)
            D1, D2 = (dx, dy) if d1x else (dy, dx)
            S1, S2 = (z.astype(np.float64) - e1) / D1, (e1.astype(np.float64) - e2) / D2
            X, Y = S2 * D1, S1 * D2
            band.append((S1 > 0) & (S2 >= 0) & (X <= Y * (1 + 1e-9)) & (X >= Y * (1 - 1e-9)))
    return np.array(st), np.array(neg), np.array(csafe), np.array(band)


def dinf_prescreen(fel, dx, dy):
    """per interior cell: the candidate count of the float pre-screen before and after its drop rules (k_dinf_stencil step 1), and
    whether a facet inside VSLOPE's 1e-9 band is a candidate"""
    st, neg, csafe, band = _facets(fel, dx, dy)
    smax = np.maximum(st.max(axis=0), np.float32(0))
    cand = (st >= smax * np.float32(0.99996)) & (st > 0)
    before = cand.sum(axis=0)
    A, B = cand & neg, cand & csafe
    drop = np.zeros_like(cand)
    for a, b in ((1, 2), (3, 4), (5, 6)):                # facets (2,3) (4,5) (6,7) share E1: the higher K goes
        drop[b] |= A[a] & A[b]
    drop[7] |= A[0] & A[7]                                 # (1, 8)
    for a in (0, 2, 4, 6):                                 # (1,2) (3,4) (5,6) (7,8) share E2
        drop[a + 1] |= B[a] & B[a + 1]
    after = (cand & ~drop).sum(axis=0)
    return before, after, (cand & band).any(axis=0)


def tie_grids():
    """(name, fel, cell sizes) of grids built to sit D-infinity cells on the tie rules of the stencil"""
    rng = np.random.default_rng(9)
    ny, nx = 70, 140
    i, j = np.mgrid[0:ny, 0:nx]
    out = []
    # isolated peaks one metre over a 100 m floor: 8 facets tie (dx = dy) or 4 (dx != dy); facets that share nothing, K order decides
    peaks = np.full((ny, nx), 100.0, np.float32)
    peaks[2::3, 2::3] = 101.0
    out.append(("peaks", peaks))
    # the same with every neighbour moved by -4..4 ulps (one ulp of 100 is 1.5e-5 of a squared slope of 1: inside and outside the band)
    out.append(("peaks +-ulps", (peaks.view(np.int32) + rng.integers(-4, 5, peaks.shape).astype(np.int32) * (peaks == 100.0)).view(np.float32)))
    # square and diamond pyramids and cones, 13 cells across: ties between mirror facets on the axes and the diagonals
    a, b = (i % 13) - 6, (j % 13) - 6
    out.append(("pyramids", (200.0 - np.maximum(np.abs(a), np.abs(b))).astype(np.float32)))
    out.append(("diamonds", (200.0 - (np.abs(a) + np.abs(b))).astype(np.float32)))
    cone = (200.0 - np.sqrt(a * a + b * b)).astype(np.float32)
    out.append(("cones", cone))
    out.append(("cones +-ulps", (cone.view(np.int32) + rng.integers(-4, 5, cone.shape).astype(np.int32)).view(np.float32)))
    # troughs running east: E1 = E lower than both diagonals, S2 < 0 on facets 1 and 8 (drop rule on a shared E1); the north and
    # south variants put the pairs (2,3) and (6,7) on it
    tr = (100.0 + 2.0 * np.abs((i % 7) - 3) - 0.25 * j).astype(np.float32)
    out.append(("troughs", tr))
    trn = (100.0 + 2.0 * np.abs((j % 7) - 3) + 0.25 * i).astype(np.float32)
    out.append(("troughs north", trn))
    out.append(("troughs +-ulps", (tr.view(np.int32) + rng.integers(-2, 3, tr.shape).astype(np.int32)).view(np.float32)))
    # valleys along the NE diagonal: E2 = NE much lower than E and N, facets 1 and 2 both clipped (drop rule on a shared E2)
    u = j - (ny - 1 - i)                                   # 0 on the diagonal through the SW corner, rows counted from the south
    diag = (300.0 - 0.5 * (j + (ny - 1 - i)) + 3.0 * np.abs(((u + 6) % 13) - 6)).astype(np.float32)
    out.append(("diagonal valleys", diag))
    # planes falling exactly along a facet diagonal (S2 D1 == S1 D2: VSLOPE's atan2 branch), and a few ulps either side of it
    for sx, sy in ((1, 1), (-1, 1), (-1, -1), (1, -1)):
        pl = (1000.0 - sx * j - sy * 4.0 * (ny - 1 - i)).astype(np.float32)    # with dx = 10, dy = 20 the fall line is the diagonal
        out.append((f"diagonal plane {sx},{sy}", pl))
    pl = (1000.0 - j - 4.0 * (ny - 1 - i)).astype(np.float32)
    out.append(("diagonal plane +-ulps", (pl.view(np.int32) + rng.integers(-3, 4, pl.shape).astype(np.int32)).view(np.float32)))
    sq = (1000.0 - j - (ny - 1 - i)).astype(np.float32)
    out.append(("square diagonal plane", sq))
    return out


TIE_SIZES = [(30.0, 30.0), (10.0, 20.0), (12.5, 40.0), (20.0, 10.0)]


def test_dinf_tie_grids_reach_the_tie_paths():
    """The pre-screen restated in numpy: the tie grids really put cells on several candidates, on both drop rules and on the 1e-9
    clip band of VSLOPE (else the tie tests below would test nothing)."""
    tot = many = dropped = band = 0
    per = {}
    for name, fel in tie_grids():
        for dx, dy in TIE_SIZES:
            b, a, bd = dinf_prescreen(fel, dx, dy)
            tot += b.size; many += int((a > 1).sum()); dropped += int((b > a).sum()); band += int(bd.sum())
            per[name] = per.get(name, 0) + int((a > 1).sum() + (b > a).sum() + bd.sum())
    assert many > tot // 10, (many, tot)
    assert dropped > 10000 and band > 20000, (dropped, band)
    assert all(v > 1000 for v in per.values()), per


# ---------------------------------------------------------------- emulated kernels (CPU)
@pytest.fixture(scope="module")
def emu():
    from test_emu import _build
    return _build()


def _emu_stencils(lib, fel, dx, dy):
    ny, nx = fel.shape
    f = np.ascontiguousarray(fel, np.float32)
    p = np.empty((ny, nx), np.int16); sd8 = np.empty((ny, nx), np.float32); n8 = np.zeros(1, np.uint64)
    assert lib.emu_d8_stencil(f.ctypes.data, p.ctypes.data, sd8.ctypes.data, nx, ny, FEL_ND, dx, dy, n8.ctypes.data) == 0
    ang = np.empty((ny, nx), np.float32); slp = np.empty((ny, nx), np.float32); nf = np.zeros(1, np.uint64)
    assert lib.emu_dinf_stencil(f.ctypes.data, ang.ctypes.data, slp.ctypes.data, nx, ny, FEL_ND, dx, dy, nf.ctypes.data) == 0
    return p, sd8, ang, slp, int(n8[0]), int(nf[0])


def _diffs(got, want):
    a, b = np.ascontiguousarray(got), np.ascontiguousarray(want)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return int((a != b).sum())


def _emu_check(lib, fel, dx, dy):
    """cells that differ from the restatement's positive-slope pass: {raster: count}"""
    from oracle import port
    p, sd8, ang, slp, n8, nf = _emu_stencils(lib, fel, dx, dy)
    p_r, sd8_r = port.d8flowdir(fel, dx=dx, dy=dy, flats=False)
    ang_r, slp_r = port.dinfflowdir(fel, dx=dx, dy=dy, flats=False)
    bad = {k: n for k, n in (("p", _diffs(p, p_r)), ("sd8", _diffs(sd8, sd8_r)), ("ang", _diffs(ang, ang_r)), ("slp", _diffs(slp, slp_r)),
                             ("d8 flats", abs(n8 - int((p_r == 0).sum()))), ("dinf flats", abs(nf - int((ang_r == -1.0).sum())))) if n}
    return bad


@pytest.mark.parametrize("dx,dy", SIZES)
def test_emulated_stencils_across_the_float_range(emu, dx, dy):
    """p, sd8, ang, slp and the flat counts of the emulated stencils against the restatement's positive-slope pass on the terrain at
    every scale 2^-149 .. 2^-40, a few normal scales, 2^126, 2^127, overflowing differences and an 8000 m + ulps grid."""
    from oracle import port
    fails = []
    for name, dem in dem_cases():
        fel = port.pitremove(dem)
        bad = _emu_check(emu, fel, dx, dy)
        if bad:
            fails.append(f"{name}: {bad}")
    assert not fails, f"{len(fails)} cases differ at {dx}x{dy}: " + "; ".join(fails[:40])


def test_emulated_dinf_stencil_ties_and_near_ties(emu):
    """The D-infinity counterpart of the D8 ties test: exact facet ties in K order, the two drop rules, float-neighbour perturbations
    inside and outside the candidate band, gradients on and next to a facet diagonal (VSLOPE's atan2 branch)."""
    fails = []
    for name, fel in tie_grids():
        for dx, dy in TIE_SIZES:
            bad = _emu_check(emu, fel, dx, dy)
            if bad:
                fails.append(f"{name} {dx}x{dy}: {bad}")
    assert not fails, "; ".join(fails)


# ---------------------------------------------------------------- the restatement on the reference tools
PINNED = [("2^-60", lambda: scaled_dem(-60, False)), ("2^-120 signed", lambda: scaled_dem(-120, True)), ("2^-140", lambda: scaled_dem(-140, False)),
          ("2^127 signed", lambda: scaled_dem(127, True)), ("overflow", overflow_dem)]
PIN_SIZES = [(30.0, 30.0), (12.5, 40.0)]


def _pinned_calls(R, dem):
    fel = R.pitremove(dem)
    return [("fel", fel)] + list(zip(("p", "sd8"), R.d8flowdir(fel))) + list(zip(("ang", "slp"), R.dinfflowdir(fel)))


def test_c_restatement_matches_the_live_reference_across_the_float_range(tmp_path, monkeypatch):
    """Where oracle/_ref is built: pitremove, d8flowdir and dinfflowdir (with flat resolution) of the restatement against the reference
    executables at 2^-60, 2^-120, 2^-140, 2^127 and on overflowing differences."""
    import port
    import refrun
    if not (refrun.available() and port.available()):
        pytest.skip("oracle/_ref not built")
    monkeypatch.setattr(refrun, "INPUTS_ONLY", False)
    for name, make in PINNED:
        dem = make()
        for dx, dy in PIN_SIZES:
            R = refrun.RefPipeline(workdir=str(tmp_path), dx=dx, dy=dy)
            fel = port.pitremove(dem)
            mine = [fel, *port.d8flowdir(fel, dx=dx, dy=dy), *port.dinfflowdir(fel, dx=dx, dy=dy)]
            for (n, r), o in zip(_pinned_calls(R, dem), mine):
                assert_bits(o, r, f"{name} {n} {dx}x{dy}")


def test_c_restatement_replays_the_reference_across_the_float_range(refrun, tmp_path):
    """The same calls against the reference outputs recorded in tests/golden/reference.json, recomputed by the restatement on the CPU;
    the count is asserted: a call that is not replayed fails here."""
    import port
    import reference
    if not port.available():
        pytest.skip("oracle/port not built")
    keys = set()
    for name, make in PINNED:
        dem = make()
        for dx, dy in PIN_SIZES:
            R = refrun.RefPipeline(workdir=str(tmp_path), dx=dx, dy=dy, np_ranks=1)
            before = set(reference.replayed)
            fel = R.pitremove(dem)
            R.d8flowdir(fel); R.dinfflowdir(fel)
            new = set(reference.replayed) - before
            assert len(new) == 3, (name, dx, dy)
            keys |= new
    assert len(keys) == len(PINNED) * len(PIN_SIZES) * 3 == 30


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def geographic_sizes(tmp_path_factory):
    """per-row metric cell sizes of a geographic raster (WGS84 ellipsoid) with the terrain's shape"""
    import taudem_b200 as td
    f = str(tmp_path_factory.mktemp("geo") / "geo.tif")
    write_geographic_dem(f, scaled_dem(0, False))
    dxc, dyc = np.zeros(NY), np.zeros(NY)
    assert td.lib().td_raster_cell_sizes(f.encode(), dxc.ctypes.data_as(C.c_void_p), dyc.ctypes.data_as(C.c_void_p), NY) == 0
    assert len(set(dxc)) > 1
    return dxc, dyc


def _gpu_check(dem, dx, dy, fill=True):
    """cells of the GPU pipeline that differ from the restatement's in any bit: {raster: count}"""
    import port
    import taudem_b200 as td
    fel_r = port.pitremove(dem) if fill else dem
    fel = td.pitremove_grid(dem) if fill else dem
    p_r, sd8_r = port.d8flowdir(fel_r, dx=dx, dy=dy)
    ang_r, slp_r = port.dinfflowdir(fel_r, dx=dx, dy=dy)
    p, sd8 = td.d8flowdir_grid(fel_r, dx=dx, dy=dy)
    ang, slp = td.dinfflowdir_grid(fel_r, dx=dx, dy=dy)
    # The one known difference: where a DEM holds both -0.0 and +0.0 (the signed terrain at 2^-149 .. 2^-139), which zero a filled
    # cell inherits depends on the order of the fill's updates, the reference's sequential one or the GPU's schedule.  Equal as
    # floats, so every later tool sees the same surface; any other bit difference of fel fails.
    zeros = (fel == 0) & (fel_r == 0)
    return {k: n for k, n in (("fel", _diffs(np.where(zeros, 0.0, fel).astype(np.float32), np.where(zeros, 0.0, fel_r).astype(np.float32))), ("p", _diffs(p, p_r)),
                              ("sd8", _diffs(sd8, sd8_r)), ("ang", _diffs(ang, ang_r)), ("slp", _diffs(slp, slp_r))) if n}


@pytest.mark.gpu
@pytest.mark.parametrize("dx,dy", SIZES + [(None, None)], ids=[f"{a}x{b}" for a, b in SIZES] + ["geographic"])
def test_gpu_stencils_across_the_float_range(dx, dy, request):
    """pitremove_grid -> d8flowdir_grid / dinfflowdir_grid (flat resolution included) against the restatement's pipeline on every
    scaled terrain: fel, p, sd8, ang and slp bit for bit."""
    if dx is None:
        dx, dy = request.getfixturevalue("geographic_sizes")
    fails = []
    for name, dem in dem_cases():
        bad = _gpu_check(dem, dx, dy)
        if bad:
            fails.append(f"{name}: {bad}")
    assert not fails, f"{len(fails)} cases differ: " + "; ".join(fails[:40])


@pytest.mark.gpu
def test_gpu_dinf_stencil_ties_and_near_ties():
    """The D-infinity tie grids through dinfflowdir_grid / d8flowdir_grid (flat resolution included) against the restatement."""
    fails = []
    for name, fel in tie_grids():
        for dx, dy in TIE_SIZES:
            bad = _gpu_check(fel, dx, dy, fill=False)
            if bad:
                fails.append(f"{name} {dx}x{dy}: {bad}")
    assert not fails, "; ".join(fails)
