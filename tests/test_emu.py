"""The kernels of taudem_b200/csrc (the warp-per-tile dataflow sweep with its scheduler / count protocols, the stencils,
the flat resolution, pit removal, the outlet restriction), executed on a CPU emulation of the CUDA thread model
(tests/emu: fibers, warp collectives, randomised interleavings) and compared bit for bit with the oracle.  This checks
protocol logic and arithmetic, not the GPU memory model — the GPU parity tests (tests/test_gpu_parity.py) do that."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from taudem_b200 import synth
from util import assert_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
CSRC = os.path.join(ROOT, "taudem_b200", "csrc")
BUILD = os.path.join(EMU, "_build")


STENCILS = ("d8_stencil", "dinf_stencil", "area_d8", "area_dinf")


def _transform(name, min_launches=6):
    """kernel<<<grid, block, smem, stream>>>(args);  ->  emu_launch(grid, block, [&]{ kernel(args); });"""
    src = open(os.path.join(CSRC, name + ".cu")).read()
    src = src.replace("extern __shared__ __align__(16) unsigned char dsm[];", "static __align__(16) unsigned char dsm[256 * 1024];")
    src = src.replace("extern __shared__ __align__(128) unsigned char dsm128[];", "static __align__(128) unsigned char dsm128[256 * 1024];")
    src, n = re.subn(r"(k_\w+(?:<[\w, ]+>)?)<<<([^,]+),\s*([^,]+),[^>]*>>>\(([^;]*)\);",
                     r"emu_launch(dim3(\2), dim3(\3), [&] { \1(\4); });", src)
    assert n >= min_launches and "<<<" not in src, (name, n)
    inc = os.path.join(BUILD, name + "_emu.inc")
    if not os.path.exists(inc) or open(inc).read() != src:
        open(inc, "w").write(src)
    return inc


def _build(tag="", defines=()):
    os.makedirs(BUILD, exist_ok=True)
    _transform("rowfact", 1)
    incs = [_transform("sweep_warp", 4), _transform("flats")] + [_transform(n, 1) for n in STENCILS] + [_transform("outlets", 2), _transform("fill", 3)]
    so = os.path.join(BUILD, f"libemu{tag}.so")
    objs = []
    for i, n in enumerate(STENCILS):                       # one translation unit per kernel file (their helper names collide)
        o = os.path.join(BUILD, f"stencil{i + 1}.o")
        deps_o = [incs[2 + i], os.path.join(EMU, "stencil_driver.cpp"), os.path.join(EMU, "cuda_runtime.h"), os.path.join(CSRC, "common.cuh"),
                  os.path.join(CSRC, "dinf_common.cuh"), os.path.join(CSRC, "tile_pipe.cuh"), os.path.join(CSRC, "rowfact.cuh"), os.path.join(BUILD, "rowfact_emu.inc")]
        if not os.path.exists(o) or any(os.path.getmtime(d) > os.path.getmtime(o) for d in deps_o):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-c", "-pthread", "-ftls-model=initial-exec", "-ffp-contract=off", "-I", EMU,
                                   "-I", BUILD, "-I", CSRC, f"-DEMU_WHICH={i + 1}", "-o", o, os.path.join(EMU, "stencil_driver.cpp")])
        objs.append(o)
    srcs = [os.path.join(EMU, f) for f in ("driver.cpp", "flats_driver.cpp", "fill_driver.cpp", "emu.cpp")] + objs
    deps = incs + srcs + [os.path.join(EMU, "cuda_runtime.h"), os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "dinf_common.cuh"),
                          os.path.join(CSRC, "ctx.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ftls-model=initial-exec", "-ffp-contract=off", "-I", EMU, "-I", BUILD, "-I", CSRC,
                               *[f"-D{d}" for d in defines], "-o", so, *srcs])
    lib = C.CDLL(so)
    lib.emu_sweep.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                              C.c_float, C.c_double, C.c_double, C.c_ulonglong, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    P = C.c_void_p
    lib.emu_set_dm.argtypes = [C.c_void_p, C.c_float]
    lib.emu_set_dm.restype = None
    lib.emu_set_extra.argtypes = [C.c_void_p, C.c_float, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
    lib.emu_set_extra.restype = None
    lib.emu_d8_stencil.argtypes = [P, P, P, C.c_int, C.c_int, C.c_float, C.c_double, C.c_double, P]
    lib.emu_dinf_stencil.argtypes = [P, P, P, C.c_int, C.c_int, C.c_float, C.c_double, C.c_double, P]
    lib.emu_deps_d8.argtypes = [P, P, P, P, C.c_int, C.c_int, C.c_short]
    lib.emu_deps_dinf.argtypes = [P, P, P, P, C.c_int, C.c_int, C.c_float, C.c_double, C.c_double]
    lib.emu_ref_deps.argtypes = [C.c_int, P, P, P, C.c_int, C.c_int, C.c_float, C.c_double, C.c_double]
    lib.emu_fill.argtypes = [P, P, P, C.c_int, C.c_int, C.c_float, C.c_int, C.c_ulonglong]
    lib.emu_flats.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_ulonglong, C.c_void_p, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def emu():
    return _build()


@pytest.fixture(scope="module")
def fields():
    from oracle import port
    dem = synth.punch_holes(synth.gen_dem(150, 190, hurst=0.8, tilt=1.0, seed=5))
    fel = port.pitremove(dem)
    p, _ = port.d8flowdir(fel)
    ang, _ = port.dinfflowdir(fel)
    w = synth.gen_weights(*dem.shape)
    return port, p, ang, w


def _run(lib, dinf, mode, passes, direction, w, contcheck, seed, nstrips=1, rounds=None, outlets=None, dx=30.0, dy=30.0):
    ny, nx = direction.shape
    out = np.empty((ny, nx), np.float32)
    d = np.ascontiguousarray(direction)
    wp = None if w is None else np.ascontiguousarray(w, np.float32)
    nodata = -3.4028234663852886e38 if dinf else -32768.0
    oc = None if outlets is None else np.ascontiguousarray(outlets[0], np.int32)
    orow = None if outlets is None else np.ascontiguousarray(outlets[1], np.int32)
    rc = lib.emu_sweep(int(dinf), mode, passes, d.ctypes.data, out.ctypes.data, None if wp is None else wp.ctypes.data, nx, ny, nodata,
                       int(w is not None), int(contcheck), -9999.0, dx, dy, seed, nstrips, None if rounds is None else rounds.ctypes.data,
                       None if oc is None else oc.ctypes.data, None if orow is None else orow.ctypes.data, -1 if oc is None else len(oc))
    assert rc == 0
    return out


def test_emulated_d8_sweep_matches_the_oracle(emu, fields):
    """The warp-per-tile dataflow sweep (sweep_warp.cu): every warp of the persistent CTA is an independent worker on 32 x 32
    tiles (ticket queue, four-state tile protocol, shared ready queue); randomised interleavings of the workers."""
    port, p, _, w = fields
    for seed in (1, 2, 3):
        assert_bits(_run(emu, False, 0, 0, p, None, True, seed), port.aread8(p), f"ad8 seed {seed}")
    assert_bits(_run(emu, False, 0, 0, p, w, False, 4), port.aread8(p, weights=w, contcheck=False), "ad8 -wg -nc")


def test_emulated_dinf_sweep_matches_the_oracle(emu, fields):
    """... D-infinity: row ready masks, fork stack, shares from the strip's prop() table with reciprocal divisions."""
    port, _, ang, w = fields
    for seed in (1, 2, 3):
        assert_bits(_run(emu, True, 0, 0, ang, None, True, seed), port.areadinf(ang), f"sca seed {seed}")
    assert_bits(_run(emu, True, 0, 0, ang, w, False, 4), port.areadinf(ang, weights=w, contcheck=False), "sca -wg -nc")


def test_emulated_dinf_angle_torture(emu):
    """areadinf on angles at and next to every place where prop() changes its mind (sector edges, the 1e-5 share threshold,
    the wrap sector, angles beyond 2 PI): the receiver field of the node words and the sector-table shares against the oracle."""
    from oracle import port
    from util import angle_torture
    for dx, dy in ((30.0, 30.0), (12.5, 40.0)):
        ang = angle_torture(dx=dx, dy=dy)
        ref = port.areadinf(ang, dx=dx, dy=dy)
        assert (ref >= 0).sum() > ang.size // 20
        assert_bits(_run(emu, True, 0, 0, ang, None, True, 21, dx=dx, dy=dy), ref, f"sca angle torture {dx}x{dy}")
        assert_bits(_run(emu, True, 0, 0, ang, None, False, 22, 3, dx=dx, dy=dy), port.areadinf(ang, dx=dx, dy=dy, contcheck=False), f"sca angle torture -nc, 3 strips {dx}x{dy}")


def test_emulated_d8_flow_path_extreme_up(emu, fields):
    """d8flowpathextremeup = the D8 sweep with the extreme-value algebra, against the reference executable
    (oracle/_ref/d8flowpathextremeup: D8flowpathextremeup.cpp compiled unchanged)."""
    import reference as refrun
    port, p, _, w = fields
    sa = (w * 100.0 - 20.0).astype(np.float32)
    R = refrun.RefPipeline()
    assert_bits(_run(emu, False, 10, 0, p, sa, True, 31), R.d8flowpathextremeup(p, sa, usemax=True), "ssa max")
    assert_bits(_run(emu, False, 11, 0, p, sa, False, 32), R.d8flowpathextremeup(p, sa, usemax=False, contcheck=False), "ssa min -nc")


def test_emulated_dinf_decay_accumulation(emu, fields):
    """dinfdecayaccum = the D-infinity sweep with the decaying-accumulation algebra, against the reference executable
    (oracle/_ref/dinfdecayaccum: dinfdecayaccum.cpp compiled unchanged)."""
    import reference as refrun
    port, _, ang, w = fields
    rng = np.random.default_rng(17)
    dm = rng.uniform(0.2, 1.0, ang.shape).astype(np.float32)
    dm[rng.random(ang.shape) < 0.002] = -9999.0              # nodata multipliers contaminate what they feed
    dmc = np.ascontiguousarray(dm)
    emu.emu_set_dm(dmc.ctypes.data, C.c_float(-9999.0))
    R = refrun.RefPipeline()
    assert_bits(_run(emu, True, 12, 0, ang, None, True, 41), R.dinfdecayaccum(ang, dm), "dsca")
    assert_bits(_run(emu, True, 12, 0, ang, w, False, 42), R.dinfdecayaccum(ang, dm, weights=w, contcheck=False), "dsca -wg -nc")


def _sibling_grids(shape, seed):
    """q / supply-like positive grids with a few nodata and non-positive cells, an indicator grid, a capacity grid"""
    rng = np.random.default_rng(seed)
    q = rng.uniform(0.5, 3.0, shape).astype(np.float32)
    q[rng.random(shape) < 0.003] = -9999.0
    q[rng.random(shape) < 0.003] = 0.0
    dm = rng.uniform(0.2, 1.0, shape).astype(np.float32)
    dm[rng.random(shape) < 0.002] = -9999.0
    dg = (rng.random(shape) < 0.02).astype(np.int16)
    tc = rng.uniform(0.0, 8.0, shape).astype(np.float32)
    tc[rng.random(shape) < 0.002] = -9999.0
    cs = rng.uniform(0.0, 2.0, shape).astype(np.float32)
    cs[rng.random(shape) < 0.002] = -9999.0
    return q, dm, dg, tc, cs


def _outlet_points(port, ang, R):
    """three outlet cells (nested and disjoint basins) as grid coordinates and as a point shapefile in the reference's work directory"""
    from util import write_point_shapefile
    ny, nx = ang.shape
    order = np.argsort(port.areadinf(ang, contcheck=False).ravel())
    cells = [int(order[-1]), int(order[-40]), int(order[-300])]
    cols = [c % nx for c in cells]; rows = [c // nx for c in cells]
    shp = R.path("outlets.shp")
    write_point_shapefile(shp, [(c + 0.5) * 30.0 for c in cols], [30.0 * ny - (r + 0.5) * 30.0 for r in rows])
    return (cols, rows), shp


def test_emulated_dinf_conc_lim_accumulation(emu, fields):
    """DinfConcLimAccum = the D-infinity sweep with the concentration-limited algebra (7), against the reference executable
    (oracle/_ref/dinfconclimaccum: DinfConcLimAccum.cpp compiled unchanged); with and without contamination checking."""
    import reference as refrun
    port, _, ang, _ = fields
    q, dm, dg, _, _ = _sibling_grids(ang.shape, 23)
    dmc, dgc = np.ascontiguousarray(dm), np.ascontiguousarray(dg)
    emu.emu_set_dm(dmc.ctypes.data, C.c_float(-9999.0))
    emu.emu_set_extra(dgc.ctypes.data, C.c_float(2.5), None, C.c_float(0.0), None, None)
    R = refrun.RefPipeline()
    assert_bits(_run(emu, True, 16, 0, ang, q, True, 61), R.dinfconclimaccum(ang, dm, q, dg, csol=2.5), "ctpt")
    assert_bits(_run(emu, True, 16, 0, ang, q, False, 62), R.dinfconclimaccum(ang, dm, q, dg, csol=2.5, contcheck=False), "ctpt -nc")
    outs, shp = _outlet_points(port, ang, R)
    assert_bits(_run(emu, True, 16, 0, ang, q, False, 63, outlets=outs), R.dinfconclimaccum(ang, dm, q, dg, csol=2.5, contcheck=False, outlets=shp), "ctpt -nc -o")
    emu.emu_set_dm(None, C.c_float(0.0))


def test_emulated_dinf_trans_lim_accumulation(emu, fields):
    """DinfTransLimAccum = the D-infinity sweep with the transport-limited algebra (8; 9 with a concentration that travels in global
    memory), against the reference executable (oracle/_ref/dinftranslimaccum: DinfTransLimAccum.cpp compiled unchanged)."""
    import reference as refrun
    port, _, ang, _ = fields
    tsup, _, _, tc, cs = _sibling_grids(ang.shape, 29)
    tcc, csc = np.ascontiguousarray(tc), np.ascontiguousarray(cs)
    dep, cout = np.empty(ang.shape, np.float32), np.empty(ang.shape, np.float32)
    emu.emu_set_dm(tcc.ctypes.data, C.c_float(-9999.0))
    R = refrun.RefPipeline()
    emu.emu_set_extra(None, C.c_float(0.0), None, C.c_float(0.0), dep.ctypes.data, None)
    tla = _run(emu, True, 17, 0, ang, tsup, True, 71)
    rt, rd, _ = R.dinftranslimaccum(ang, tsup, tc)
    assert_bits(tla, rt, "tla"); assert_bits(dep, rd, "tdep")
    for contcheck, seed in ((True, 72), (False, 73)):
        emu.emu_set_extra(None, C.c_float(0.0), csc.ctypes.data, C.c_float(-9999.0), dep.ctypes.data, cout.ctypes.data)
        tla = _run(emu, True, 18, 0, ang, tsup, contcheck, seed)
        rt, rd, rc = R.dinftranslimaccum(ang, tsup, tc, cs=cs, contcheck=contcheck)
        assert_bits(tla, rt, "tla (cs)"); assert_bits(dep, rd, "tdep (cs)"); assert_bits(cout, rc, "ctpt")
    outs, shp = _outlet_points(port, ang, R)
    tla = _run(emu, True, 18, 0, ang, tsup, False, 74, outlets=outs)
    rt, rd, rc = R.dinftranslimaccum(ang, tsup, tc, cs=cs, contcheck=False, outlets=shp)
    assert_bits(tla, rt, "tla -o"); assert_bits(dep, rd, "tdep -o"); assert_bits(cout, rc, "ctpt -o")
    assert 100 < int((tla > -1e38).sum()) < tla.size
    emu.emu_set_dm(None, C.c_float(0.0))


def test_emulated_gridnet(emu, fields):
    """gridnet = three D8 sweeps (longest upstream path, total upstream path, Strahler order), against the reference executable
    (oracle/_ref/gridnet: gridnet.cpp compiled unchanged); with and without a mask grid."""
    import reference as refrun
    port, p, _, _ = fields
    R = refrun.RefPipeline()

    def ours(skip):
        out = []
        for mode in (13, 14, 15):
            ny, nx = p.shape
            res = np.empty((ny, nx), np.float32)
            d = np.ascontiguousarray(p)
            rc = emu.emu_sweep(0, mode, 0, d.ctypes.data, res.ctypes.data, None, nx, ny, -32768.0, 0, 0, skip, 30.0, 30.0, 50 + mode, 1, None, None, None, -1)
            assert rc == 0
            out.append(res)
        return out[0], out[1], out[2].astype(np.int16)

    emu.emu_set_dm(None, C.c_float(0.0))
    plen, tlen, gord = ours(-1.0)
    rp, rt, rg = R.gridnet(p)
    assert_bits(plen, rp, "plen"); assert_bits(tlen, rt, "tlen"); assert_bits(gord, rg, "gord")
    assert gord.max() >= 3
    ad8 = port.aread8(p, contcheck=False)
    mask = np.where(ad8 >= 0, ad8, 0).astype(np.int32)              # "streams": cells with at least 5 cells draining through them
    ok = np.ascontiguousarray((mask >= 5).astype(np.float32))
    emu.emu_set_dm(ok.ctypes.data, C.c_float(0.0))
    plen, tlen, gord = ours(-1.0)
    emu.emu_set_dm(None, C.c_float(0.0))
    rp, rt, rg = R.gridnet(p, mask=mask, thresh=5)
    assert_bits(plen, rp, "plen -mask"); assert_bits(tlen, rt, "tlen -mask"); assert_bits(gord, rg, "gord -mask")


def test_emulated_small_stacks_spill(fields):
    """A two-entry fork stack drops nearly every second receiver (the rescan of the shared-memory counts must find them);
    the outlet flood with a four-entry stack per warp spills nearly every discovered contributor to the host-drained list."""
    port, _, ang, w = fields
    lib = _build("_wstk2", ["TD_WSTK=2", "TD_UP_UQ=4"])
    assert_bits(_run(lib, True, 0, 0, ang, None, True, 7), port.areadinf(ang), "sca, fork stack of 2")
    assert_bits(_run(lib, True, 0, 0, ang, w, False, 8), port.areadinf(ang, weights=w, contcheck=False), "sca -wg -nc, fork stack of 2")
    full = port.areadinf(ang)
    c = int(np.argsort(full.ravel())[-1]); outs = ([c % ang.shape[1]], [c // ang.shape[1]])
    assert_bits(_run(lib, True, 0, 0, ang, None, True, 9, outlets=outs), port.areadinf(ang, outlets=outs), "sca -o, spilling flood")


@pytest.mark.parametrize("nstrips", [2, 3])
def test_emulated_row_strips_with_exchange_rounds(emu, fields, nstrips):
    """The row-strip protocol of the sweep (halo decrement counts, area rows, k_wapply_halo re-activating the tiles whose
    cells became ready, one kernel per round) reproduces the single-strip rasters."""
    port, p, ang, w = fields
    rounds = np.zeros(1, np.int32)
    assert_bits(_run(emu, False, 1, 3, p, None, True, 11, nstrips, rounds), port.aread8(p), "ad8 strips")
    assert rounds[0] > 1
    assert_bits(_run(emu, False, 0, 0, p, w, False, 12, nstrips), port.aread8(p, weights=w, contcheck=False), "ad8 -wg -nc strips")
    assert_bits(_run(emu, True, 1, 3, ang, None, True, 13, nstrips, rounds), port.areadinf(ang), "sca strips")
    assert rounds[0] > 1
    assert_bits(_run(emu, True, 0, 0, ang, w, False, 14, nstrips), port.areadinf(ang, weights=w, contcheck=False), "sca -wg -nc strips")


# ---------------------------------------------------------------- flat resolution (taudem_b200/csrc/flats.cu)
@pytest.fixture(scope="module")
def terraces():
    """A filled DEM with wide flats (quantised elevations: terraces with higher and lower rims) and nodata holes."""
    from oracle import port
    dem = synth.gen_dem(120, 150, hurst=0.8, tilt=1.0, seed=17)
    q = (dem.max() - dem.min()) / 14
    dem = (np.round(dem / q) * q).astype(np.float32)
    dem = synth.punch_holes(dem, seed=3)
    fel = port.pitremove(dem)
    return port, fel


def _flats(lib, dinf, fel, d0, nstrips, seed, dx=30.0, dy=30.0):
    ny, nx = fel.shape
    d = np.ascontiguousarray(d0).copy()
    left = np.zeros(1, np.int64); coll = np.zeros(1, np.int64)
    rc = lib.emu_flats(int(dinf), np.ascontiguousarray(fel, np.float32).ctypes.data, d.ctypes.data, nx, ny, dx, dy, nstrips, seed,
                       left.ctypes.data, coll.ctypes.data)
    assert rc == 0
    return d, int(left[0]), int(coll[0])


@pytest.mark.parametrize("nstrips", [1, 2, 3, 5])
def test_emulated_flat_resolution_d8(emu, terraces, nstrips):
    port, fel = terraces
    p0, _ = port.d8flowdir(fel, flats=False)
    p_ref, _ = port.d8flowdir(fel)
    assert (p0 == 0).sum() > 2000, "the test DEM must have wide flats"
    p, left, coll = _flats(emu, False, fel, p0, nstrips, 21 + nstrips)
    assert_bits(p, p_ref, f"p, {nstrips} strips")
    assert left == int((p_ref == 0).sum()) and (nstrips == 1 or coll > 10)


@pytest.mark.parametrize("nstrips", [1, 2, 3, 5])
def test_emulated_flat_resolution_dinf(emu, terraces, nstrips):
    port, fel = terraces
    a0, _ = port.dinfflowdir(fel, flats=False)
    a_ref, _ = port.dinfflowdir(fel)
    a, left, _ = _flats(emu, True, fel, a0, nstrips, 31 + nstrips)
    assert_bits(a, a_ref, f"ang, {nstrips} strips")


# ---------------------------------------------------------------- stencil and dependency kernels
def test_emulated_slope_stencils_match_the_oracle(emu, terraces):
    """k_d8_stencil / k_dinf_stencil (positive-slope pass): p, sd8, ang, slp bit for bit, and the flat count."""
    port, fel = terraces
    ny, nx = fel.shape
    f = np.ascontiguousarray(fel, np.float32)
    for dx, dy in ((30.0, 30.0), (10.0, 25.0)):
        p = np.empty((ny, nx), np.int16); sd8 = np.empty((ny, nx), np.float32); nflat = np.zeros(1, np.uint64)
        assert emu.emu_d8_stencil(f.ctypes.data, p.ctypes.data, sd8.ctypes.data, nx, ny, -3.0e38, dx, dy, nflat.ctypes.data) == 0
        p_ref, sd8_ref = port.d8flowdir(fel, dx=dx, dy=dy, flats=False)
        assert_bits(p, p_ref, f"p (stencil) {dx}x{dy}"); assert_bits(sd8, sd8_ref, f"sd8 {dx}x{dy}")
        assert int(nflat[0]) == int((p_ref == 0).sum())
        ang = np.empty((ny, nx), np.float32); slp = np.empty((ny, nx), np.float32)
        assert emu.emu_dinf_stencil(f.ctypes.data, ang.ctypes.data, slp.ctypes.data, nx, ny, -3.0e38, dx, dy, nflat.ctypes.data) == 0
        ang_ref, slp_ref = port.dinfflowdir(fel, dx=dx, dy=dy, flats=False)
        assert_bits(ang, ang_ref, f"ang (stencil) {dx}x{dy}"); assert_bits(slp, slp_ref, f"slp {dx}x{dy}")
        assert int(nflat[0]) == int((ang_ref == -1.0).sum())


def test_emulated_dependency_stencils(emu, fields):
    """k_deps_d8 / k_deps_dinf against the plain-loop restatement the emulated sweeps are fed with."""
    _, p, ang, _ = fields
    ny, nx = p.shape
    rng = np.random.default_rng(3)
    podd = p.copy()                                       # direction codes outside 0..8 (the generic path of k_deps_d8) and zeros
    idx = rng.integers(0, p.size, 400)
    podd.ravel()[idx] = rng.choice(np.array([0, 0, 9, 10, 12, -1, -3, 100, -32768], np.int16), 400)
    from util import angle_torture
    MISS = -3.4028234663852886e38
    cases = [(0, np.ascontiguousarray(p), -32768.0, 30.0, 30.0), (0, np.ascontiguousarray(podd), -32768.0, 30.0, 30.0),
             (1, np.ascontiguousarray(ang), MISS, 30.0, 30.0)]
    # angles on, next to and around every sector edge and every threshold of the float pre-screens (square and oblong cells)
    cases += [(1, angle_torture(ny=ny, nx=nx, dx=dx, dy=dy, seed=7 + i), MISS, dx, dy) for i, (dx, dy) in enumerate(((30.0, 30.0), (30.0, 20.0), (10.0, 45.0)))]
    for dx, dy in ((30.0, 30.0), (30.0, 12.0)):           # random angles within +-1.2e-5 sector widths of the edges, and float neighbours of the edges
        t = np.arctan2(dy, dx); PI = 3.14159265359
        edges = np.array([0.0, t, 0.5 * PI, PI - t, PI, PI + t, 1.5 * PI, 2 * PI - t, 2 * PI])
        e = rng.integers(0, 9, (ny, nx))
        w = np.minimum(np.diff(edges, append=edges[-1] + t)[e], np.diff(edges, prepend=-t)[e])
        near = (edges[e] + rng.uniform(-1.2e-5, 1.2e-5, (ny, nx)) * w).astype(np.float32)
        ulps = rng.integers(-3, 4, (ny, nx))
        snap = rng.random((ny, nx)) < 0.3
        near[snap] = (np.ascontiguousarray(edges[e].astype(np.float32)).view(np.int32) + ulps.astype(np.int32))[snap].view(np.float32)
        near[near < 0] = 0.0
        cases.append((1, np.ascontiguousarray(near, np.float32), MISS, dx, dy))
    for dinf, d, nd, dx, dy in cases:
        node = np.empty((ny, nx), np.uint16); cnt = np.empty((ny, nx), np.uint8); area = np.empty((ny, nx), np.float32)
        rn = np.empty((ny, nx), np.uint16); rc = np.empty((ny, nx), np.uint8)
        if dinf:
            assert emu.emu_deps_dinf(d.ctypes.data, node.ctypes.data, cnt.ctypes.data, area.ctypes.data, nx, ny, nd, dx, dy) == 0
        else:
            assert emu.emu_deps_d8(d.ctypes.data, node.ctypes.data, cnt.ctypes.data, area.ctypes.data, nx, ny, int(nd)) == 0
        assert emu.emu_ref_deps(dinf, d.ctypes.data, rn.ctypes.data, rc.ctypes.data, nx, ny, nd, dx, dy) == 0
        assert np.array_equal(cnt, rc), f"counts dinf={dinf}: {int((cnt != rc).sum())} differ"
        assert np.array_equal(node, rn), f"node words dinf={dinf}: {int((node != rn).sum())} differ"
        assert np.all(area == -1.0)


def test_emulated_d8_stencil_ties_and_near_ties(emu):
    """Exact ties (quantised elevations) and drops that are adjacent floats whose slopes round to the same float32: the
    scan-order rule of the reference (first k in 1,3,5,7,2,4,6,8 with the strictly largest rounded slope) must survive
    the three-product shortcut.  (Without the literal fallback of d8_cell about 170 cells of the second grid differ.)"""
    from oracle import port
    rng = np.random.default_rng(5)
    ny, nx = 96, 128
    base = (1000.0 + rng.integers(0, 4, (ny, nx)) * 2.5).astype(np.float32)          # many exact ties
    grids = [(base.view(np.int32) + rng.integers(-3, 4, (ny, nx)).astype(np.int32)).view(np.float32)]
    # peaks near 1000 over a floor near 10 / 26: the drops lie in the top of a binade, where neighbouring float drops
    # collapse onto one slope after the multiplication by 1/distance
    rng = np.random.default_rng(7)
    ny, nx = 192, 256
    g = (10.0 + rng.integers(0, 2, (ny, nx)) * 16.0 + rng.integers(-4, 5, (ny, nx)) * 3.0e-5).astype(np.float32)
    g[1::3, 1::3] = (np.float32(1000.0).view(np.int32) + rng.integers(-2, 3, g[1::3, 1::3].shape).astype(np.int32)).view(np.float32)
    grids.append(g)
    for fel in grids:
        ny, nx = fel.shape
        f = np.ascontiguousarray(fel)
        for dx, dy in ((30.0, 30.0), (30.0, 30.000001), (12.5, 40.0), (7.0, 7.1)):
            p = np.empty((ny, nx), np.int16); sd8 = np.empty((ny, nx), np.float32); nflat = np.zeros(1, np.uint64)
            assert emu.emu_d8_stencil(f.ctypes.data, p.ctypes.data, sd8.ctypes.data, nx, ny, -3.0e38, dx, dy, nflat.ctypes.data) == 0
            p_ref, sd8_ref = port.d8flowdir(fel, dx=dx, dy=dy, flats=False)
            assert_bits(p, p_ref, f"p ties {dx}x{dy}"); assert_bits(sd8, sd8_ref, f"sd8 ties {dx}x{dy}")


def test_emulated_outlets_restrict_the_sweep(emu, fields):
    """-o: k_upstream floods the contributor links from the outlet cells, k_restrict removes every other cell from the
    flow field; the sweep then evaluates exactly what the reference's outlet branch evaluates."""
    port, p, ang, w = fields
    full = port.aread8(p)
    order = np.argsort(full.ravel())
    ny, nx = p.shape
    cells = [int(order[-1]), int(order[-40]), int(order[-300]), int(order[len(order) // 2])]      # nested and disjoint basins, a small one
    outs = ([c % nx for c in cells] + [-5, nx + 3], [c // nx for c in cells] + [2, 1])              # two points off the grid are ignored
    ref = port.aread8(p, outlets=outs)
    assert 100 < int((ref != -1).sum()) < p.size
    assert_bits(_run(emu, False, 1, 3, p, None, True, 61, outlets=outs), ref, "ad8 -o")
    assert_bits(_run(emu, False, 0, 0, p, w, False, 62, outlets=outs), port.aread8(p, weights=w, contcheck=False, outlets=outs), "ad8 -o -wg -nc")
    assert_bits(_run(emu, True, 1, 3, ang, None, True, 63, outlets=outs), port.areadinf(ang, outlets=outs), "sca -o")
    assert_bits(_run(emu, False, 0, 0, p, None, True, 64, outlets=([], [])), np.full(p.shape, -1.0, np.float32), "ad8 -o without points")
    # an outlet on a cell WITHOUT a flow direction (a grid-edge cell that interior cells drain into; ADVICE r1): the reference floods
    # its contributors and evaluates it (contaminated here: it has off-grid neighbours) — not "ignored"
    d1 = np.array([0, 1, 1, 0, -1, -1, -1, 0, 1]); d2 = np.array([0, 0, -1, -1, -1, 0, 1, 1, 1])
    edge = [(r, c) for r in range(ny) for c in (0, nx - 1) for k in range(1, 9)
            if 0 <= r - d2[k] < ny and 0 <= c - d1[k] < nx and p[r - d2[k], c - d1[k]] == k and not (1 <= p[r, c] <= 8)]
    assert edge, "the test field has no interior cell draining into an edge cell"
    er, ec = edge[len(edge) // 2]
    eo = ([ec], [er])
    ref_e = port.aread8(p, contcheck=False, outlets=eo)
    assert int((ref_e != -1).sum()) > 1, "the oracle evaluates the outlet and its upstream cells"
    assert_bits(_run(emu, False, 0, 0, p, None, False, 67, outlets=eo), ref_e, "ad8 -o -nc, outlet on an edge cell")
    assert_bits(_run(emu, False, 0, 0, p, None, True, 68, outlets=eo), port.aread8(p, outlets=eo), "ad8 -o, outlet on an edge cell")
    # row strips: the flood crosses the strip boundaries in rounds of requests
    for n in (2, 5):
        assert_bits(_run(emu, False, 1, 3, p, None, True, 65, n, outlets=outs), ref, f"ad8 -o, {n} strips")
        assert_bits(_run(emu, True, 1, 3, ang, None, True, 66, n, outlets=outs), port.areadinf(ang, outlets=outs), f"sca -o, {n} strips")


@pytest.mark.parametrize("rows_per_strip", [1, 2, 3])
def test_emulated_thin_strips(emu, rows_per_strip):
    """Strip heights of one to three rows (SURVEY.md extra parity cases): flat resolution and both sweeps over row strips
    whose first and last row coincide or touch."""
    from oracle import port
    ny, nx = 18, 70
    dem = synth.gen_dem(ny, nx, hurst=0.8, tilt=1.0, seed=23)
    q = (dem.max() - dem.min()) / 6
    dem = (np.round(dem / q) * q).astype(np.float32)
    fel = port.pitremove(dem)
    n = ny // rows_per_strip
    p0, _ = port.d8flowdir(fel, flats=False); p_ref, _ = port.d8flowdir(fel)
    assert (p0 == 0).sum() > 50
    p, _, _ = _flats(emu, False, fel, p0, n, 71)
    assert_bits(p, p_ref, f"p, {n} strips of {rows_per_strip} rows")
    a0, _ = port.dinfflowdir(fel, flats=False); a_ref, _ = port.dinfflowdir(fel)
    a, _, _ = _flats(emu, True, fel, a0, n, 72)
    assert_bits(a, a_ref, f"ang, {n} strips of {rows_per_strip} rows")
    assert_bits(_run(emu, False, 1, 2, p_ref, None, True, 73, n), port.aread8(p_ref), "ad8 thin strips")
    assert_bits(_run(emu, True, 1, 2, a_ref, None, True, 74, n), port.areadinf(a_ref), "sca thin strips")


@pytest.mark.parametrize("name", ["tiny", "plateau", "lake", "hills_holes", "rough"])
def test_emulated_pipeline_reproduces_the_reference_golden_vectors(emu, name):
    """fel (golden) -> emulated k_d8_stencil / k_dinf_stencil -> emulated flat resolution (1 and 2 strips) -> emulated
    dependency state, level passes, walkers and rivers: p, sd8, ang, slp, ad8, sca of the REFERENCE-generated golden
    vectors (tests/golden/make_golden.py), bit for bit."""
    from util import load_golden
    g = load_golden(name)
    fel = np.ascontiguousarray(g["fel"], np.float32)
    ny, nx = fel.shape
    dx, dy = float(g["dx"]), float(g["dy"])
    f = fel
    p = np.empty((ny, nx), np.int16); sd8 = np.empty((ny, nx), np.float32); nflat = np.zeros(1, np.uint64)
    assert emu.emu_d8_stencil(f.ctypes.data, p.ctypes.data, sd8.ctypes.data, nx, ny, -3.0e38, dx, dy, nflat.ctypes.data) == 0
    assert_bits(sd8, g["sd8"], "sd8")
    ang = np.empty((ny, nx), np.float32); slp = np.empty((ny, nx), np.float32)
    assert emu.emu_dinf_stencil(f.ctypes.data, ang.ctypes.data, slp.ctypes.data, nx, ny, -3.0e38, dx, dy, nflat.ctypes.data) == 0
    assert_bits(slp, g["slp"], "slp")
    for strips in ((1, 2) if ny >= 8 else (1,)):
        pr, _, _ = _flats(emu, False, fel, p, strips, 81, dx, dy)
        assert_bits(pr, g["p"], f"p ({strips} strips)")
        ar, _, _ = _flats(emu, True, fel, ang, strips, 82, dx, dy)
        assert_bits(ar, g["ang"], f"ang ({strips} strips)")
    w = np.ascontiguousarray(g["w"], np.float32)
    assert_bits(_run(emu, False, 1, 3, g["p"], None, True, 83, dx=dx, dy=dy), g["ad8"], "ad8")
    assert_bits(_run(emu, False, 0, 0, g["p"], w, True, 84, dx=dx, dy=dy), g["ad8_w"], "ad8 -wg")
    assert_bits(_run(emu, False, 1, 3, g["p"], None, False, 85, dx=dx, dy=dy), g["ad8_nc"], "ad8 -nc")
    assert_bits(_run(emu, True, 1, 3, g["ang"], None, True, 86, dx=dx, dy=dy), g["sca"], "sca")
    assert_bits(_run(emu, True, 0, 0, g["ang"], w, True, 87, dx=dx, dy=dy), g["sca_w"], "sca -wg")
    assert_bits(_run(emu, True, 1, 3, g["ang"], None, False, 88, dx=dx, dy=dy), g["sca_nc"], "sca -nc")


def test_emulated_sweep_on_the_reference_golden_vectors(emu):
    """The sweep on the reference-generated golden vectors (nodata holes, dx != dy, plateau, lake, 5 x 7 grid)."""
    from util import golden_cases, load_golden
    for name in golden_cases():
        g = load_golden(name)
        dx, dy = float(g["dx"]), float(g["dy"])
        assert_bits(_run(emu, False, 0, 0, g["p"], None, True, 111, dx=dx, dy=dy), g["ad8"], f"{name} ad8")
        assert_bits(_run(emu, False, 0, 0, g["p"], g["w"], True, 112, dx=dx, dy=dy), g["ad8_w"], f"{name} ad8 -wg")
        assert_bits(_run(emu, True, 0, 0, g["ang"], None, True, 113, dx=dx, dy=dy), g["sca"], f"{name} sca")
        assert_bits(_run(emu, True, 0, 0, g["ang"], g["w"], True, 114, dx=dx, dy=dy), g["sca_w"], f"{name} sca -wg")
        assert_bits(_run(emu, True, 0, 0, g["ang"], None, False, 115, dx=dx, dy=dy), g["sca_nc"], f"{name} sca -nc")


def test_emulated_pitremove(emu):
    """k_fill_init + k_fill_relax (tile-local Planchon-Darboux relaxation, active-tile lists): fel of the reference-generated
    golden vectors, 8- and 4-way, and the depression mask case."""
    from util import load_golden
    for name in ("tiny", "plateau", "lake", "hills_holes", "rough"):
        g = load_golden(name)
        dem = np.ascontiguousarray(g["dem"], np.float32); ny, nx = dem.shape
        for four, key in ((0, "fel"), (1, "fel4")):
            out = np.empty_like(dem)
            assert emu.emu_fill(dem.ctypes.data, out.ctypes.data, None, nx, ny, -9999.0, four, 5) == 0
            assert_bits(out, g[key], f"{name} {key}")
        if "depmask" in g:
            m = np.ascontiguousarray(g["depmask"], np.int16)
            for four, key in ((0, "fel_mask"), (1, "fel_mask4")):
                out = np.empty_like(dem)
                assert emu.emu_fill(dem.ctypes.data, out.ctypes.data, m.ctypes.data, nx, ny, -9999.0, four, 6) == 0
                assert_bits(out, g[key], f"{name} {key}")


@pytest.mark.parametrize("batch", [1, 3, 64])
def test_emulated_flat_resolution_batched_levels(emu, terraces, batch, monkeypatch):
    """TAUDEM_B200_FLATS_BATCH: several BFS levels per host round trip (k_bfs_level: device-resident level bounds, the last
    block of a level records where it ends) — same directions, D8 and D-infinity, and the golden plateau / lake cases."""
    from util import load_golden
    port, fel = terraces
    monkeypatch.setenv("TAUDEM_B200_FLATS_BATCH", str(batch))
    p0, _ = port.d8flowdir(fel, flats=False); p_ref, _ = port.d8flowdir(fel)
    assert_bits(_flats(emu, False, fel, p0, 1, 101)[0], p_ref, f"p, batch {batch}")
    a0, _ = port.dinfflowdir(fel, flats=False); a_ref, _ = port.dinfflowdir(fel)
    assert_bits(_flats(emu, True, fel, a0, 1, 102)[0], a_ref, f"ang, batch {batch}")
    for name in ("plateau", "lake"):
        g = load_golden(name)
        f = np.ascontiguousarray(g["fel"], np.float32)
        q0, _ = port.d8flowdir(f, dx=float(g["dx"]), dy=float(g["dy"]), flats=False)
        assert_bits(_flats(emu, False, f, q0, 1, 103, float(g["dx"]), float(g["dy"]))[0], g["p"], f"{name} p, batch {batch}")


def test_emulated_sweeps_on_a_larger_grid(emu):
    """500 x 700 cells (352 tiles, rivers of several hundred cells): single strip and four strips."""
    from oracle import port
    dem = synth.punch_holes(synth.gen_dem(500, 700, hurst=0.8, tilt=1.0, seed=31))
    fel = port.pitremove(dem); p, _ = port.d8flowdir(fel); ang, _ = port.dinfflowdir(fel)
    ad8 = port.aread8(p); sca = port.areadinf(ang)
    assert ad8.max() > 1.0e4
    assert_bits(_run(emu, False, 0, 0, p, None, True, 203), ad8, "ad8")
    assert_bits(_run(emu, True, 0, 0, ang, None, True, 204), sca, "sca")
    assert_bits(_run(emu, False, 0, 0, p, None, True, 205, 4), ad8, "ad8, 4 strips")
    assert_bits(_run(emu, True, 0, 0, ang, None, True, 206, 4), sca, "sca, 4 strips")


def test_emulated_random_configurations(emu):
    """A short deterministic slice of scripts/emu_stress.py: random grid sizes, flats, holes, strip counts, sweeps and strip
    flats against the oracle; every sibling algebra 1-9 at least once on random value grids."""
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "emu_stress.py"), "777", "14", "120"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and " bad 0 " in r.stdout, r.stdout[-2000:]
    runs = r.stdout.split("algebra runs ")[1].split()[0]
    assert all(int(n) >= 1 for n in runs.split(",")) and len(runs.split(",")) == 9, r.stdout[-2000:]


def test_emulated_sibling_tools_on_the_golden_vectors(emu):
    """The sibling sweep tools (algebras 1-9 of sweep_warp.cu) on the emulated thread model against tests/golden/siblings.npz — outputs of
    the reference executables (tests/golden/make_golden.py::siblings) on the hills_holes case, whose cells are 30 x 20 m (oblong: the
    prop() table is not the square one)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "hills_holes.npz"))
    x = np.load(os.path.join(ROOT, "tests", "golden", "siblings.npz"))
    dx, dy = float(g["dx"]), float(g["dy"])
    p, ang, w = g["p"], g["ang"], g["w"]
    ny, nx = p.shape
    kw = dict(dx=dx, dy=dy)
    assert_bits(_run(emu, False, 10, 0, p, x["sa"], True, 81, **kw), x["ssa_max"], "ssa max")
    assert_bits(_run(emu, False, 11, 0, p, x["sa"], False, 82, **kw), x["ssa_min_nc"], "ssa min -nc")

    def gridnet(okgrid):
        out = []
        for mode in (13, 14, 15):
            res = np.empty((ny, nx), np.float32)
            d = np.ascontiguousarray(p)
            emu.emu_set_dm(None if okgrid is None else okgrid.ctypes.data, C.c_float(0.0))
            assert emu.emu_sweep(0, mode, 0, d.ctypes.data, res.ctypes.data, None, nx, ny, -32768.0, 0, 0, -1.0, dx, dy, 90 + mode, 1, None, None, None, -1) == 0
            out.append(res)
        emu.emu_set_dm(None, C.c_float(0.0))
        return out[0], out[1], out[2].astype(np.int16)

    for suffix, ok in (("", None), ("_m", np.ascontiguousarray((x["gn_mask"] >= 5).astype(np.float32)))):
        plen, tlen, gord = gridnet(ok)
        assert_bits(plen, x["plen" + suffix], "plen" + suffix); assert_bits(tlen, x["tlen" + suffix], "tlen" + suffix); assert_bits(gord, x["gord" + suffix], "gord" + suffix)
    dm, q, dg, tc, cs = (np.ascontiguousarray(x[k]) for k in ("dm", "q", "dg", "tc", "cs"))
    emu.emu_set_dm(dm.ctypes.data, C.c_float(-9999.0))
    assert_bits(_run(emu, True, 12, 0, ang, None, True, 83, **kw), x["dsca"], "dsca")
    assert_bits(_run(emu, True, 12, 0, ang, w, False, 84, **kw), x["dsca_w_nc"], "dsca -wg -nc")
    emu.emu_set_extra(dg.ctypes.data, C.c_float(2.5), None, C.c_float(0.0), None, None)
    assert_bits(_run(emu, True, 16, 0, ang, q, True, 85, **kw), x["ctpt"], "ctpt")
    assert_bits(_run(emu, True, 16, 0, ang, q, False, 86, **kw), x["ctpt_nc"], "ctpt -nc")
    dep, cout = np.empty((ny, nx), np.float32), np.empty((ny, nx), np.float32)
    emu.emu_set_dm(tc.ctypes.data, C.c_float(-9999.0))
    emu.emu_set_extra(None, C.c_float(0.0), None, C.c_float(0.0), dep.ctypes.data, None)
    assert_bits(_run(emu, True, 17, 0, ang, q, True, 87, **kw), x["tla"], "tla"); assert_bits(dep, x["tdep"], "tdep")
    emu.emu_set_extra(None, C.c_float(0.0), cs.ctypes.data, C.c_float(-9999.0), dep.ctypes.data, cout.ctypes.data)
    assert_bits(_run(emu, True, 18, 0, ang, q, False, 88, **kw), x["tla_c"], "tla -cs -nc"); assert_bits(dep, x["tdep_c"], "tdep -cs -nc"); assert_bits(cout, x["ctpt_c"], "ctpt -cs -nc")
    emu.emu_set_dm(None, C.c_float(0.0))


def test_emulated_stencils_on_odd_shapes(emu):
    """The tile-ring kernels (k_fill_init, k_deps_d8) and k_deps_dinf on grids narrower / shorter than a tile, one cell wide, a few columns
    past a tile edge: the rim logic of the staged tiles (columns off the grid, partial words, halo rows that do not exist)."""
    from oracle import port
    rng = np.random.default_rng(11)
    MISS = -3.4028234663852886e38
    for ny, nx in ((1, 1), (1, 7), (5, 3), (2, 260), (33, 129), (65, 132), (7, 127), (130, 5)):
        p = rng.integers(1, 9, (ny, nx)).astype(np.int16)
        p[rng.random((ny, nx)) < 0.1] = -32768
        p[rng.random((ny, nx)) < 0.05] = rng.choice(np.array([0, 9, -3, 100], np.int16))
        a = (rng.random((ny, nx)) * 6.4).astype(np.float32)
        k = rng.random((ny, nx)) < 0.4
        a[k] = (np.float32(np.pi / 4) * rng.integers(0, 9, (ny, nx)).astype(np.float32))[k]
        a[rng.random((ny, nx)) < 0.1] = np.float32(MISS)
        node = np.empty((ny, nx), np.uint16); cnt = np.empty((ny, nx), np.uint8); area = np.empty((ny, nx), np.float32)
        rn = np.empty((ny, nx), np.uint16); rc = np.empty((ny, nx), np.uint8)
        d = np.ascontiguousarray(p)
        assert emu.emu_deps_d8(d.ctypes.data, node.ctypes.data, cnt.ctypes.data, area.ctypes.data, nx, ny, -32768) == 0
        assert emu.emu_ref_deps(0, d.ctypes.data, rn.ctypes.data, rc.ctypes.data, nx, ny, -32768.0, 30.0, 30.0) == 0
        assert np.array_equal(node, rn) and np.array_equal(cnt, rc) and np.all(area == -1.0), f"k_deps_d8 on {ny} x {nx}"
        d = np.ascontiguousarray(a)
        assert emu.emu_deps_dinf(d.ctypes.data, node.ctypes.data, cnt.ctypes.data, area.ctypes.data, nx, ny, MISS, 10.0, 25.0) == 0
        assert emu.emu_ref_deps(1, d.ctypes.data, rn.ctypes.data, rc.ctypes.data, nx, ny, MISS, 10.0, 25.0) == 0
        assert np.array_equal(node, rn) and np.array_equal(cnt, rc), f"k_deps_dinf on {ny} x {nx}"
        dem = np.ascontiguousarray(synth.gen_dem(max(ny, 4), max(nx, 4), seed=ny * 31 + nx, hurst=0.7, tilt=0.3)[:ny, :nx])
        dem[rng.random((ny, nx)) < 0.08] = -9999.0
        mask = np.ascontiguousarray((rng.random((ny, nx)) < 0.05).astype(np.int16))
        for four in (0, 1):
            out = np.empty((ny, nx), np.float32)
            assert emu.emu_fill(dem.ctypes.data, out.ctypes.data, mask.ctypes.data, nx, ny, -9999.0, four, 5) == 0
            assert_bits(out, port.pitremove(dem, four_way=bool(four), depmask=mask), f"fel on {ny} x {nx}, 4-way {four}")
