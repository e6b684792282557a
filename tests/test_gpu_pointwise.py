"""The point-wise tools on the GPU (threshold, twi, slopearea, slopearearatio, lengtharea; pointwise.cu) against the restatements of
tests/pointwise_cases.py, cell by cell: the grids of the emulated tests at the host-grid level and through the executables on files
whose nodata tags are not -1; twi and slopearea on every positive finite float, where the cells that differ from the host's libm
must be exactly the inputs on which libm is not correctly rounded (and the GPU correctly rounded on all of them); and lengtharea
on a few thousand cells whose decision flips with the last bit of powf."""
import os
import subprocess
import time

import numpy as np
import pytest

import libm_oracle as L
import pointwise_cases as P
import taudem_b200 as td
from util import assert_bits

pytestmark = pytest.mark.gpu
F = np.float32
BIN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "taudem_b200", "bin")


def _pair_grid(nd, width=1025, seed=0):
    a, b = P.pairs(P.value_set(nd, seed=seed, nrandom=200))
    return P.on_shape((a, b), (-(-len(a) // width), width))


@pytest.mark.parametrize("nd", P.NODATAS)
def test_twi_slopearearatio_and_threshold_grids_on_value_pairs(nd):
    slp, sca = _pair_grid(nd)
    for snd, and_ in ((nd, nd), (nd, -1.0), (-1.0, nd)):
        P.assert_log_pow_contract(td.twi_grid(slp, sca, snd, and_), P.twi(slp, sca, snd, and_), P.twi(slp, sca, snd, and_, libm=False),
                                  f"twi nodata {snd} {and_}")
    P.assert_float_bits(td.slopearearatio_grid(slp, sca, nd), P.slopearearatio(slp, sca, nd), f"slopearearatio nodata {nd}")
    mask = sca.copy()
    mask.flat[::7] = F(-0.0); mask.flat[1::7] = F(np.nan); mask.flat[2::7] = P.fbits(0x80000001)
    for t in (F(656.0), F(nd), F(0.0), F(1.0), F(np.inf), F(slp.flat[12345])):
        for th in P._steps(t, 1):
            assert_bits(td.threshold_grid(slp, th, nodata=nd), P.threshold(slp, th, nodata=nd), f"threshold {th} nodata {nd}")
            assert_bits(td.threshold_grid(slp, th, mask=mask, nodata=nd), P.threshold(slp, th, mask, nd), f"threshold {th} -mask nodata {nd}")


@pytest.mark.parametrize("m", P.EXPONENTS)
def test_slopearea_grid_on_value_pairs(m):
    slp, sca = _pair_grid(-1.0, seed=1)
    for n in (1.0, m, 0.5 if m != 0.5 else 1.3):
        P.assert_log_pow_contract(td.slopearea_grid(slp, sca, m, n), P.slopearea(slp, sca, m, n), P.slopearea(slp, sca, m, n, libm=False),
                                  f"slopearea m={m} n={n}")
    z = np.array([[-0.0, 0.0, -0.0, 4.0]], np.float32), np.array([[1.0, 1.0, 3.0, -0.0]], np.float32)
    assert_bits(P.bits(td.slopearea_grid(*z, m, 1.0)), P.bits(P.slopearea(*z, m, 1.0)), f"slopearea m={m} on signed zeros")


def _la_cells():
    import test_pointwise as T
    p, a = T._la_values()
    return p, a


@pytest.mark.parametrize("y", P.EXPONENTS)
def test_lengtharea_grid_on_special_values(y):
    p, a = _la_cells()
    plen, ad8 = P.on_shape((p, a), (-(-len(p) // 1025), 1025))
    for m in P.COEFFS:
        assert_bits(td.lengtharea_grid(plen, ad8, m=m, y=y), P.lengtharea(plen, ad8, m, y), f"lengtharea M={m} y={y}")


@pytest.mark.parametrize("m,y", [(0.03, 1.3), (1.0, 2.0), (0.03, 2.0), (0.5, 0.5)])
def test_lengtharea_grid_on_cells_that_flip_with_the_last_bit_of_the_power(m, y):
    import test_pointwise as T
    plen, ad8, total = T.flip_cells(m, y, 4000)
    for shape in ((1, len(plen)), (2, (len(plen) + 1) // 2), (-(-len(plen) // 1025), 1025)):
        pl, a = P.on_shape((plen, ad8), shape, 3)
        assert_bits(td.lengtharea_grid(pl, a, m=m, y=y), P.lengtharea(pl, a, m, y), f"lengtharea flip cells M={m} y={y} {shape} ({total} in [1, 2^31))")


@pytest.mark.parametrize("shape", P.SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_pointwise_grids_on_edge_shapes(shape):
    import test_pointwise as T
    a, b = P.pairs(P.value_set(-9999.0, seed=3, nrandom=40))
    off = shape[0] * 7919 + shape[1] * 104729
    slp, sca = P.on_shape((a, b), shape, off)
    P.assert_log_pow_contract(td.twi_grid(slp, sca, -9999.0, -9999.0), P.twi(slp, sca, -9999.0, -9999.0), P.twi(slp, sca, -9999.0, -9999.0, libm=False), f"twi {shape}")
    P.assert_log_pow_contract(td.slopearea_grid(slp, sca, 1.3, 0.5), P.slopearea(slp, sca, 1.3, 0.5), P.slopearea(slp, sca, 1.3, 0.5, libm=False), f"slopearea {shape}")
    P.assert_float_bits(td.slopearearatio_grid(slp, sca, -9999.0), P.slopearearatio(slp, sca, -9999.0), f"slopearearatio {shape}")
    assert_bits(td.threshold_grid(slp, F(sca.flat[0]), mask=sca, nodata=-9999.0), P.threshold(slp, F(sca.flat[0]), sca, -9999.0), f"threshold {shape}")
    fp, fa, _ = T.flip_cells(0.03, 1.3, 3000)
    plen, ad8 = P.on_shape((fp, fa), shape, off)
    assert_bits(td.lengtharea_grid(plen, ad8), P.lengtharea(plen, ad8, 0.03, 1.3), f"lengtharea {shape}")


def _exe(tool, *args):
    r = subprocess.run([os.path.join(BIN, tool), *map(str, args)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "rror" not in r.stdout, r.stdout
    return r.stdout


@pytest.mark.parametrize("nd", [-9999.0, -3.4e38, 7.25])
def test_pointwise_executables_on_files_with_other_nodata_tags(tmp_path, nd):
    """the five executables read each raster's own nodata tag: twi and slopearearatio test it (|v - nodata| < 1e-5), threshold the
    area's; values next to the tag on both sides of 1e-5"""
    import test_pointwise as T
    slp, sca = _pair_grid(nd, seed=5)
    d = lambda n: str(tmp_path / n)
    td.write_raster(d("slp.tif"), slp, nd)
    td.write_raster(d("sca.tif"), sca, nd)
    _exe("twi", "-slp", d("slp.tif"), "-sca", d("sca.tif"), "-twi", d("twi.tif"))
    P.assert_log_pow_contract(td.read_raster(d("twi.tif")), P.twi(slp, sca, nd, nd), P.twi(slp, sca, nd, nd, libm=False), f"twi (files) {nd}")
    _exe("slopearea", "-slp", d("slp.tif"), "-sca", d("sca.tif"), "-sa", d("sa.tif"), "-par", 0.5, 1.3)
    P.assert_log_pow_contract(td.read_raster(d("sa.tif")), P.slopearea(slp, sca, 0.5, 1.3), P.slopearea(slp, sca, 0.5, 1.3, libm=False), f"slopearea (files) {nd}")
    _exe("slopearearatio", "-slp", d("slp.tif"), "-sca", d("sca.tif"), "-sar", d("sar.tif"))
    P.assert_float_bits(td.read_raster(d("sar.tif")), P.slopearearatio(slp, sca, nd), f"slopearearatio (files) {nd}")
    th = F(sca.flat[777])
    _exe("threshold", "-ssa", d("sca.tif"), "-src", d("src.tif"), "-thresh", repr(float(th)), "-mask", d("slp.tif"))
    assert_bits(td.read_raster(d("src.tif"), np.int16), P.threshold(sca, th, slp, nd), f"threshold (files) {nd}")
    plen, ad8, _ = T.flip_cells(0.03, 1.3, 3000)
    plen, ad8 = P.on_shape((plen, ad8), (3, 1001), 0)
    plen.flat[::97] = F(-1.0)                                                 # nodata cells of the length
    td.write_raster(d("plen.tif"), plen, nd)
    td.write_raster(d("ad8.tif"), ad8.astype(np.float32), nd)
    _exe("lengtharea", "-plen", d("plen.tif"), "-ad8", d("ad8.tif"), "-ss", d("ss.tif"))
    assert_bits(td.read_raster(d("ss.tif"), np.int16), P.lengtharea(plen, ad8, 0.03, 1.3), f"lengtharea (files) {nd}")


# ---------------------------------------------------------------- every positive finite float
CHUNK = 1 << 26
NCOL = 1 << 13


def _sweep(which, e, u_first):
    """which 0: twi with slp = 1 and sca = x; 1: slopearea with sca = 1 (n = 1) and slp = x, m = e; x = every finite float from
    the bit pattern u_first on"""
    one = np.ones((CHUNK // NCOL, NCOL), np.float32)
    tot = np.zeros(4, np.int64)
    bad = []
    t0 = time.time()
    for u0 in range(u_first, L.FLT_POS_FINITE, CHUNK):
        n = min(CHUNK, L.FLT_POS_FINITE - u0)
        x = np.arange(u0, u0 + CHUNK, dtype=np.uint32).view(np.float32).reshape(one.shape)
        got = td.twi_grid(one, x) if which == 0 else td.slopearea_grid(x, one, e, 1.0)
        cnt, b = L.sweep(which, e, u0, got.ravel()[:n])
        tot += cnt
        bad += list(b)
    return tuple(int(c) for c in tot), np.array(bad, np.uint32), time.time() - t0


@pytest.mark.parametrize("which,e", [(0, 0.0), (1, 2.0), (1, 0.5), (1, 1.3)], ids=["twi", "slopearea-m2", "slopearea-m0.5", "slopearea-m1.3"])
def test_every_positive_float(which, e):
    """twi = ln(sca) on every positive finite sca (slp = 1); slopearea = slp^m on every non-negative finite slp (sca = 1): the cells
    that differ from the host's logf / powf are exactly the inputs where libm is not correctly rounded, and the GPU is correctly
    rounded on every one of the 2^31 - 2^23 - 1 inputs"""
    (ndiff, nlibm, nwrong, nsym), bad, secs = _sweep(which, e, 1 if which == 0 else 0)
    print(f"\n{'twi' if which == 0 else f'slopearea m={e}'}: cells that differ from libm {ndiff}, inputs where libm is not correctly "
          f"rounded {nlibm}, GPU not correctly rounded {nwrong} ({secs:.1f} s)")
    assert nwrong == 0 and nsym == 0 and ndiff == nlibm, (ndiff, nlibm, nwrong, nsym, [float(v) for v in bad.view(np.float32)[:16]])
