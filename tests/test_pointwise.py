"""The point-wise kernels (k_threshold, k_twi, k_slopearea, k_slopearearatio, k_lengtharea with its host resolve; pointwise.cu) on
the CPU emulation (tests/emu) against the restatements of tests/pointwise_cases.py, cell by cell: on every pair of special values,
values next to four nodata values and inputs where libm is not correctly rounded; at every exponent branch of the power; on
lengtharea cells whose decision depends on the last bit of powf; on widths that end inside a float4, at and past one column block
of 1024 cells.  And the premise of lengtharea's resolve: libm's powf is faithful on every positive float at the tested exponents."""
import functools

import numpy as np
import pytest

import libm_oracle as L
import pointwise_cases as P
from test_stream_definition import build_pd_emu
from util import assert_bits

F = np.float32


@pytest.fixture(scope="module")
def emu():
    return build_pd_emu()


def _twi(lib, slp, sca, snd=-1.0, and_=-1.0):
    out = np.empty(slp.shape, np.float32)
    assert lib.emu_slp_sca(0, slp.ctypes.data, sca.ctypes.data, out.ctypes.data, slp.shape[1], slp.shape[0], snd, and_) == 0
    return out


def _sa(lib, slp, sca, m, n):
    out = np.empty(slp.shape, np.float32)
    assert lib.emu_slp_sca(1, slp.ctypes.data, sca.ctypes.data, out.ctypes.data, slp.shape[1], slp.shape[0], m, n) == 0
    return out


def _sar(lib, slp, sca, nd=-1.0):
    out = np.empty(slp.shape, np.float32)
    assert lib.emu_slp_sca(2, slp.ctypes.data, sca.ctypes.data, out.ctypes.data, slp.shape[1], slp.shape[0], nd, 0.0) == 0
    return out


def _thr(lib, ssa, thresh, mask=None, nd=-1.0):
    out = np.empty(ssa.shape, np.int16)
    assert lib.emu_threshold(ssa.ctypes.data, None if mask is None else mask.ctypes.data, out.ctypes.data, ssa.shape[1], ssa.shape[0], thresh, nd) == 0
    return out


def _la(lib, plen, ad8, m, y):
    out = np.empty(plen.shape, np.int16)
    npend = np.zeros(1, np.uint32)
    assert lib.emu_lengtharea(plen.ctypes.data, ad8.ctypes.data, out.ctypes.data, plen.shape[1], plen.shape[0], m, y, npend.ctypes.data) == 0
    return out, int(npend[0])


def _pair_grid(nd, width=1025, seed=0):
    a, b = P.pairs(P.value_set(nd, seed=seed, nrandom=40))
    return P.on_shape((a, b), (-(-len(a) // width), width))


@pytest.mark.parametrize("nd", P.NODATAS)
def test_emulated_twi_and_slopearearatio_on_value_pairs(emu, nd):
    slp, sca = _pair_grid(nd)
    for snd, and_ in ((nd, nd), (nd, -1.0), (-1.0, nd)):
        got = _twi(emu, slp, sca, snd, and_)
        P.assert_log_pow_contract(got, P.twi(slp, sca, snd, and_), P.twi(slp, sca, snd, and_, libm=False), f"twi nodata {snd} {and_}")
    P.assert_float_bits(_sar(emu, slp, sca, nd), P.slopearearatio(slp, sca, nd), f"slopearearatio nodata {nd}")


@pytest.mark.parametrize("m", P.EXPONENTS)
def test_emulated_slopearea_on_value_pairs(emu, m):
    slp, sca = _pair_grid(-1.0, seed=1)
    for n in (1.0, m, 0.5 if m != 0.5 else 1.3):
        got = _sa(emu, slp, sca, m, n)
        P.assert_log_pow_contract(got, P.slopearea(slp, sca, m, n), P.slopearea(slp, sca, m, n, libm=False), f"slopearea m={m} n={n}")


def test_emulated_slopearea_keeps_the_sign_of_a_negative_zero_power_like_powf(emu):
    """powf(-0, 0.5) is +0; a square root would give -0 (which assert_allclose cannot see)"""
    slp = np.array([[-0.0, 0.0, -0.0, 4.0]], np.float32)
    sca = np.array([[1.0, 1.0, 3.0, -0.0]], np.float32)
    for m, n in ((0.5, 1.0), (0.5, 0.5), (2.0, 0.5), (3.0, 1.0)):
        got = _sa(emu, slp, sca, m, n)
        want = P.slopearea(slp, sca, m, n)
        assert_bits(P.bits(got), P.bits(want), f"slopearea m={m} n={n} on signed zeros")


@pytest.mark.parametrize("nd", P.NODATAS)
def test_emulated_threshold(emu, nd):
    """thresholds equal to a cell value and one ulp either side; masks -0, NaN, -tiny, +tiny, and the values next to nodata"""
    vals = P.value_set(nd, seed=2, nrandom=40)
    masks = np.array([-0.0, np.nan, -1e-45, 1e-45, 0.0, -1.0, 2.0, np.inf, -np.inf], np.float32)
    ssa, mask = P.pairs(np.concatenate([vals, masks]))
    ssa, mask = P.on_shape((ssa, mask), (-(-len(ssa) // 1025), 1025))
    for t in (F(656.0), F(nd), F(0.0), F(-0.0), F(1.0), F(2.0 ** -126), F(np.inf), F(-np.inf), F(3.4e38)):
        for th in P._steps(t, 1):
            assert_bits(_thr(emu, ssa, th, nd=nd), P.threshold(ssa, th, nodata=nd), f"threshold {th} nodata {nd}")
            assert_bits(_thr(emu, ssa, th, mask, nd), P.threshold(ssa, th, mask, nd), f"threshold {th} -mask nodata {nd}")


def _la_values():
    """plen values: special ones (negative: nodata) and random; ad8 values: around the products, negative, extremes"""
    plen = np.concatenate([P.special_values(), np.array([1e-3, 0.25, 10.0, 123.456, 2179.18677, 64.015625, 1e4, 3e4], np.float32)])
    ad8 = np.array([0, 1, -1, 2, 7, 656, 4098, 100, 2 ** 24 + 1, 2 ** 31 - 1, -2 ** 31, 30], np.int32)
    p, a = np.meshgrid(plen, ad8.astype(np.float64), indexing="ij")
    return p.ravel().astype(np.float32), a.ravel().astype(np.int32)


@pytest.mark.parametrize("y", P.EXPONENTS)
def test_emulated_lengtharea_on_special_values(emu, y):
    p, a = _la_values()
    plen, ad8 = P.on_shape((p, a), (-(-len(p) // 1025), 1025))
    for m in P.COEFFS:
        got, _ = _la(emu, plen, ad8, m, y)
        assert_bits(got, P.lengtharea(plen, ad8, m, y), f"lengtharea M={m} y={y}")


@functools.lru_cache(maxsize=None)
def _flips(m, y):
    return L.lengtharea_flips(m, y, 0x3F800000, 0x4F000000 - 0x3F800000, 1 << 20)


def flip_cells(m, y, count):
    """lengtharea cells whose decision flips with the last bit of the power: the two cells the tool is known to flip on, and up to
    `count` (plen, ad8) pairs from plen in [1, 2^31) where libm's powf and the correctly rounded power decide differently"""
    plen, ad8, total = _flips(m, y)
    assert total > 0, (m, y)
    pick = np.linspace(0, len(plen) - 1, min(count, len(plen))).astype(np.int64)
    known = (np.array([2179.18677, 64.015625], np.float32), np.array([656, 4098], np.int32))
    return np.concatenate([known[0], plen[pick]]), np.concatenate([known[1], ad8[pick]]), total


@pytest.mark.parametrize("m,y", [(0.03, 1.3), (1.0, 2.0), (0.03, 2.0), (0.5, 0.5)])
def test_emulated_lengtharea_on_cells_that_flip_with_the_last_bit_of_the_power(emu, m, y):
    """The kernel decides them through the host resolve with libm's powf: every constructed cell matches the reference, and the
    two known cells are what the reference writes (plen = 0x1.1065fap+11, ad8 = 656 at the defaults -> 0; plen = 0x1.001p+6,
    ad8 = 4098 at M = 1, y = 2 -> 0)."""
    plen, ad8, total = flip_cells(m, y, 400)
    want = P.lengtharea(plen[None], ad8[None], m, y)
    got, npend = _la(emu, np.ascontiguousarray(plen[None]), np.ascontiguousarray(ad8[None]), m, y)
    assert_bits(got, want, f"lengtharea flip cells M={m} y={y} ({total} in [1, 2^31))")
    assert npend >= len(plen) - 2, (npend, len(plen))
    if (m, y) == (0.03, 1.3):
        assert want[0, 0] == 0
    if (m, y) == (1.0, 2.0):
        assert want[0, 1] == 0


@pytest.mark.parametrize("shape", P.SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_emulated_pointwise_kernels_on_edge_shapes(emu, shape):
    """widths that end inside a float4, one column block (1024 cells) and more; the values cycled with an offset per shape"""
    vals = P.value_set(-9999.0, seed=3, nrandom=40)
    a, b = P.pairs(vals)
    off = shape[0] * 7919 + shape[1] * 104729
    slp, sca = P.on_shape((a, b), shape, off)
    P.assert_log_pow_contract(_twi(emu, slp, sca, -9999.0, -9999.0), P.twi(slp, sca, -9999.0, -9999.0), P.twi(slp, sca, -9999.0, -9999.0, libm=False), f"twi {shape}")
    P.assert_log_pow_contract(_sa(emu, slp, sca, 1.3, 0.5), P.slopearea(slp, sca, 1.3, 0.5), P.slopearea(slp, sca, 1.3, 0.5, libm=False), f"slopearea {shape}")
    P.assert_float_bits(_sar(emu, slp, sca, -9999.0), P.slopearearatio(slp, sca, -9999.0), f"slopearearatio {shape}")
    assert_bits(_thr(emu, slp, F(sca.flat[0]), sca, -9999.0), P.threshold(slp, F(sca.flat[0]), sca, -9999.0), f"threshold {shape}")
    fp, fa, _ = flip_cells(0.03, 1.3, 3000)
    plen, ad8 = P.on_shape((fp, fa), shape, off)
    assert_bits(_la(emu, plen, ad8, 0.03, 1.3)[0], P.lengtharea(plen, ad8, 0.03, 1.3), f"lengtharea {shape}")


def test_the_restatements_agree_with_the_python_ones():
    """the C helper's lengtharea and slopearea against the numpy / frompyfunc restatements the reference tests replay with"""
    import reference
    import stream_restate
    rng = np.random.default_rng(4)
    plen = (rng.random((7, 300)) * 3000 - 100).astype(np.float32)
    a = (rng.random((7, 300)) * 3000).astype(np.float32)
    for m, y in ((0.03, 1.3), (1.0, 2.0), (0.5, 0.5)):
        assert_bits(P.lengtharea(plen, stream_restate.ad8_int32(a), m, y), stream_restate.lengtharea(plen, a, m, y), f"lengtharea {m} {y}")
    slp, sca = np.abs(plen) / 1000, a
    assert_bits(P.slopearea(slp, sca, 0.5, 1.75), reference._slopearea(slp, sca, 0.5, 1.75), "slopearea")
    assert_bits(P.twi(slp, sca), reference._twi(slp, sca), "twi")


@pytest.mark.parametrize("e", [2.0, 0.5, 1.3, 1.75, 3.0, -1.0])
def test_libm_powf_is_faithful_on_every_positive_float(e):
    """lengtharea's resolve assumes the reference's powf lies within one float step of the kernel's power: true when both are
    faithful (one of the two floats around the exact power).  Checked for libm on all 2^31 non-negative finite floats at every
    exponent the tests use (0 and 1 are exact)."""
    n, bad = L.powf_unfaithful(e)
    assert n == 0, (e, n, [float(x) for x in bad.view(np.float32)])
