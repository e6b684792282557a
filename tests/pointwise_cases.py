"""Inputs, restatements and the cell-by-cell contract of the point-wise tools (threshold, twi, slopearea, slopearearatio,
lengtharea; taudem_b200/csrc/pointwise.cu), shared by the emulated kernel tests (tests/test_pointwise.py) and the GPU tests
(tests/test_gpu_pointwise.py).

The restatements follow the reference's loops (src/Threshold.cpp, TWI.cpp, SlopeArea.cpp, SlopeAreaRatio.cpp, LengthArea.cpp) in
float32, with linearpart's nodata test |v - nodata| < 1e-5 in float.  Where the reference calls logf / powf there are two of them:
`libm=True` calls the host's libm like the reference does, `libm=False` the correctly rounded function (tests/libm_oracle.c).
threshold, slopearearatio and lengtharea are held to the reference's bits.  twi and slopearea compute correctly rounded logarithms
and powers: they must equal the correctly rounded restatement on every cell, and therefore differ from the reference exactly
where libm is not correctly rounded (assert_log_pow_contract)."""
import functools

import numpy as np

import libm_oracle as L

F = np.float32
MINEPS = F(1e-5)
NODATAS = (-1.0, -9999.0, -3.4e38, 7.25)                     # the tools' nodata values worth a test: the default, common tags, a positive one
EXPONENTS = (0.0, 1.0, 2.0, 0.5, 1.3, 1.75, 3.0, -1.0)        # every branch of pow_float
COEFFS = (0.03, 1.0, 0.0, -0.5)                               # lengtharea's M
SHAPES = [(h, w) for h in (1, 2) for w in (1, 3, 4, 5, 1023, 1024, 1025, 4100)]


def bits(a):
    """the bit patterns, every NaN as one pattern (the device writes its canonical NaN, x86 the negative default NaN)"""
    a = np.ascontiguousarray(a, np.float32)
    return np.where(np.isnan(a), np.uint32(0x7FC00000), a.view(np.uint32))


def fbits(u):
    return np.asarray(u, np.uint32).view(np.float32)


def _steps(v, k):
    """v and its float neighbours up to k steps on either side"""
    v = F(v)
    out = [v]
    lo = hi = v
    for _ in range(k):
        lo, hi = np.nextafter(lo, F(-np.inf)), np.nextafter(hi, F(np.inf))
        out += [lo, hi]
    return out


def special_values():
    """+-0, the smallest and largest subnormals, 2^-126 +- 1 ulp, 1 +- ulps, FLT_MAX, +-inf, NaN, negative values and a few ordinary
    ones"""
    v = [F(0.0), F(-0.0), fbits(1), fbits(0x007FFFFF), fbits(0x80000001), *_steps(2.0 ** -126, 1), *_steps(1.0, 3), fbits(0x7F7FFFFF),
         fbits(0x7F7FFFFE), F(np.inf), F(-np.inf), F(np.nan), F(-1.0), F(-2.5), F(-1e-30), F(-3.4e38), F(0.5), F(2.0), F(3.0), F(1e-3),
         F(0.0123), F(30.0), F(656.0), F(1e6), F(2.0 ** 24), F(2.0 ** 24 + 2), F(1e19), F(1e30), F(2179.18677), F(64.015625)]
    return np.array(v, np.float32)


def near_nodata(nd):
    """nd +- k ulps and nd +- (1e-5 +- ulps): both sides of linearpart's |v - nd| < 1e-5 in float"""
    v = _steps(nd, 3)
    for s in (1.0, -1.0):
        edge = F(F(nd) + F(s) * MINEPS)
        v += _steps(edge, 3)
        # the first float where |v - nd| < 1e-5 fails, found by walking (the float subtraction rounds)
        w = F(nd)
        d = F(s * np.inf)
        for _ in range(2000):
            w2 = np.nextafter(w, d)
            if not abs(F(w2 - F(nd))) < MINEPS:
                v += [w, w2]
                break
            w = w2
    return np.unique(np.array(v, np.float32).view(np.uint32)).view(np.float32)


@functools.lru_cache(maxsize=None)
def libm_hard_inputs(which, e=0.0, count=64, start=0x3F000000, span=1 << 22):
    """positive floats where the host's logf (which 0) / powf(x, e) (1) is not correctly rounded, found by sweeping span bit patterns
    from start: the inputs on which a kernel that calls libm, or any other not correctly rounded log / power, differs"""
    u = np.arange(start, start + span, dtype=np.uint32)
    x = u.view(np.float32)
    lib = L.logf(x) if which == 0 else L.powf(x, e)
    cr = L.log_cr(x) if which == 0 else L.pow_cr(x, e)
    hard = x[bits(lib) != bits(cr)]
    return hard[:: max(1, len(hard) // count)][:count]


def value_set(nodata=-1.0, seed=0, nrandom=200):
    """one list of float values: the special values, the values next to nodata, random floats of every magnitude and sign, and
    inputs on which libm's logf and powf at the tested exponents are not correctly rounded"""
    rng = np.random.default_rng(seed)
    rnd = rng.integers(0, 0x7F800000, size=nrandom, dtype=np.uint32).view(np.float32)
    rnd = np.where(rng.random(nrandom) < 0.2, -rnd, rnd).astype(np.float32)
    hard = [libm_hard_inputs(0, count=24)] + [libm_hard_inputs(1, e, count=12) for e in (2.0, 0.5, 1.3, 1.75, 3.0, -1.0)]
    return np.concatenate([special_values(), near_nodata(nodata), rnd, *hard]).astype(np.float32)


def pairs(vals):
    """every ordered pair of vals as two flat arrays (a, b)"""
    a, b = np.meshgrid(vals, vals, indexing="ij")
    return a.ravel().astype(np.float32), b.ravel().astype(np.float32)


def on_shape(arrays, shape, offset=0):
    """the flat arrays cycled from offset onto a (ny, nx) grid"""
    n = shape[0] * shape[1]
    idx = (np.arange(n) + offset) % len(arrays[0])
    return [np.ascontiguousarray(a[idx].reshape(shape)) for a in arrays]


# ---------------------------------------------------------------- restatements
def isnd(v, nd):
    with np.errstate(all="ignore"):
        return np.abs((np.asarray(v, np.float32) - F(nd)).astype(np.float32)) < MINEPS


def threshold(ssa, thresh, mask=None, nodata=-1.0):
    ssa = np.asarray(ssa, np.float32)
    with np.errstate(invalid="ignore"):
        ok = (ssa >= F(thresh)) & (True if mask is None else np.asarray(mask, np.float32) >= 0)
    return np.where(isnd(ssa, nodata), np.int16(-32768), ok.astype(np.int16)).astype(np.int16)


def twi(slp, sca, slp_nodata=-1.0, sca_nodata=-1.0, libm=True):
    slp, sca = np.asarray(slp, np.float32), np.asarray(sca, np.float32)
    with np.errstate(all="ignore"):
        ok = ~isnd(sca, sca_nodata) & ~isnd(slp, slp_nodata) & (slp > 0) & (sca > 0)
        q = (sca / slp).astype(np.float32)
    return np.where(ok, L.logf(q) if libm else L.log_cr(q), F(-1.0)).astype(np.float32)


def slopearea(slp, sca, m=2.0, n=1.0, libm=True):
    slp, sca = np.asarray(slp, np.float32), np.asarray(sca, np.float32)
    with np.errstate(all="ignore"):
        ok = (slp >= 0) & (sca >= 0)
        v = L.slopearea_product(slp, sca, m, n) if libm else (L.pow_cr(slp, m) * L.pow_cr(sca, n)).astype(np.float32)
    return np.where(ok, v, F(-1.0)).astype(np.float32)


def slopearearatio(slp, sca, sca_nodata=-1.0):
    slp, sca = np.asarray(slp, np.float32), np.asarray(sca, np.float32)
    with np.errstate(all="ignore"):
        return np.where(isnd(sca, sca_nodata), F(-1.0), (slp / sca).astype(np.float32)).astype(np.float32)


def lengtharea(plen, ad8, m=0.03, y=1.3):
    """ad8 as int32 (the reference's reading of the area)"""
    return L.lengtharea(plen, ad8, m, y)


# ---------------------------------------------------------------- the contract
def assert_float_bits(got, want, what):
    g, w = bits(got), bits(want)
    bad = np.argwhere(g != w)
    assert len(bad) == 0, (f"{what}: {len(bad)} of {g.size} cells differ; first (cell, got, want): "
                           f"{[(tuple(map(int, i)), float(np.asarray(got)[tuple(i)]), float(np.asarray(want)[tuple(i)])) for i in bad[:5]]}")


def assert_log_pow_contract(got, want_libm, want_cr, what):
    """twi / slopearea: every cell is bit-identical to the restatement with correctly rounded logarithms / powers; so a cell differs
    from the reference (libm) exactly where libm is not correctly rounded.  Returns (cells that differ from libm, cells where libm is
    not correctly rounded), equal by construction when the assertion holds."""
    assert np.array_equal(np.asarray(got) == F(-1.0), np.asarray(want_libm) == F(-1.0)), f"{what}: the nodata masks differ"
    assert_float_bits(got, want_cr, what + " (against correctly rounded log / pow)")
    d = bits(got) != bits(want_libm)
    b = bits(want_libm) != bits(want_cr)
    assert np.array_equal(d, b), f"{what}: cells that differ from libm {int(d.sum())}, where libm is not correctly rounded {int(b.sum())}"
    return int(d.sum()), int(b.sum())
