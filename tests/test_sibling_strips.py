"""The five sibling sweep tools on row strips: algebras 1-9 of the sweep (taudem_b200/csrc/sweep_warp.cu) on 2, 3 and 5 strips and on
strips of one to three rows, with the exchange rounds a row-strip caller makes (the decrement counts, the edge rows of the travelling
value, ALG 9's concentration rows; gridnet's mask grid and D8 codes with their halo rows), executed on the CPU emulation of the thread
model (tests/emu) and compared bit for bit with the C restatement (oracle/port).  Flow must really cross the strip boundaries: every
case asserts more than one round and decrements handed over.

The emulation has no CUDA IPC, so the peer mode (deliveries into the neighbour GPU, ALG 9's concentration in the second half of the
peer halo buffer) is not emulated here; tests/test_gpu_sibling_strips.py runs it on GPUs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from util import assert_bits

import sibling_cases
import test_emu

MISS = np.float32(-3.4028234663852886e38)
ND = -9999.0


@pytest.fixture(scope="module")
def emu():
    test_emu._build()                                  # the transformed kernel sources
    so = os.path.join(test_emu.BUILD, "libemu_sibling_strips.so")
    srcs = [os.path.join(test_emu.EMU, f) for f in ("sibling_strips_driver.cpp", "emu.cpp")]
    deps = srcs + [os.path.join(test_emu.EMU, "driver.cpp"), os.path.join(test_emu.BUILD, "sweep_warp_emu.inc"),
                   os.path.join(test_emu.BUILD, "outlets_emu.inc"), os.path.join(test_emu.EMU, "cuda_runtime.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ftls-model=initial-exec", "-ffp-contract=off",
                               "-I", test_emu.EMU, "-I", test_emu.BUILD, "-I", test_emu.CSRC, "-o", so, *srcs])
    lib = C.CDLL(so)
    P = C.c_void_p
    lib.emu_sibling_strips.argtypes = [C.c_int, P, C.c_int, C.c_int, C.c_int, P, P, P, P, P, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                                       P, P, C.c_ulonglong, P, P, P, P]
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data


def layouts(ny):
    """strip heights: 2, 3 and 5 even strips (the last takes the remainder), and strips of one to three rows at both edges and inside"""
    out = []
    for n in (2, 3, 5):
        out.append([ny // n] * (n - 1) + [ny - (n - 1) * (ny // n)])
    mid = ny // 2 - 3
    out.append([1, 2, 3, mid, 1, 2, ny - mid - 9])
    return out


def run(lib, alg, d, rows, v=(None, None, None), dg=None, nd=(ND, ND, ND), csol=1.0, contcheck=True, dxr=None, dyr=None, seed=1):
    """(out0, out1, out2, rounds, handed) of one emulated run on row strips of the given heights"""
    ny, nx = d.shape
    d = np.ascontiguousarray(d)
    dxr = np.ascontiguousarray(np.full(ny, 30.0) if dxr is None else dxr, np.float64)
    dyr = np.ascontiguousarray(np.full(ny, 30.0) if dyr is None else dyr, np.float64)
    vv = [None if a is None else np.ascontiguousarray(a, np.float32) for a in v]
    dgc = None if dg is None else np.ascontiguousarray(dg, np.int16)
    r = np.ascontiguousarray(rows, np.int32)
    o0, o1, o2 = (np.empty((ny, nx), np.float32) for _ in range(3))
    st = np.zeros(2, np.int64)
    rc = lib.emu_sibling_strips(alg, d.ctypes.data, nx, ny, len(rows), r.ctypes.data, _ptr(vv[0]), _ptr(vv[1]), _ptr(vv[2]), _ptr(dgc),
                                nd[0], nd[1], nd[2], csol, int(contcheck), dxr.ctypes.data, dyr.ctypes.data, seed,
                                o0.ctypes.data, o1.ctypes.data, o2.ctypes.data, st.ctypes.data)
    assert rc == 0, rc
    return o0, o1, o2, int(st[0]), int(st[1])


def gord_finish(order, p, ok):
    """k_gord_finish without outlets: a cell the sweep never evaluated is 1 with a direction inside the mask, -1 elsewhere"""
    inside = np.ones(p.shape, bool) if ok is None else ok != 0
    return np.where(order >= 0, order.astype(np.int16), np.where((p != -32768) & inside, 1, -1)).astype(np.int16)


def meander(ny=150, nx=96, pitch=6):
    """D8 codes and D-infinity angles of one channel meandering north and south through the whole grid (columns 2, 2 + pitch, ...),
    so that it crosses every strip boundary many times; every other cell drains east or west into the nearest channel column"""
    p = np.zeros((nx, ny), np.int16)                   # built east-west (rows = columns of the result), then transposed
    rows = list(range(2, nx - 2, pitch))
    path = []
    for i, r in enumerate(rows):
        cols = range(2, ny - 2) if i % 2 == 0 else range(ny - 3, 1, -1)
        path += [(r, c) for c in cols]
        if i + 1 < len(rows):
            path += [(rr, cols[-1]) for rr in range(r + 1, rows[i + 1])]
    on = np.zeros(p.shape, bool)
    for r, c in path:
        on[r, c] = True
    for r in range(p.shape[0]):
        for c in range(p.shape[1]):
            if not on[r, c]:
                near = min(rows, key=lambda q: (abs(q - r), q))
                p[r, c] = 7 if near > r else 3 if near < r else 1 if c < 2 else 5
    for (r, c), (r2, c2) in zip(path, path[1:]):
        p[r, c] = {(0, 1): 1, (0, -1): 5, (1, 0): 7}[(r2 - r, c2 - c)]
    r_out, c_out = path[-1]
    west = p[path[-2]] == 5
    p[r_out, :c_out + 1] = 5 if west else p[r_out, :c_out + 1]
    p[r_out, c_out:] = p[r_out, c_out:] if west else 1
    p = np.ascontiguousarray(np.choose(p.T, [0, 7, 0, 5, 0, 3, 0, 1]).astype(np.int16))    # transposed: east <-> south, north <-> west
    ang = np.choose(p, [0, 0, 0, np.pi / 2, 0, np.pi, 0, 1.5 * np.pi]).astype(np.float32)
    return p, ang


def values(shape, seed, lo=0.0, hi=3.0):
    """a value grid with nodata, zero and negative cells"""
    rng = np.random.default_rng(seed)
    v = rng.uniform(lo, hi, shape).astype(np.float32)
    v[rng.random(shape) < 0.01] = ND
    v[rng.random(shape) < 0.01] = 0.0
    v[rng.random(shape) < 0.01] = -rng.uniform(0.1, 1.0)
    return v


@pytest.fixture(scope="module")
def terrains(tmp_path_factory):
    """(name, p, ang) of the sibling_cases terrains (cropped to keep the emulation short) and of the meandering channel"""
    import port
    out = []
    for i, case in enumerate((sibling_cases.flowpathextremeup, sibling_cases.gridnet, sibling_cases.dinfdecayaccum)):
        x, _ = case(tmp_path_factory.mktemp(f"case{i}"))
        if "p" in x:
            p = x["p"][:120, :150]
            ang = port.dinfflowdir(port.pitremove(x["fel"][:120, :150]))[0] if "fel" in x else None
        else:
            ang = x["ang"][:120, :150]
            p = None
        out.append((case.__name__, p, ang))
    mp, mang = meander()
    out.append(("meander", mp, mang))
    return out


def _crossed(rounds, handed, what):
    assert rounds > 1 and handed > 0, f"{what}: {rounds} rounds, {handed} decrements handed over"


def test_extreme_up_on_strips(emu, terrains):
    import port
    for name, p, _ in terrains:
        if p is None:
            continue
        sa = values(p.shape, 3, -1.0, 5.0)
        for li, rows in enumerate(layouts(p.shape[0])):
            for usemax, cc in ((True, True), (False, False)):
                out, _, _, rounds, handed = run(emu, 1 if usemax else 2, p, rows, (sa, None, None), contcheck=cc, seed=li)
                what = f"ssa {name} {rows} max={usemax} cc={cc}"
                assert_bits(out, port.d8flowpathextremeup(p, sa, usemax=usemax, contcheck=cc), what)
                _crossed(rounds, handed, what)


def test_gridnet_on_strips(emu, terrains):
    import port
    for name, p, _ in terrains:
        if p is None:
            continue
        ny = p.shape[0]
        dxr, dyr = np.full(ny, 12.5), np.full(ny, 40.0)
        rng = np.random.default_rng(7)
        mask = rng.integers(0, 40, p.shape).astype(np.int32)
        for masked in (False, True):
            ok = (mask >= 20).astype(np.float32) if masked else None
            ref = port.gridnet(p, mask=mask if masked else None, thresh=20, dx=12.5, dy=40.0)
            for li, rows in enumerate(layouts(ny)):
                outs = []
                for alg in (4, 5, 6):
                    o, _, _, rounds, handed = run(emu, alg, p, rows, (ok, None, None), dxr=dxr, dyr=dyr, seed=10 * alg + li)
                    _crossed(rounds, handed, f"gridnet {alg} {name} {rows}")
                    outs.append(o)
                what = f"gridnet {name} {rows} mask={masked}"
                assert_bits(outs[0], ref[0], "plen " + what)
                assert_bits(outs[1], ref[1], "tlen " + what)
                assert_bits(gord_finish(outs[2], p, ok), ref[2], "gord " + what)


def _cell_sizes(ny, kind):
    if kind == "square":
        return np.full(ny, 30.0), np.full(ny, 30.0)
    if kind == "oblong":
        return np.full(ny, 12.5), np.full(ny, 40.0)
    lat = np.deg2rad(40.0 + 0.01 * np.arange(ny))       # geographic: the east-west size shrinks row by row
    return 111320.0 * 0.0083 * np.cos(lat), np.full(ny, 111320.0 * 0.0083)


def _dinf_terrains(terrains):
    return [(name, ang) for name, _, ang in terrains if ang is not None]


@pytest.mark.parametrize("kind", ["square", "oblong", "geographic"])
def test_decay_on_strips(emu, terrains, kind):
    import port
    for name, ang in _dinf_terrains(terrains):
        ny = ang.shape[0]
        dxr, dyr = _cell_sizes(ny, kind)
        dm = values(ang.shape, 5, 0.2, 1.0)
        w = values(ang.shape, 6, -1.0, 2.0)
        for li, rows in enumerate(layouts(ny)):
            for weights, cc in ((None, True), (w, False)):
                out, _, _, rounds, handed = run(emu, 3, ang, rows, (dm, weights, None), contcheck=cc, dxr=dxr, dyr=dyr, seed=li)
                what = f"dsca {name} {kind} {rows} w={weights is not None} cc={cc}"
                assert_bits(out, port.dinfdecayaccum(ang, dm, weights=weights, contcheck=cc, dxc=dxr, dyc=dyr), what)
                _crossed(rounds, handed, what)


@pytest.mark.parametrize("kind", ["square", "oblong", "geographic"])
def test_conc_lim_on_strips(emu, terrains, kind):
    import port
    for name, ang in _dinf_terrains(terrains):
        ny = ang.shape[0]
        dxr, dyr = _cell_sizes(ny, kind)
        q, dm, dg, _, _ = sibling_cases.sibling_inputs(ang.shape, 21)
        q[::17, ::13] = -0.5                              # negative discharge: no concentration
        for li, rows in enumerate(layouts(ny)):
            for cc in (True, False):
                out, _, _, rounds, handed = run(emu, 7, ang, rows, (dm, q, None), dg=dg, csol=2.5, contcheck=cc, dxr=dxr, dyr=dyr, seed=li)
                what = f"ctpt {name} {kind} {rows} cc={cc}"
                assert_bits(out, port.dinfconclimaccum(ang, dm, q, dg, csol=2.5, contcheck=cc, dxc=dxr, dyc=dyr), what)
                _crossed(rounds, handed, what)


@pytest.mark.parametrize("kind", ["square", "oblong", "geographic"])
def test_trans_lim_on_strips(emu, terrains, kind):
    import port
    for name, ang in _dinf_terrains(terrains):
        ny = ang.shape[0]
        dxr, dyr = _cell_sizes(ny, kind)
        tsup, _, _, tc, cs = sibling_cases.sibling_inputs(ang.shape, 23)
        tsup[::19, ::7] = -0.25
        tc[::11, ::23] = 0.0
        for li, rows in enumerate(layouts(ny)):
            for usec in (False, True):
                for cc in (True, False):
                    tla, dep, cout, rounds, handed = run(emu, 9 if usec else 8, ang, rows, (tsup, tc, cs if usec else None), contcheck=cc, dxr=dxr,
                                                         dyr=dyr, seed=li)
                    rt, rd, rc = port.dinftranslimaccum(ang, tsup, tc, cs=cs if usec else None, contcheck=cc, dxc=dxr, dyc=dyr)
                    what = f"{name} {kind} {rows} cs={usec} cc={cc}"
                    assert_bits(tla, rt, "tla " + what)
                    assert_bits(dep, rd, "tdep " + what)
                    if usec:
                        assert_bits(cout, rc, "ctpt " + what)
                    _crossed(rounds, handed, what)
