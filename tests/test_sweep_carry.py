"""The carry of the contributing-area sweep (taudem_b200/csrc/sweep_warp.cu): a worker whose visit makes a cell of another tile
ready through its last crossing claims that tile and visits it next, without the ticket queue.  Values do not depend on the
schedule, so every result must equal the C restatement with the carry on and off (TAUDEM_B200_EXP bit 16); the statistics
counters (TAUDEM_B200_TIMING) show that a river winding through many tiles is carried from tile to tile."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from taudem_b200 import synth
from util import assert_bits

import test_emu

EXP_NO_CARRY = 16
MISS = -3.4028234663852886e38
TS = 32                       # tile edge of the sweep


@pytest.fixture(scope="module")
def emu():
    test_emu._build()                                  # the transformed kernel sources and the test library
    so = os.path.join(test_emu.BUILD, "libemu_carry.so")
    srcs = [os.path.join(test_emu.EMU, f) for f in ("carry_driver.cpp", "emu.cpp")]
    deps = srcs + [os.path.join(test_emu.EMU, "driver.cpp"), os.path.join(test_emu.BUILD, "sweep_warp_emu.inc"),
                   os.path.join(test_emu.BUILD, "outlets_emu.inc"), os.path.join(test_emu.EMU, "cuda_runtime.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-ftls-model=initial-exec", "-ffp-contract=off",
                               "-I", test_emu.EMU, "-I", test_emu.BUILD, "-I", test_emu.CSRC, "-o", so, *srcs])
    lib = C.CDLL(so)
    lib.emu_sweep_stats.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_double, C.c_double,
                                    C.c_ulonglong, C.c_int, C.c_void_p]
    return lib


def _sweep(lib, dinf, d, contcheck, seed, nstrips=1):
    """(result raster, [carried visits, cells, wavefront iterations, visits]) of one emulated sweep"""
    ny, nx = d.shape
    d = np.ascontiguousarray(d)
    out = np.empty((ny, nx), np.float32)
    st = np.zeros(8, np.uint64)
    rc = lib.emu_sweep_stats(int(dinf), d.ctypes.data, out.ctypes.data, nx, ny, MISS if dinf else -32768.0, int(contcheck), 30.0, 30.0,
                             seed, nstrips, st.ctypes.data)
    assert rc == 0
    return out, [int(v) for v in st[:4]]


def _channel(ny=192, nx=320, pitch=6):
    """D8 directions and D-infinity angles of one channel winding east and west through the whole grid (rows 2, 2 + pitch, ...,
    turning at columns 2 and nx - 3), every other cell draining straight into the nearest channel row; and the channel's path."""
    p = np.zeros((ny, nx), np.int16)
    rows = list(range(2, ny - 2, pitch))
    path = []
    for i, r in enumerate(rows):
        east = i % 2 == 0
        cols = range(2, nx - 2) if east else range(nx - 3, 1, -1)
        path += [(r, c) for c in cols]
        if i + 1 < len(rows):
            path += [(rr, cols[-1]) for rr in range(r + 1, rows[i + 1])]
    on = np.zeros((ny, nx), bool)
    for r, c in path:
        on[r, c] = True
    for r in range(ny):                                   # off the channel: north (3) or south (7) towards the nearest channel row,
        for c in range(nx):                               # along a channel row beside its ends: east (1) / west (5) into it
            if not on[r, c]:
                near = min(rows, key=lambda q: (abs(q - r), q))
                p[r, c] = 7 if near > r else 3 if near < r else 1 if c < 2 else 5
    for (r, c), (r2, c2) in zip(path, path[1:]):
        p[r, c] = {(0, 1): 1, (0, -1): 5, (1, 0): 7}[(r2 - r, c2 - c)]
    r_out, c_out = path[-1]                               # the outlet drains on along its row and off the grid
    west = p[path[-2]] == 5
    p[r_out, :c_out + 1] = 5 if west else p[r_out, :c_out + 1]
    p[r_out, c_out:] = p[r_out, c_out:] if west else 1
    ang = np.choose(p, [0, 0, 0, np.pi / 2, 0, np.pi, 0, 1.5 * np.pi]).astype(np.float32)    # the cardinal D8 codes used here
    return p, ang, path


def _tile_entries(path):
    """how many times the channel enters a tile (a change of tile along the path)"""
    tiles = [(r // TS, c // TS) for r, c in path]
    return sum(1 for a, b in zip(tiles, tiles[1:]) if a != b)


@pytest.fixture(scope="module")
def channel():
    from oracle import port
    p, ang, path = _channel()
    assert len(path) > 9000
    return port, p, ang, _tile_entries(path)


@pytest.fixture(scope="module")
def random_field():
    from oracle import port
    dem = synth.punch_holes(synth.gen_dem(200, 260, hurst=0.8, tilt=1.0, seed=41))
    fel = port.pitremove(dem)
    p, _ = port.d8flowdir(fel)
    ang, _ = port.dinfflowdir(fel)
    return port, p, ang


def test_channel_matches_the_oracle_and_is_carried(emu, channel, monkeypatch):
    """A river crossing ~100 tiles: results bit for bit (with and without contamination checking), and nearly every time the river
    enters a tile the tile is carried.  (A tile entered while it is queued or running already goes through the queue.)"""
    port, p, ang, entries = channel
    assert entries > 80
    monkeypatch.setenv("TAUDEM_B200_TIMING", "1")
    monkeypatch.delenv("TAUDEM_B200_EXP", raising=False)
    ad8_nc = port.aread8(p, contcheck=False)
    assert ad8_nc.max() > 9000
    for dinf, d, ref, what in ((False, p, ad8_nc, "ad8 -nc"), (True, ang, port.areadinf(ang, contcheck=False), "sca -nc")):
        out, (carried, cells, _, visits) = _sweep(emu, dinf, d, False, 3 + dinf)
        assert_bits(out, ref, what)
        assert cells == p.size
        assert carried >= entries - 10, f"{what}: {carried} carried visits, the river enters a tile {entries} times"
        assert carried < visits
    for dinf, d, ref, what in ((False, p, port.aread8(p), "ad8"), (True, ang, port.areadinf(ang), "sca")):
        assert_bits(_sweep(emu, dinf, d, True, 5 + dinf)[0], ref, what)


def test_random_field_matches_the_oracle(emu, random_field, monkeypatch):
    port, p, ang = random_field
    monkeypatch.setenv("TAUDEM_B200_TIMING", "1")
    monkeypatch.delenv("TAUDEM_B200_EXP", raising=False)
    for seed in (11, 12):
        out, st = _sweep(emu, False, p, True, seed)
        assert_bits(out, port.aread8(p), f"ad8 seed {seed}")
        assert st[0] > 0
        out, st = _sweep(emu, True, ang, True, seed)
        assert_bits(out, port.areadinf(ang), f"sca seed {seed}")
        assert st[0] > 0


def test_carry_off_gives_the_same_results(emu, channel, random_field, monkeypatch):
    """TAUDEM_B200_EXP bit 16: every activation through the ticket queue — no carried visit, the same rasters."""
    port, p, ang, _ = channel
    _, rp, rang = random_field
    monkeypatch.setenv("TAUDEM_B200_TIMING", "1")
    monkeypatch.setenv("TAUDEM_B200_EXP", str(EXP_NO_CARRY))
    for dinf, d, ref, what in ((False, p, port.aread8(p, contcheck=False), "ad8 -nc channel"), (True, ang, port.areadinf(ang, contcheck=False), "sca -nc channel"),
                               (False, rp, port.aread8(rp), "ad8 random"), (True, rang, port.areadinf(rang), "sca random")):
        out, st = _sweep(emu, dinf, d, "-nc" not in what, 21 + dinf)
        assert_bits(out, ref, what + ", carry off")
        assert st[0] == 0 and st[3] > 0


@pytest.mark.parametrize("nstrips", [2, 3])
def test_row_strips_with_exchange_rounds(emu, channel, random_field, monkeypatch, nstrips):
    """The carry never leaves a strip: the halo counts of the exchange rounds still carry the river between strips."""
    port, p, ang, _ = channel
    _, rp, rang = random_field
    monkeypatch.setenv("TAUDEM_B200_TIMING", "1")
    monkeypatch.delenv("TAUDEM_B200_EXP", raising=False)
    for dinf, d, ref, cc, what in ((False, p, port.aread8(p, contcheck=False), False, "ad8 -nc channel"), (True, ang, port.areadinf(ang, contcheck=False), False, "sca -nc channel"),
                                   (False, rp, port.aread8(rp), True, "ad8 random"), (True, rang, port.areadinf(rang), True, "sca random")):
        out, st = _sweep(emu, dinf, d, cc, 31 + nstrips + dinf, nstrips)
        assert_bits(out, ref, f"{what}, {nstrips} strips")
        assert st[0] > 0
