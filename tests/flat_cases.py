"""The DEMs of the flat-resolution tests (taudem_b200/csrc/flats.cu against the C restatement), each from a seed or a closed form.

Each case returns (dem, fel): dem the raw DEM, fel the input of d8flowdir / dinfflowdir (dem itself for the unfilled cases).
REACH states what the case is there for; tests/test_cpu.py checks it with port.flat_stats() on every call, so a case that no
longer reaches it fails on the CPU.  CALLS lists the reference calls of the GPU tests (tests/test_gpu_parity.py), which the
CPU suite replays through tests/reference.py.
"""
import numpy as np

import port
from taudem_b200 import synth

SIZES = ((30.0, 30.0), (10.0, 25.0))          # square cells and dx != dy
BATCH_THREADS_132 = 132 * 4 * 256               # one pass of k_bfs_level's fixed grid on a 132-SM H100


def deep_lake():
    """A 600 x 600 bowl that pitremove fills into one lake of about 200 000 cells, spilling through a single channel cut into
    the east rim: about 510 fall levels (8 batches of 64) and 255 rise levels."""
    n = 600
    y, x = np.mgrid[0:n, 0:n].astype(np.float64)
    r = np.hypot(x - 299.5, y - 299.5)
    dem = np.where(r < 270, r / 270 * 95, 120.0)
    row = (y >= 298) & (y <= 301) & (x >= 299.5 + 250)          # the channel: 90 at its head, falling to 80 at the edge
    dem = np.where(row, 90.0 - (x - 549.5) / 50 * 10, dem).astype(np.float32)
    return dem, port.pitremove(dem)


def pockets():
    """90 x 90 flat-bottomed pockets of 10 x 10 cells behind walls, each spilling through one notch in its east wall into the
    next pocket (floors step down by 1 eastward and southward): 810 000 flat cells resolved at once, 267 300 of them in the
    first rise level, which k_bfs_level's stride loop crosses in two passes of its fixed grid on a 132-SM H100."""
    P, w = 90, 11
    n = P * w + 2
    i = np.arange(n)
    blk, pos = (i - 1) // w, (i - 1) % w
    floor_r = (pos != 0) & (i > 0) & (i < n - 1)
    F = 200.0 - (np.clip(blk, 0, P - 1)[:, None] + np.clip(blk, 0, P - 1)[None, :])
    dem = np.full((n, n), 1000.0)
    inside = floor_r[:, None] & floor_r[None, :]
    dem[inside] = F[inside]
    notch_c = np.nonzero((pos == 0) & (blk >= 1))[0]            # east wall of pocket blk-1
    notch_r = np.nonzero(floor_r & (pos == 6))[0]                # one row per pocket
    for c in notch_c:
        J = blk[c] - 1
        dem[notch_r, c] = 200.0 - (blk[notch_r] + J) - 0.5
    dem = dem.astype(np.float32)
    return dem, port.pitremove(dem)


def multipass():
    """The terrace family of tests/test_emu.py (quantised elevations, nodata holes), seed 0: three outer iterations."""
    dem = synth.gen_dem(120, 150, hurst=0.8, tilt=1.0, seed=0)
    q = (dem.max() - dem.min()) / 14
    dem = synth.punch_holes((np.round(dem / q) * q).astype(np.float32), seed=3)
    return dem, port.pitremove(dem)


def pits():
    """Unfilled: 40 closed flat-bottomed basins (5 x 5 floors behind walls, which become pits) beside a 1-wide corridor of 150
    cells that drains at its east end, so that T (and with it the pits' elev2 = 1 + T) comes from the corridor."""
    ny, nx = 40, 160
    dem = np.full((ny, nx), 50.0)
    dem[2, 1:nx - 1] = 100.0; dem[4, 1:nx - 1] = 100.0
    dem[3, 1:nx - 1] = 10.0; dem[3, nx - 1] = 5.0               # the corridor and its outlet on the edge
    for k in range(40):
        r0, c0 = 8 + 8 * (k // 16), 3 + 9 * (k % 16)
        dem[r0:r0 + 7, c0:c0 + 7] = 80.0
        dem[r0 + 1:r0 + 6, c0 + 1:c0 + 6] = 20.0 + k % 3
    dem += np.linspace(0, 1, nx)[None, :] * (dem == 50.0) * -1.0 # the open ground drains east
    dem = dem.astype(np.float32)
    return dem, dem


def edges():
    """A quantised rough DEM, filled, with nodata holes and a band along the north and west edges lowered onto one terrace:
    flats that touch the grid edge and cells beside nodata (equal neighbours outside the flat set), and a second outer
    iteration."""
    dem = synth.gen_dem(200, 260, hurst=0.5, tilt=0.2, seed=23)
    q = (dem.max() - dem.min()) / 10
    dem = (np.round(dem / q) * q).astype(np.float32)
    lo = dem.min()
    dem[:12, :] = lo; dem[:, :12] = lo
    dem = synth.punch_holes(dem, seed=7)
    return dem, port.pitremove(dem)


def wrap16(length=16500):
    """Two flats side by side on an 8-row strip.  A (row 5) is a corridor of `length` cells between higher walls that drains at
    its east end: fall levels 1 .. length.  B (row 1) is a strip of `length` cells whose south neighbours (row 2) have the same
    elevation and drain to a lower row; the only higher ground at B is the west edge: every B cell is at fall level 1 and the
    rise passes run along B, U = length + 1.  A's cells all rise (walls), so its elev2 = level + U passes 32767 at the far end
    while T and U stay below it: the reference stores a negative elev2 there, that cell stays flat and becomes a pit in the
    second outer iteration."""
    nx = length + 2
    dem = np.empty((8, nx))
    dem[0:3, :] = 10.0                                           # edge row, B, and B's draining neighbours
    dem[3, :] = 5.0 - np.arange(nx) * 1e-4                       # the lower row they drain to, falling east
    dem[4, :] = dem[6, :] = dem[7, :] = 30.0                     # A's walls
    dem[5, :] = 1.0; dem[5, nx - 1] = 0.0                        # A and its outlet on the east edge
    dem[:, 0] = 20.0                                             # higher ground at B's west end (and beside A's)
    dem = dem.astype(np.float32)
    return dem, dem


def corridor(length=32768):
    """A single corridor of `length` cells between higher walls, draining at its east end (its last cell directly): `length` fall
    passes."""
    nx = length + 2
    dem = np.full((5, nx), 30.0)
    dem[2, 1:] = 1.0; dem[2, nx - 1] = 0.0
    return dem.astype(np.float32), dem.astype(np.float32)


CASES = {"deep_lake": deep_lake, "pockets": pockets, "multipass": multipass, "pits": pits, "edges": edges, "wrap16": wrap16}


def reach(name, stats):
    """What the case must reach (port.flat_stats() of one d8flowdir / dinfflowdir call); returns the failed conditions."""
    s = stats
    want = {
        "deep_lake": [("T > 2 + 2 * 64 (three batches of levels)", s["T"] > 130), ("U > 150", s["U"] > 150)],
        "pockets": [("a rise level holds more cells than one pass of the 132-SM grid", s["rise_level"] > BATCH_THREADS_132)],
        "multipass": [("3 outer iterations", s["iters"] >= 3)],
        "pits": [("pits", s["pits"] > 0), ("T from the corridor", s["T"] > 150)],
        "edges": [("2 outer iterations", s["iters"] >= 2), ("deep flats", s["T"] > 50)],
        "wrap16": [("level + s > 32767", s["elev2"] > 32767), ("T < 32767", s["T"] < 32767), ("U < 32767", s["U"] < 32767),
                   ("2 outer iterations", s["iters"] >= 2), ("pits", s["pits"] > 0)],
    }[name]
    return [w for w, ok in want if not ok]


def edge_features(fel):
    """(flat cells beside an equal grid-edge cell, flat cells beside an equal cell that has a nodata neighbour): the seeds of
    k_classify's "equal neighbour outside the flat set" in the first outer iteration"""
    p0, _ = port.d8flowdir(fel, flats=False)
    ny, nx = fel.shape
    nd = fel < -1e38
    near_nd = np.zeros_like(nd)
    pad = np.pad(nd, 1)
    for dr in (-1, 0, 1):
        for dc in (-1, 0, 1):
            near_nd |= pad[1 + dr:1 + dr + ny, 1 + dc:1 + dc + nx]
    edge = np.zeros_like(nd); edge[0, :] = edge[-1, :] = edge[:, 0] = edge[:, -1] = True
    seed_edge = seed_nd = 0
    d1 = (0, 1, 1, 0, -1, -1, -1, 0, 1); d2 = (0, 0, -1, -1, -1, 0, 1, 1, 1)
    rr, cc = np.nonzero(p0 == 0)
    for k in range(1, 9):
        nr, nc = rr + d2[k], cc + d1[k]
        eq = fel[nr, nc] == fel[rr, cc]
        seed_edge += int((eq & edge[nr, nc]).sum())
        seed_nd += int((eq & ~edge[nr, nc] & near_nd[nr, nc] & ~nd[nr, nc]).sum())
    return seed_edge, seed_nd


def calls(name):
    """The reference calls of case `name`'s tests, one reference rank: (dx, dy, tool, args) — pitremove of the raw DEM where the
    case fills it, then d8flowdir and dinfflowdir for each cell size."""
    dem, fel = CASES[name]()
    out = [] if fel is dem else [(30.0, 30.0, "pitremove", dem)]
    return out + [(dx, dy, tool, fel) for dx, dy in SIZES for tool in ("d8flowdir", "dinfflowdir")]
