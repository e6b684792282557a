"""Constructed D-infinity angle grids for the contributing-area sweep (taudem_b200/csrc/sweep_warp.cu), built directly as angles
(no DEM, no flow-direction tool): each one puts many cells on one path of the sweep where a lost or doubled share would change
bits that a relative tolerance cannot see.  Every grid is acyclic by construction, and its border cells drain off the grid, so
with contamination checking only the border itself (and what the border drains into) is nodata.

The sweep works on 32 x 32 tiles (TS, TH in sweep_warp.cu): tile row r // 32, tile column c // 32 (grid rows and columns from 0,
north first).  Angles: 0 = east, counter-clockwise, the reference's PI literal for the sector edges."""
import numpy as np

TS = 32                                         # tile edge of the sweep
PI = 3.14159265359                              # the reference's PI
ANG_ND = np.float32(-3.4028234663852886e38)
E, N, W, S = np.float32(0.0), np.float32(0.5 * PI), np.float32(PI), np.float32(1.5 * PI)
LARGE = (1040, 3300)                            # the GPU tests' size: rivers of 103 tiles, outlets above 3e6 cell units
MODERATE = (600, 1300)                          # the size recorded from the reference executables


def sector_edges(dx=30.0, dy=30.0):
    """the nine angles where the receivers change (E, NE, N, ..., E again at 2 PI), as the reference computes them"""
    t = np.arctan2(dy, dx)
    return [0.0, t, 0.5 * PI, PI - t, PI, PI + t, 1.5 * PI, 2 * PI - t, 2 * PI]


def in_sector(rng, k, size, dx=30.0, dy=30.0, lo=0.02, hi=0.98):
    """angles strictly inside sector k (0 = between E and NE, ..., 7 = between SE and E): both receivers get a share"""
    e = sector_edges(dx, dy)
    return (e[k] + rng.uniform(lo, hi, size) * (e[k + 1] - e[k])).astype(np.float32)


# direction d = 1..8 (E, NE, N, NW, W, SW, S, SE): row and column offsets; sector k = 0..7 lies between directions k + 1 and k + 2
DROW = (0, 0, -1, -1, -1, 0, 1, 1, 1)
DCOL = (0, 1, 1, 0, -1, -1, -1, 0, 1)


def receivers(r, c, k):
    """the two receivers (row, column) of cell (r, c) with an angle inside sector k"""
    d1, d2 = k + 1, k + 2 if k < 7 else 1
    return (r + DROW[d1], c + DCOL[d1]), (r + DROW[d2], c + DCOL[d2])


def tile_of(rc):
    return rc[0] // TS, rc[1] // TS


def _ulps(v):
    f = np.float32(v)
    return [f, np.nextafter(f, np.float32(10)), np.nextafter(f, np.float32(-10))]


def _border(ang):
    """border cells drain straight off the grid (north row north, west column west, ...): they are the only contaminated cells"""
    ang[0, :] = N
    ang[-1, :] = S
    ang[:, 0] = W
    ang[:, -1] = E


def river_comb(ny, nx, rivers, seed, dx=30.0, dy=30.0):
    """Rivers running east along the given rows, fed from both sides by single-cell tributaries that split their flow.

    Every other cell drains towards the nearest river row: hillslope cells with an angle anywhere between SW and SE (north of a
    river) or NW and NE (south of it), so every share moves one row closer.  The rows beside a river are its banks: a bank cell
    splits between E (the next bank cell, beside the river) and SE / NE (the next river cell), so every river cell is a junction
    of three contributors and every bank cell hands a share across to the river.  Rivers need 4 rows between them."""
    rng = np.random.default_rng(seed)
    ang = np.empty((ny, nx), np.float32)
    rows = np.arange(ny)
    rv = np.array(sorted(rivers))
    assert len(rv) and (np.diff(rv) >= 4).all() and rv[0] >= 2 and rv[-1] <= ny - 3, rivers
    near = rv[np.abs(rows[:, None] - rv[None, :]).argmin(axis=1)]
    south = near > rows                          # rows north of their river drain south
    e = sector_edges(dx, dy)
    for r in range(ny):
        if near[r] == r:
            ang[r] = E
        elif abs(near[r] - r) == 1:              # bank: E + SE (north bank) or E + NE (south bank), a few exact edges among them
            ang[r] = in_sector(rng, 7 if south[r] else 0, nx, dx, dy)
            pick = rng.random(nx) < 0.03
            ang[r, pick] = np.float32(e[7] if south[r] else e[1])
        else:                                    # hillslope: anywhere from SW to SE (or NW to NE), cardinal and split
            lo, hi = (e[5], e[7]) if south[r] else (e[1], e[3])
            ang[r] = rng.uniform(lo, hi, nx).astype(np.float32)
            pick = rng.random(nx) < 0.1
            ang[r, pick] = S if south[r] else N
    _border(ang)
    return ang


def diagonal_rivers(ang, r0, seed, spacing=64, dx=30.0, dy=30.0):
    """Overwrites rows r0.. of `ang` with rivers running SE along diagonals through tile corners (cell (32i - 1, 32j - 1) drains
    into (32i, 32j), a tile diagonal to its own) every `spacing` columns, on angles exactly at the SE sector edge and one ulp
    either side of it (the second receiver, E or S, appears and disappears).  Every other cell drains towards its nearest
    diagonal with an angle between S and SE (right of it) or SE and E (left of it): every share moves south or east, so nothing
    can flow back.  The block's west column drains west; its rows above drain north, away from it."""
    rng = np.random.default_rng(seed)
    ny, nx = ang.shape
    i, j = np.mgrid[r0:ny, 0:nx]
    c0 = r0 % TS                                             # a diagonal through (r0, c0 + k spacing) meets the tile corners
    d = (j - c0 - (i - r0)) % spacing
    d = np.where(d > spacing // 2, d - spacing, d)           # signed distance (columns) to the nearest diagonal
    blk = np.where(d > 0, in_sector(rng, 6, d.shape, dx, dy), in_sector(rng, 7, d.shape, dx, dy))
    ulps = np.array(_ulps(sector_edges(dx, dy)[7]) + _ulps(1.75 * np.pi), np.float32)
    on = d == 0
    blk[on] = ulps[rng.integers(0, len(ulps), int(on.sum()))]
    ang[r0:] = blk
    _border(ang)
    return ang


def comb(ny, nx, seed=1, dx=30.0, dy=30.0):
    """Reaches: rivers carried from tile to tile (the sweep's carry and its one-chain mode), each river crossing nx / 32 tiles.
    Rivers alternate between the first row of a tile row (row 64 k: its north bank lies in the tile row above, so every
    bank share crosses a tile edge) and an interior row (64 k + 45); below them, the rows from ny - 128 hold diagonal rivers
    through tile corners (diagonal_rivers).  At LARGE the river outlets exceed 3e6 cell units (30 per cell at dx = 30), so one
    tributary cell is below 1e-5 of the river it joins near the outlet."""
    r_diag = ny - 4 * TS
    rivers = [r for k in range(1, ny // 64 + 1) for r in (64 * k, 64 * k + 45) if r < r_diag - 20]
    ang = river_comb(ny, nx, rivers, seed, dx, dy)
    return diagonal_rivers(ang, r_diag, seed + 1000, dx=dx, dy=dy)


def comb_rivers(ny):
    """the river rows of comb(ny, ...)"""
    r_diag = ny - 4 * TS
    return [r for k in range(1, ny // 64 + 1) for r in (64 * k, 64 * k + 45) if r < r_diag - 20]


def edge_splits(ny, nx, seed=2, dx=30.0, dy=30.0):
    """Reaches: second receivers in another tile.  Cells on every tile edge and at every tile corner split their flow between
    two receivers, in all eight sectors: at a corner, sectors whose receivers lie in the two edge neighbour tiles or in an
    edge neighbour and the diagonal neighbour tile; on an edge, one receiver in the cell's own tile and one across.

    Background: every cell drains between S and E (angle in [3 PI / 2, 2 PI]), so r + c grows along every share and there is no
    cycle.  A split cell (any sector) can only be re-entered from its N, W or NW neighbour: those three are fixed to drain away
    from it (N neighbour east, W and NW neighbours south).  Split cells are 3 cells apart at least."""
    rng = np.random.default_rng(seed)
    ang = np.where(rng.random((ny, nx)) < 0.5, in_sector(rng, 6, (ny, nx), dx, dy, 0.0, 1.0), in_sector(rng, 7, (ny, nx), dx, dy, 0.0, 1.0))
    taken = np.zeros((ny, nx), bool)
    cells = []
    for corners in (True, False):                            # the tile corners first, then cells along the tile edges
        for tr in range(ny // TS + 1):
            for tc in range(nx // TS + 1):
                r0, c0 = tr * TS, tc * TS
                if corners:                                  # all four corners of every other tile (its neighbours' corners touch them)
                    cand = [(r0, c0), (r0, c0 + TS - 1), (r0 + TS - 1, c0), (r0 + TS - 1, c0 + TS - 1)] if tr % 2 == tc % 2 == 0 else []
                else:
                    x = [int(v) for v in rng.integers(2, TS - 2, 8)]
                    cand = [(r0, c0 + x[0]), (r0, c0 + x[1]), (r0 + TS - 1, c0 + x[2]), (r0 + TS - 1, c0 + x[3]),
                            (r0 + x[4], c0), (r0 + x[5], c0), (r0 + x[6], c0 + TS - 1), (r0 + x[7], c0 + TS - 1)]
                rng.shuffle(cand)
                for r, c in cand:
                    if 2 <= r < ny - 2 and 2 <= c < nx - 2 and not taken[r - 2:r + 3, c - 2:c + 3].any():
                        taken[r, c] = True
                        cells.append((r, c))
    cells = np.array(cells)
    r, c = cells[:, 0], cells[:, 1]
    k = np.zeros(len(cells), np.int64)
    turn = {}
    for n, (cr, cc) in enumerate(cells):
        q = (int(cr) % TS, int(cc) % TS)
        if q[0] in (0, TS - 1) and q[1] in (0, TS - 1):      # the corners of each kind take the eight sectors in turn
            k[n] = turn.get(q, int(rng.integers(0, 8))) % 8
            turn[q] = k[n] + 1
        else:                                                # an edge cell: a sector with one receiver on each side of the edge
            ok = [kk for kk in range(8) if len({tile_of(x) for x in receivers(int(cr), int(cc), kk)}) == 2]
            k[n] = ok[int(rng.integers(0, len(ok)))]
    e = np.array(sector_edges(dx, dy))
    ang[r, c] = (e[k] + rng.uniform(0.02, 0.98, len(cells)) * (e[k + 1] - e[k])).astype(np.float32)
    ang[r - 1, c] = E                            # the three neighbours that could drain back into a split cell drain away from it
    ang[r, c - 1] = S
    ang[r - 1, c - 1] = S
    _border(ang)
    return ang, cells, k


def fork_flood(ny, nx, seed=3, dx=30.0, dy=30.0):
    """Reaches: the fork stack's overflow and the rescan of the shared-memory counts (sweep_warp.cu, STKCAP = 128).

    Every row of every tile is one third sources and two thirds sinks, on diagonal stripes: cell (r, c) is a source when
    (c - r) % 3 == 0 and splits between E (a sink of its own row) and NE (a sink of the row above), angles anywhere inside
    the sector; every other cell has no direction (angle -1) and exactly one contributor.  So every lane of a visit starts
    with ~10 ready sources in its own tile row, and every source it evaluates makes both of its receivers ready: the lane
    continues with one and pushes the other on the fork stack, while no lane is idle to take from it: about 300 second
    receivers become pending in one visit."""
    rng = np.random.default_rng(seed)
    i, j = np.mgrid[0:ny, 0:nx]
    ang = np.full((ny, nx), -1.0, np.float32)
    src = (j - i) % 3 == 0
    ang[src] = in_sector(rng, 0, int(src.sum()), dx, dy)
    _border(ang)
    return ang


def strip_boundaries(ny, worlds=(2, 3)):
    """the first rows of the row strips after the first, for the rank counts of `worlds` (taudem_b200.dist.partition)"""
    from taudem_b200.dist import partition
    return sorted({row0 for w in worlds for row0, _ in partition(ny, w)[1:]})


def strip_edges(ny, nx, seed=4, dx=30.0, dy=30.0):
    """Reaches: the exchange of areas and dependency counts between row strips (rounds mode: halo counts; peer mode: deliveries
    into the neighbour GPU).  The rivers of river_comb run along the row-strip boundaries of the 2- and 3-rank partitions: along
    the first row of a strip (its north bank, in the strip above, hands every share across the boundary) and along the last row
    of the strip above (its south bank, in the strip below, hands them back up).  Every river cell is a junction of a share that
    crosses the boundary and one that does not."""
    b = strip_boundaries(ny)
    rivers = []
    for i, r in enumerate(b):
        rivers.append(r if i % 2 == 0 else r - 1)
    return river_comb(ny, nx, rivers, seed, dx, dy)


FIELDS = {"comb": comb, "edge_splits": lambda ny, nx, **kw: edge_splits(ny, nx, **kw)[0], "fork_flood": fork_flood, "strip_edges": strip_edges}
