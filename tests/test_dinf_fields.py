"""The D-infinity contributing-area sweep on the constructed angle fields of tests/dinf_fields.py: rivers carried from tile to
tile along tile-boundary rows, interior rows and through tile corners; second receivers in another tile at every tile edge and
corner; visits whose fork stack overflows; and the same junctions on the row-strip boundaries of 2 and 3 ranks.  Every result
is compared bit for bit: with the reference executables (their outputs recorded in tests/golden/reference.json at a moderate
size, replayed by the C restatement), with the restatement in the CPU emulation of the sweep (1, 2 and 3 strips), and with the
restatement on the GPU (one device, the executables on 2 and 3 strips in rounds and peer mode, and a 4096^2 DEM end to end)."""
import os
import subprocess

import numpy as np
import pytest

import dinf_fields as F
from taudem_b200 import synth
from util import ANG_ND, assert_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")
EMU_SIZE = (300, 330)
_receivers, _tile = F.receivers, F.tile_of


# ---------------------------------------------------------------- the fields reach what they claim
@pytest.mark.parametrize("shape", [F.MODERATE, F.LARGE], ids=["moderate", "large"])
def test_fields_reach_their_paths(shape):
    """Structure only (no sweep): the rivers' rows and lengths, the split cells' sectors and tiles, the strip boundaries."""
    ny, nx = shape
    # comb: rivers on the first row of a tile row and on interior rows, crossing nx / 32 tiles; banks split across to them
    ang = F.comb(ny, nx)
    rivers = F.comb_rivers(ny)
    assert any(r % F.TS == 0 for r in rivers) and any(r % F.TS not in (0, F.TS - 1) for r in rivers)
    for r in rivers:
        assert (ang[r, 1:] == F.E).all() and (ang[r - 1, 1:-1] > F.sector_edges()[7]).mean() > 0.9
    if shape == F.LARGE:
        assert nx // F.TS >= 90
    # the diagonal rivers pass through tile corners on the SE edge angle and its float neighbours
    e7 = np.float32(F.sector_edges()[7])
    corner = [(r, c) for r in range(ny - 4 * F.TS, ny - 1) for c in range(1, nx - 1) if r % F.TS == F.TS - 1 and c % F.TS == F.TS - 1
              and abs(float(ang[r, c]) - float(e7)) < 1e-6]
    assert len(corner) >= 3 * (nx // 64)
    vals = set(ang[ny - 4 * F.TS:, 1:-1][np.abs(ang[ny - 4 * F.TS:, 1:-1] - e7) < 1e-6].tolist())
    assert {float(e7), float(np.nextafter(e7, np.float32(10))), float(np.nextafter(e7, np.float32(-10)))} <= vals
    # edge splits: at each of the four tile corners every sector, with the two receivers in two different tiles (diagonal one included)
    _, cells, k = F.edge_splits(ny, nx)
    seen, diag, edge = set(), 0, 0
    for (r, c), kk in zip(cells, k):
        lr, lc = r % F.TS, c % F.TS
        a, b = _receivers(r, c, kk)
        if lr in (0, F.TS - 1) and lc in (0, F.TS - 1):
            seen.add((int(lr), int(lc), int(kk)))
            t = _tile((r, c))
            diag += any(abs(_tile(x)[0] - t[0]) == 1 and abs(_tile(x)[1] - t[1]) == 1 for x in (a, b))
        else:
            assert _tile(a) != _tile(b), (r, c, kk)
            edge += 1
    assert len(seen) == 32, sorted(seen)
    assert diag > 20 and edge > nx * ny // 200, (diag, edge)
    # fork flood: a third of the cells split, and each of the others has one contributor
    ff = F.fork_flood(ny, nx)
    assert abs((ff[1:-1, 1:-1] >= 0).mean() - 1 / 3) < 0.01
    # strip edges: a river on (or next to) every boundary row of the 2- and 3-rank partitions, its banks on both sides of it
    se = F.strip_edges(ny, nx)
    for b in F.strip_boundaries(ny):
        assert (se[b, 1:] == F.E).all() or (se[b - 1, 1:] == F.E).all(), b


# ---------------------------------------------------------------- the C restatement on the reference executables
def test_restatement_replays_the_reference_on_the_fields(refrun, tmp_path):
    """areadinf plain, -wg and -nc of the reference executables on every field at 600 x 1300 (recorded in reference.json),
    recomputed by the restatement; the count is asserted: a call that is not replayed fails here."""
    import port
    import reference
    if not port.available():
        pytest.skip("oracle/port not built")
    ny, nx = F.MODERATE
    w = synth.gen_weights(ny, nx, seed=5)
    keys = set()
    for name, make in F.FIELDS.items():
        ang = make(ny, nx)
        R = refrun.RefPipeline(workdir=str(tmp_path), dx=30.0, dy=30.0, np_ranks=1)
        before = set(reference.replayed)
        sca = R.areadinf(ang)
        R.areadinf(ang, weights=w)
        R.areadinf(ang, contcheck=False)
        assert (np.asarray(sca) > 0).mean() > 0.9, name
        if not reference.RECORD:
            new = set(reference.replayed) - before
            assert len(new) == 3, name
            keys |= new
    assert reference.RECORD or len(keys) == len(F.FIELDS) * 3 == 12


# ---------------------------------------------------------------- emulated sweep (CPU)
@pytest.fixture(scope="module")
def carry_emu():
    import test_sweep_carry
    return test_sweep_carry.build_lib()


@pytest.mark.parametrize("name", list(F.FIELDS))
def test_emulated_sweep_on_the_fields(carry_emu, name, monkeypatch):
    """Each field through the emulated sweep on 1, 2 and 3 row strips (the exchange rounds), several interleaving seeds, with
    and without contamination checking, bit for bit against the restatement.  The fork flood runs with the default fork stack
    and must overflow it in every run: the statistics counter of such visits is positive."""
    from oracle import port
    from test_sweep_carry import _sweep
    monkeypatch.setenv("TAUDEM_B200_TIMING", "1")
    monkeypatch.delenv("TAUDEM_B200_EXP", raising=False)
    ang = F.FIELDS[name](*EMU_SIZE)
    ref = {True: port.areadinf(ang), False: port.areadinf(ang, contcheck=False)}
    for nstrips, seed, cont in ((1, 1, True), (1, 2, False), (2, 3, True), (3, 4, True), (3, 5, False)):
        out, st = _sweep(carry_emu, True, ang, cont, seed, nstrips)
        assert_bits(out, ref[cont], f"sca {name}, {nstrips} strips, seed {seed}, contcheck={cont}")
        if name == "fork_flood":
            assert st[4] > 0, f"the fork stack never overflowed: {st}"
    if name != "fork_flood":
        assert ref[True].max() > 5e4


# ---------------------------------------------------------------- GPU
def _values(rng, shape):
    dm = rng.uniform(0.5, 1.0, shape).astype(np.float32)
    dm[rng.random(shape) < 0.01] = -9999.0
    q = rng.uniform(0.0, 3.0, shape).astype(np.float32)
    dg = (rng.random(shape) < 0.002).astype(np.int16)
    return dm, q, dg


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(F.FIELDS))
def test_gpu_fields_against_the_restatement(name):
    """areadinf_grid plain, -wg and -nc, dinfdecayaccum_grid and dinfconclimaccum_grid on each field at 1040 x 3300 (103 tiles
    across), bit for bit against the restatement."""
    import port
    import taudem_b200 as td
    ny, nx = F.LARGE
    ang = F.FIELDS[name](ny, nx)
    w = synth.gen_weights(ny, nx, seed=6)
    sca = port.areadinf(ang)
    assert_bits(td.areadinf_grid(ang), sca, f"sca {name}")
    assert_bits(td.areadinf_grid(ang, weights=w), port.areadinf(ang, weights=w), f"sca -wg {name}")
    assert_bits(td.areadinf_grid(ang, contcheck=False), port.areadinf(ang, contcheck=False), f"sca -nc {name}")
    dm, q, dg = _values(np.random.default_rng(7), ang.shape)
    assert_bits(td.dinfdecayaccum_grid(ang, dm), port.dinfdecayaccum(ang, dm), f"dsca {name}")
    assert_bits(td.dinfconclimaccum_grid(ang, dm, q, dg, csol=1.5, contcheck=False), port.dinfconclimaccum(ang, dm, q, dg, csol=1.5, contcheck=False),
                f"ctpt -nc {name}")
    if name == "comb":
        assert min(sca[r, nx - 2] for r in F.comb_rivers(ny)) > 3e6          # every river outlet


@pytest.mark.gpu
def test_gpu_fork_stack_overflows_on_the_fork_flood(monkeypatch):
    """With TAUDEM_B200_TIMING=1 the sweep counts the visits whose fork stack overflowed (td_ctx_counter 32): positive on the
    fork flood, where the rescan of the counts then finds the second receivers that did not fit; the result bit for bit."""
    import torch
    import port
    from taudem_b200.device import DeviceStrip, Tools
    monkeypatch.setenv("TAUDEM_B200_TIMING", "1")
    ny, nx = F.LARGE
    ang = F.fork_flood(ny, nx)
    s = DeviceStrip(nx, ny)
    a = s.empty(torch.float32)
    a.fill_(float(ANG_ND))
    s.owned(a).copy_(torch.from_numpy(ang))
    T = Tools()
    try:
        sca = T.areadinf(s, a, s.rows(30.0), s.rows(30.0))
        torch.cuda.synchronize()
        c = [T.l.td_ctx_counter(T.ctx, 24 + i) for i in range(9)]
        out = s.owned(sca).cpu().numpy()
    finally:
        T.close()
    assert_bits(out, port.areadinf(ang), "sca fork flood (device call)")
    assert c[3] >= (ny // 32) * (nx // 32) and c[8] > c[3] // 4, f"visits {c[3]}, overflowed {c[8]}"


def _areadinf_exe(gpus, args, peer):
    env = dict(os.environ, TAUDEM_B200_GPUS=str(gpus))
    env.pop("TAUDEM_B200_PEER", None)
    if peer is not None:
        env["TAUDEM_B200_PEER"] = peer
    r = subprocess.run([os.path.join(BIN, "areadinf")] + [str(a) for a in args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0 and "error" not in r.stdout.lower(), r.stdout
    assert f"Processors: {gpus}" in r.stdout, r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["rounds", "peer"])
def test_gpu_executables_on_row_strips(mode, tmp_path):
    """The areadinf executable with TAUDEM_B200_GPUS=2 and 3 on the strip-edge and comb fields, plain and -wg: rounds mode
    (TAUDEM_B200_PEER=0, ranks may share a device) and peer mode (one device per rank), bit for bit against the restatement."""
    import port
    import taudem_b200 as td
    counts = (2, 3) if mode == "rounds" else [n for n in (2, 3) if td.device_count() >= n]
    if not counts:
        pytest.skip(f"peer mode needs one device per rank: {td.device_count()} device(s)")
    peer = "0" if mode == "rounds" else None
    ny, nx = F.LARGE
    w = synth.gen_weights(ny, nx, seed=8)
    td.write_raster(str(tmp_path / "w.tif"), w, -9999.0, dx=30.0, dy=30.0)
    for name in ("strip_edges", "comb"):
        ang = F.FIELDS[name](ny, nx)
        td.write_raster(str(tmp_path / "ang.tif"), ang, ANG_ND, dx=30.0, dy=30.0)
        for extra, ref in (([], port.areadinf(ang)), (["-wg", tmp_path / "w.tif"], port.areadinf(ang, weights=w))):
            for n in counts:
                out = tmp_path / f"sca_{name}_{n}.tif"
                _areadinf_exe(n, ["-ang", tmp_path / "ang.tif", "-sca", out] + extra, peer)
                assert_bits(td.read_raster(str(out)), ref, f"sca {name} {' '.join(map(str, extra[:1]))} on {n} ranks ({mode})")


@pytest.mark.gpu
def test_gpu_dinf_large():
    """4096^2 end to end on the D-infinity side: pitremove_grid -> dinfflowdir_grid, ang bit for bit against the restatement's
    dinfflowdir of the same fel, then areadinf_grid bit for bit against the restatement's areadinf."""
    import port
    import taudem_b200 as td
    dem = synth.gen_dem(4096, hurst=0.8, tilt=1.0, seed=77)
    fel = td.pitremove_grid(dem)
    ang, slp = td.dinfflowdir_grid(fel)
    ang_o, slp_o = port.dinfflowdir(fel)
    assert_bits(slp, slp_o, "slp 4096^2")
    assert_bits(ang, ang_o, "ang 4096^2")
    sca = td.areadinf_grid(ang_o)
    assert_bits(sca, port.areadinf(ang_o), "sca 4096^2")
    assert sca.max() > 1e7
