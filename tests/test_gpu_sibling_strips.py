"""The five sibling sweep tools on row strips on the GPU: the device-strip level in one process (2 and 3 strips, each with its own
context, the exchange rounds made one strip after the other) against the host-grid call, and the executables under
TAUDEM_B200_GPUS=2 and 3 against the single-GPU run and the C restatement, in rounds mode and, with one device per rank, in peer
mode.  The target is always the single-rank result (the reference's own multi-rank dinfdecayaccum -nc is not deterministic on a
strip's first row)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import port
import sibling_cases
import taudem_b200 as td
from taudem_b200._lib import check, lib
from taudem_b200.device import DeviceStrip, Tools
from taudem_b200.dist import partition
from util import ANG_ND, assert_bits, write_geographic_dem

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "taudem_b200", "bin")


# ---------------------------------------------------------------- device-strip level, one process
class Strips:
    """n row strips of a grid on the current device, each with its own td_ctx"""

    def __init__(self, shape, n):
        import torch
        self.torch = torch
        self.ny, self.nx = shape
        self.S = [DeviceStrip(self.nx, k, has_top=i > 0, has_bot=i < n - 1, row0=r0, total_ny=self.ny) for i, (r0, k) in enumerate(partition(self.ny, n))]
        self.T = [Tools() for _ in self.S]

    def load(self, a, dtype):
        """every strip's rows of `a` with their halo rows"""
        out = []
        for s in self.S:
            t = s.empty(dtype).zero_()
            lo, hi = max(s.row0 - 1, 0), min(s.row0 + s.ny + 1, self.ny)
            t[lo - s.row0 + 1:hi - s.row0 + 1, :self.nx] = self.torch.from_numpy(np.ascontiguousarray(a[lo:hi]))
            out.append(t)
        return out

    def empty(self, dtype):
        return [s.empty(dtype) for s in self.S]

    def rows(self, v):
        return [self.torch.from_numpy(np.ascontiguousarray(v[s.row0:s.row0 + s.ny], np.float64)).cuda() for s in self.S]

    def gather(self, ts):
        return np.concatenate([s.owned(t).cpu().numpy() for s, t in zip(self.S, ts)])

    @staticmethod
    def st():
        import torch
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def rounds(self, run, vals):
        """begin, then rounds of run(i, halo_out) + the exchange of the decrements and the edge rows of every value in vals[v][i]"""
        torch, l = self.torch, lib()
        halos = [torch.zeros(2 * s.pitch, dtype=torch.int32, device="cuda") for s in self.S]
        for s, T in zip(self.S, self.T):
            check(l.td_sweep_begin_dev(T.ctx, s.c, self.st()))
        n, handed_total = 0, 0
        while True:
            for i, h in enumerate(halos):
                h.zero_()
                run(i, C.c_void_p(h.data_ptr()))
            torch.cuda.synchronize()
            n += 1
            handed = int(sum(int(h.sum()) for h in halos))
            handed_total += handed
            for i in range(len(self.S) - 1):
                a, b = self.S[i], self.S[i + 1]
                for v in vals:
                    v[i + 1][0].copy_(v[i][a.ny]); v[i][a.ny + 1].copy_(v[i + 1][1])
            if handed == 0:
                break
            for i, (s, T) in enumerate(zip(self.S, self.T)):
                top = C.c_void_p(halos[i - 1][s.pitch:].data_ptr()) if i > 0 else None
                bot = C.c_void_p(halos[i + 1][:self.S[i + 1].pitch].data_ptr()) if i + 1 < len(self.S) else None
                check(l.td_sweep_apply_halo_dev(T.ctx, s.c, top, bot, self.st()))
        assert n > 1 and handed_total > 0
        return n

    def close(self):
        for T in self.T:
            T.close()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _geo_rows(ny):
    lat = np.deg2rad(41.9 - 0.001 * np.arange(ny))
    return 111320.0 * 0.001 * np.cos(lat), np.full(ny, 110950.0 * 0.001)


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    return {c.__name__: c(tmp_path_factory.mktemp(c.__name__))[0] for c in sibling_cases.CASES}


@pytest.mark.parametrize("n", [2, 3])
def test_device_strips_match_the_grid_call(cases, n):
    import torch
    l = lib()
    # d8flowpathextremeup
    x = cases["flowpathextremeup"]
    p, sa = x["p"], x["sa"]
    S = Strips(p.shape, n)
    P, SA, OUT = S.load(p, torch.int16), S.load(sa, torch.float32), S.empty(torch.float32)
    for s, T, pp, o in zip(S.S, S.T, P, OUT):
        check(l.td_d8flowpathextremeup_deps_dev(T.ctx, _p(pp), _p(o), s.c, -32768, S.st()))
    S.rounds(lambda i, h: check(l.td_d8flowpathextremeup_sweep_run_dev(S.T[i].ctx, _p(SA[i]), _p(OUT[i]), S.S[i].c, 1, 1, h, S.st())), [OUT])
    assert_bits(S.gather(OUT), td.d8flowpathextremeup_grid(p, sa), f"ssa, {n} strips")
    S.close()

    # gridnet with a mask: three sweeps, then the Strahler orders
    x = cases["gridnet"]
    p, mask = x["p"], x["mask"]
    S = Strips(p.shape, n)
    P, M, OK, OUT, G = S.load(p, torch.int16), S.load(mask, torch.int32), S.empty(torch.float32), S.empty(torch.float32), S.empty(torch.int16)
    e1, e2 = np.array([0, 1, 1, 0, -1, -1, -1, 0, 1]), np.array([0, 0, -1, -1, -1, 0, 1, 1, 1])
    dist = [torch.from_numpy(np.sqrt(30.0 ** 2 * e1[1:] ** 2 + 30.0 ** 2 * e2[1:] ** 2).astype(np.float32)[None, :].repeat(s.ny, 0).copy()).cuda()
            for s in S.S]
    res = []
    for i, (s, T) in enumerate(zip(S.S, S.T)):
        check(l.td_gridnet_mask_dev(T.ctx, _p(M[i]), _p(OK[i]), s.c, 20, S.st()))
    for which in range(3):
        for i, (s, T) in enumerate(zip(S.S, S.T)):
            check(l.td_gridnet_deps_dev(T.ctx, _p(P[i]), _p(OUT[i]), s.c, -32768, S.st()))
        S.rounds(lambda i, h: check(l.td_gridnet_sweep_run_dev(S.T[i].ctx, which, _p(OK[i]), _p(dist[i]), _p(OUT[i]), S.S[i].c, 0, h, S.st())), [OUT])
        res.append(S.gather(OUT))
    for i, (s, T) in enumerate(zip(S.S, S.T)):
        check(l.td_gridnet_order_dev(T.ctx, _p(OUT[i]), _p(P[i]), _p(OK[i]), _p(G[i]), s.c, -32768, 0, S.st()))
    ref = td.gridnet_grid(p, mask=mask, thresh=20)
    assert_bits(res[0], ref[0], f"plen, {n} strips"); assert_bits(res[1], ref[1], f"tlen, {n} strips")
    assert_bits(S.gather(G), ref[2], f"gord, {n} strips")
    S.close()

    # the three D-infinity tools, on geographic per-row cell sizes
    x = cases["conc_and_trans_lim"]
    ang, q, dm, dg, tc, cs = x["ang"], x["q"], x["dm"], x["dg"], x["tc"], x["cs"]
    dxr, dyr = _geo_rows(ang.shape[0])
    S = Strips(ang.shape, n)
    A, Q, DM, DG, TC, CS = S.load(ang, torch.float32), S.load(q, torch.float32), S.load(dm, torch.float32), S.load(dg, torch.int16), \
        S.load(tc, torch.float32), S.load(cs, torch.float32)
    DX, DY = S.rows(dxr), S.rows(dyr)
    for s, T in zip(S.S, S.T):
        l.td_set_halo_cell_sizes_dev(T.ctx, dxr[s.row0 - 1] if s.has_top else 0.0, dyr[s.row0 - 1] if s.has_top else 0.0,
                                     dxr[s.row0 + s.ny] if s.has_bot else 0.0, dyr[s.row0 + s.ny] if s.has_bot else 0.0)
    OUT = S.empty(torch.float32)
    for i, (s, T) in enumerate(zip(S.S, S.T)):
        check(l.td_dinfdecayaccum_deps_dev(T.ctx, _p(A[i]), _p(OUT[i]), s.c, ANG_ND, _p(DX[i]), _p(DY[i]), S.st()))
    S.rounds(lambda i, h: check(l.td_dinfdecayaccum_sweep_run_dev(S.T[i].ctx, _p(A[i]), _p(DM[i]), _p(Q[i]), _p(OUT[i]), S.S[i].c, -9999.0, 0, _p(DX[i]), h,
                                                                  S.st())), [OUT])
    assert_bits(S.gather(OUT), td.dinfdecayaccum_grid(ang, dm, weights=q, contcheck=False, dxc=dxr, dyc=dyr), f"dsca -wg -nc, {n} strips")
    for i, (s, T) in enumerate(zip(S.S, S.T)):
        check(l.td_dinfconclimaccum_deps_dev(T.ctx, _p(A[i]), _p(OUT[i]), s.c, ANG_ND, _p(DX[i]), _p(DY[i]), S.st()))
    S.rounds(lambda i, h: check(l.td_dinfconclimaccum_sweep_run_dev(S.T[i].ctx, _p(A[i]), _p(DM[i]), _p(Q[i]), _p(DG[i]), _p(OUT[i]), S.S[i].c, -9999.0, -9999.0,
                                                                    2.5, 1, _p(DX[i]), h, S.st())), [OUT])
    assert_bits(S.gather(OUT), td.dinfconclimaccum_grid(ang, dm, q, dg, csol=2.5, dxc=dxr, dyc=dyr), f"ctpt, {n} strips")
    DEP, CO = S.empty(torch.float32), S.empty(torch.float32)
    for i, (s, T) in enumerate(zip(S.S, S.T)):
        check(l.td_dinftranslimaccum_deps_dev(T.ctx, _p(A[i]), _p(OUT[i]), _p(DEP[i]), _p(CO[i]), s.c, ANG_ND, _p(DX[i]), _p(DY[i]), S.st()))
    S.rounds(lambda i, h: check(l.td_dinftranslimaccum_sweep_run_dev(S.T[i].ctx, _p(A[i]), _p(Q[i]), _p(TC[i]), _p(CS[i]), _p(OUT[i]), _p(DEP[i]), _p(CO[i]),
                                                                     S.S[i].c, -9999.0, -9999.0, -9999.0, 1, _p(DX[i]), h, S.st())), [OUT, CO])
    rt, rd, rc = td.dinftranslimaccum_grid(ang, q, tc, cs=cs, dxc=dxr, dyc=dyr)
    assert_bits(S.gather(OUT), rt, f"tla -cs, {n} strips"); assert_bits(S.gather(DEP), rd, f"tdep -cs, {n} strips")
    assert_bits(S.gather(CO), rc, f"ctpt -cs, {n} strips")
    S.close()


# ---------------------------------------------------------------- executables
def _tool(gpus, tool, args, peer):
    env = dict(os.environ, TAUDEM_B200_GPUS=str(gpus))
    env.pop("TAUDEM_B200_PEER", None)
    if peer is not None:
        env["TAUDEM_B200_PEER"] = peer
    r = subprocess.run([os.path.join(BIN, tool)] + [str(a) for a in args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=600)
    assert r.returncode == 0 and "error" not in r.stdout.lower(), r.stdout
    assert f"Processors: {gpus}" in r.stdout, r.stdout
    return r.stdout


def _runs(d):
    """(tool, name, args, outputs [(flag, name, dtype)], reference outputs) of the option matrix of sibling_cases.py without -o"""
    q = lambda n: str(d / n)
    return [
        ("d8flowpathextremeup", "ssa", ["-p", q("p.tif"), "-sa", q("sa.tif")], [("-ssa", "ssa", np.float32)]),
        ("d8flowpathextremeup", "ssamin", ["-p", q("p.tif"), "-sa", q("fel.tif"), "-min", "-nc"], [("-ssa", "ssa", np.float32)]),
        ("gridnet", "gn", ["-p", q("gp.tif")], [("-plen", "plen", np.float32), ("-tlen", "tlen", np.float32), ("-gord", "gord", np.int16)]),
        ("gridnet", "gnm", ["-p", q("gp.tif"), "-mask", q("mask.tif"), "-thresh", "20"],
         [("-plen", "plen", np.float32), ("-tlen", "tlen", np.float32), ("-gord", "gord", np.int16)]),
        ("dinfdecayaccum", "dsca", ["-ang", q("dang.tif"), "-dm", q("ddm.tif")], [("-dsca", "dsca", np.float32)]),
        ("dinfdecayaccum", "dscaw", ["-ang", q("dang.tif"), "-dm", q("ddm.tif"), "-wg", q("dw.tif"), "-nc"], [("-dsca", "dsca", np.float32)]),
        ("dinfconclimaccum", "ctpt", ["-ang", q("ang.tif"), "-dm", q("dm.tif"), "-q", q("q.tif"), "-dg", q("dg.tif"), "-csol", "2.5"],
         [("-ctpt", "ctpt", np.float32)]),
        ("dinfconclimaccum", "ctptnc", ["-ang", q("ang.tif"), "-dm", q("dm.tif"), "-q", q("q.tif"), "-dg", q("dg.tif"), "-nc"], [("-ctpt", "ctpt", np.float32)]),
    ] + [("dinftranslimaccum", f"tl{i}", ["-ang", q("ang.tif"), "-tsup", q("q.tif"), "-tc", q("tc.tif")] + extra,
          [("-tla", "tla", np.float32), ("-tdep", "tdep", np.float32)] + ([("-ctpt", "ctpt", np.float32)] if "-cs" in extra else []))
         for i, extra in enumerate(([], ["-nc"], ["-cs", q("cs.tif")], ["-cs", q("cs.tif"), "-nc"]))]


def _write_inputs(cases, d):
    x = cases["flowpathextremeup"]
    td.write_raster(str(d / "p.tif"), x["p"], -32768); td.write_raster(str(d / "sa.tif"), x["sa"], -9999.0); td.write_raster(str(d / "fel.tif"), x["fel"], -9999.0)
    x = cases["gridnet"]
    td.write_raster(str(d / "gp.tif"), x["p"], -32768); td.write_raster(str(d / "mask.tif"), x["mask"], -2147483648)
    x = cases["dinfdecayaccum"]
    td.write_raster(str(d / "dang.tif"), x["ang"], ANG_ND); td.write_raster(str(d / "ddm.tif"), x["dm"], -9999.0); td.write_raster(str(d / "dw.tif"), x["w"], -9999.0)
    x = cases["conc_and_trans_lim"]
    td.write_raster(str(d / "ang.tif"), x["ang"], ANG_ND)
    for n in ("q", "dm", "tc", "cs"):
        td.write_raster(str(d / f"{n}.tif"), x[n], -9999.0)
    td.write_raster(str(d / "dg.tif"), x["dg"], -32768)


def _reference(cases, name):
    """the C restatement's outputs of one run of _runs"""
    a, g, dd, c = cases["flowpathextremeup"], cases["gridnet"], cases["dinfdecayaccum"], cases["conc_and_trans_lim"]
    if name == "ssa":
        return [port.d8flowpathextremeup(a["p"], a["sa"])]
    if name == "ssamin":
        return [port.d8flowpathextremeup(a["p"], a["fel"], usemax=False, contcheck=False)]
    if name == "gn":
        return list(port.gridnet(g["p"]))
    if name == "gnm":
        return list(port.gridnet(g["p"], mask=g["mask"], thresh=20))
    if name == "dsca":
        return [port.dinfdecayaccum(dd["ang"], dd["dm"])]
    if name == "dscaw":
        return [port.dinfdecayaccum(dd["ang"], dd["dm"], weights=dd["w"], contcheck=False)]
    if name == "ctpt":
        return [port.dinfconclimaccum(c["ang"], c["dm"], c["q"], c["dg"], csol=2.5)]
    if name == "ctptnc":
        return [port.dinfconclimaccum(c["ang"], c["dm"], c["q"], c["dg"], contcheck=False)]
    i = int(name[2:])
    out = port.dinftranslimaccum(c["ang"], c["q"], c["tc"], cs=c["cs"] if i >= 2 else None, contcheck=i % 2 == 0)
    return [o for o in out if o is not None]


def _matrix(cases, d, peer, counts):
    _write_inputs(cases, d)
    for tool, name, args, outs in _runs(d):
        files = lambda n: sum(([flag, str(d / f"{name}_{o}_{n}.tif")] for flag, o, _ in outs), [])
        env_one = dict(os.environ); env_one.pop("TAUDEM_B200_GPUS", None)
        r = subprocess.run([os.path.join(BIN, tool)] + args + files(1), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env_one, timeout=600)
        assert r.returncode == 0, r.stdout
        one = [td.read_raster(str(d / f"{name}_{o}_1.tif"), dt) for _, o, dt in outs]
        for got, ref, (_, o, _) in zip(one, _reference(cases, name), outs):
            assert_bits(got, ref, f"{tool} {name} {o}: one GPU vs the C restatement")
        for n in counts:
            _tool(n, tool, args + files(n), peer)
            for (_, o, dt), ref in zip(outs, one):
                assert_bits(td.read_raster(str(d / f"{name}_{o}_{n}.tif"), dt), ref, f"{tool} {name} {o} on {n} ranks, peer={peer}")


def test_executables_in_rounds(cases, tmp_path):
    """TAUDEM_B200_GPUS=2 and 3 with TAUDEM_B200_PEER=0 (ranks may share a device): bit-identical to one GPU and to the restatement"""
    _matrix(cases, tmp_path, "0", (2, 3))


def test_executables_in_peer_mode(cases, tmp_path):
    """one device per rank, the kernels delivering over NVLink (TAUDEM_B200_PEER unset: peer mode where every pair of neighbours can)"""
    counts = [n for n in (2, 3) if td.device_count() >= n]
    if not counts:
        pytest.skip(f"peer mode needs one device per rank: {td.device_count()} device(s)")
    _matrix(cases, tmp_path, None, counts)


def test_executables_on_a_geographic_raster(cases, tmp_path):
    """rows of different cell sizes on both sides of every strip boundary: dinfdecayaccum -wg and dinftranslimaccum -cs"""
    d = tmp_path
    c = cases["conc_and_trans_lim"]
    ang = c["ang"]
    write_geographic_dem(str(d / "geo.tif"), np.zeros(ang.shape, np.float32))
    like = str(d / "geo.tif")
    td.write_raster(str(d / "ang.tif"), ang, ANG_ND, like=like)
    for n in ("q", "dm", "tc", "cs"):
        td.write_raster(str(d / f"{n}.tif"), c[n], -9999.0, like=like)
    ny, nx = ang.shape
    dxc, dyc = np.empty(ny), np.empty(ny)
    assert lib().td_raster_cell_sizes(str(d / "ang.tif").encode(), dxc.ctypes.data_as(C.c_void_p), dyc.ctypes.data_as(C.c_void_p), ny) == 0
    assert dxc.min() < dxc.max()
    runs = [("dinfdecayaccum", ["-ang", "ang.tif", "-dm", "dm.tif", "-wg", "q.tif"], ["-dsca"],
             [port.dinfdecayaccum(ang, c["dm"], weights=c["q"], dxc=dxc, dyc=dyc)]),
            ("dinftranslimaccum", ["-ang", "ang.tif", "-tsup", "q.tif", "-tc", "tc.tif", "-cs", "cs.tif"], ["-tla", "-tdep", "-ctpt"],
             list(port.dinftranslimaccum(ang, c["q"], c["tc"], cs=c["cs"], dxc=dxc, dyc=dyc)))]
    for tool, args, flags, refs in runs:
        args = [str(d / a) if a.endswith(".tif") else a for a in args]
        for n in (2, 3):
            _tool(n, tool, args + sum(([f, str(d / f"{tool}{f}_{n}.tif")] for f in flags), []), "0")
            for f, ref in zip(flags, refs):
                assert_bits(td.read_raster(str(d / f"{tool}{f}_{n}.tif")), ref, f"{tool} {f} geographic on {n} ranks")
