"""The inputs of the sibling sweep tools' GPU tests (tests/test_gpu_parity.py) and the reference calls those tests compare
against.  The CPU suite (tests/test_cpu.py) replays the same calls through tests/reference.py, so every stored output they
use is reproduced by the C restatement without a GPU.

Each case returns (x, calls): x the input rasters (and the outlet cells and shapefile), calls a list of
(label, tool, args, kwargs) for reference.RefPipeline, in the order the GPU test makes them (the last call's input files are
the ones the test then runs our executable on).
"""
import numpy as np

import port
from taudem_b200 import synth
from util import write_point_shapefile


def outlets(acc, workdir, dx=30.0, dy=30.0):
    """Three outlets at the cells with the 1st, 40th and 700th largest accumulation: (cols, rows) and a point shapefile of them"""
    ny, nx = acc.shape
    order = np.argsort(acc.ravel())
    cells = [int(order[-1]), int(order[-40]), int(order[-700])]
    cols = [c % nx for c in cells]; rows = [c // nx for c in cells]
    shp = str(workdir / "outlets.shp")
    write_point_shapefile(shp, [(c + 0.5) * dx for c in cols], [dy * ny - (r + 0.5) * dy for r in rows])
    return cols, rows, shp


def flowpathextremeup(workdir):
    dem = synth.punch_holes(synth.gen_dem(330, 410, hurst=0.8, tilt=1.0, seed=41))
    fel = port.pitremove(dem); p, sd8 = port.d8flowdir(fel)
    sa = np.where(sd8 < 0, np.float32(0.0), sd8).astype(np.float32)           # "largest slope upstream"
    cols, rows, shp = outlets(port.aread8(p, contcheck=False), workdir)
    x = dict(p=p, sa=sa, fel=fel, cols=cols, rows=rows, shp=shp)
    return x, [("ssa max", "d8flowpathextremeup", (p, sa), {}),
               ("ssa min -nc", "d8flowpathextremeup", (p, fel), dict(usemax=False, contcheck=False)),
               ("ssa max -o", "d8flowpathextremeup", (p, sa), dict(outlets=shp))]


def gridnet(workdir):
    dem = synth.punch_holes(synth.gen_dem(330, 410, hurst=0.8, tilt=1.0, seed=47))
    fel = port.pitremove(dem); p, _ = port.d8flowdir(fel)
    ad8 = port.aread8(p, contcheck=False)
    mask = np.where(ad8 >= 0, ad8, 0).astype(np.int32)
    cols, rows, shp = outlets(ad8, workdir)
    x = dict(p=p, mask=mask, cols=cols, rows=rows, shp=shp)
    return x, [("", "gridnet", (p,), {}),
               ("-mask -thresh 20", "gridnet", (p,), dict(mask=mask, thresh=20)),
               ("-o", "gridnet", (p,), dict(outlets=shp)),
               ("-o -mask", "gridnet", (p,), dict(mask=mask, thresh=20, outlets=shp))]


def dinfdecayaccum(workdir):
    dem = synth.punch_holes(synth.gen_dem(330, 410, hurst=0.8, tilt=1.0, seed=43))
    fel = port.pitremove(dem); ang, _ = port.dinfflowdir(fel)
    rng = np.random.default_rng(9)
    dm = rng.uniform(0.3, 1.0, ang.shape).astype(np.float32)
    dm[rng.random(ang.shape) < 0.001] = -9999.0
    w = rng.uniform(0.0, 2.0, ang.shape).astype(np.float32)
    cols, rows, shp = outlets(port.areadinf(ang, contcheck=False), workdir)
    x = dict(ang=ang, dm=dm, w=w, cols=cols, rows=rows, shp=shp)
    return x, [("dsca", "dinfdecayaccum", (ang, dm), {}),
               ("dsca -wg -nc", "dinfdecayaccum", (ang, dm), dict(weights=w, contcheck=False)),
               ("dsca -o", "dinfdecayaccum", (ang, dm), dict(outlets=shp))]


def sibling_inputs(shape, seed):
    """q (= tsup), dm, dg, tc, cs of the concentration / transport limited accumulations, with a few nodata cells each"""
    rng = np.random.default_rng(seed)
    q = rng.uniform(0.5, 3.0, shape).astype(np.float32)
    q[rng.random(shape) < 0.001] = -9999.0
    q[rng.random(shape) < 0.001] = 0.0
    dm = rng.uniform(0.2, 1.0, shape).astype(np.float32)
    dm[rng.random(shape) < 0.0005] = -9999.0
    dg = (rng.random(shape) < 0.02).astype(np.int16)
    tc = rng.uniform(0.0, 8.0, shape).astype(np.float32)
    tc[rng.random(shape) < 0.0005] = -9999.0
    cs = rng.uniform(0.0, 2.0, shape).astype(np.float32)
    cs[rng.random(shape) < 0.0005] = -9999.0
    return q, dm, dg, tc, cs


def conc_and_trans_lim(workdir):
    dem = synth.punch_holes(synth.gen_dem(340, 430, hurst=0.8, tilt=1.0, seed=47))
    fel = port.pitremove(dem); ang, _ = port.dinfflowdir(fel)
    q, dm, dg, tc, cs = sibling_inputs(ang.shape, 11)
    cols, rows, shp = outlets(port.areadinf(ang, contcheck=False), workdir)
    x = dict(ang=ang, q=q, dm=dm, dg=dg, tc=tc, cs=cs, cols=cols, rows=rows, shp=shp)
    tsup = q
    calls = [("ctpt", "dinfconclimaccum", (ang, dm, q, dg), dict(csol=2.5)),
             ("ctpt -nc", "dinfconclimaccum", (ang, dm, q, dg), dict(contcheck=False)),
             ("ctpt -o", "dinfconclimaccum", (ang, dm, q, dg), dict(csol=0.75, contcheck=False, outlets=shp))]
    for kw in ({}, {"contcheck": False}, {"cs": cs}, {"cs": cs, "contcheck": False}):
        calls.append((f"translim {sorted(kw)}", "dinftranslimaccum", (ang, tsup, tc), kw))
    calls.append(("translim -cs -nc -o", "dinftranslimaccum", (ang, tsup, tc), dict(cs=cs, contcheck=False, outlets=shp)))
    return x, calls


CASES = (flowpathextremeup, gridnet, dinfdecayaccum, conc_and_trans_lim)
