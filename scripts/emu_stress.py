"""Randomised stress of the emulated kernels (tests/emu): random grid sizes, flats, nodata holes, strip counts, the warp-per-tile
sweep (single strip and exchange rounds) and strip flats against the oracle; per seed two of the sibling algebras 1-9 (algebra
seed % 9 + 1 and a random one) on random value grids with nodata, zero and negative values, against the C restatement.
python scripts/emu_stress.py [first_seed] [n_seeds] [seconds]"""
import sys, os, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import ctypes as C
import numpy as np, test_emu
from taudem_b200 import synth
from oracle import port


def sibling_values(rng, shape):
    """value grids of the sibling algebras with nodata (-9999), zero and negative values"""
    def vals(lo, hi):
        v = rng.uniform(lo, hi, shape).astype(np.float32)
        v[rng.random(shape) < 0.04] = 0.0
        v[rng.random(shape) < 0.02] = -9999.0
        return v
    return dict(sa=vals(-50.0, 50.0), dm=vals(-0.2, 1.2), w=vals(-0.5, 2.0), q=vals(-0.5, 3.0), tc=vals(-0.5, 6.0), cs=vals(-0.2, 2.0),
                dg=(rng.random(shape) < 0.05).astype(np.int16), mask=rng.integers(-1, 4, shape).astype(np.int32))


def run_algebra(lib, alg, p, ang, v, contcheck, seed, dx=30.0, dy=30.0, usew=False):
    """Algebra `alg` (1-9) of k_sweep_warp on the emulated thread model (single strip), and the C restatement's result:
    [(name, emulated, restated)].  v: sibling_values; gridnet (4-6) with v["mask"] >= 1 as its mask."""
    ny, nx = ang.shape if p is None else p.shape
    name = f"algebra {alg} contcheck={contcheck} usew={usew}"
    try:
        if alg in (1, 2):
            return [(name, test_emu._run(lib, False, 9 + alg, 0, p, v["sa"], contcheck, seed, dx=dx, dy=dy),
                     port.d8flowpathextremeup(p, v["sa"], usemax=alg == 1, contcheck=contcheck))]
        if alg in (4, 5, 6):
            ok = np.ascontiguousarray((v["mask"] >= 1).astype(np.float32))
            lib.emu_set_dm(ok.ctypes.data, C.c_float(0.0))
            res, d = np.empty((ny, nx), np.float32), np.ascontiguousarray(p)
            assert lib.emu_sweep(0, 9 + alg, 0, d.ctypes.data, res.ctypes.data, None, nx, ny, -32768.0, 0, 0, -1.0, dx, dy, seed, 1, None, None, None, -1) == 0
            ref = port.gridnet(p, mask=v["mask"], thresh=1, dx=dx, dy=dy)[alg - 4]
            return [(name, res.astype(np.int16) if alg == 6 else res, ref)]
        kw = dict(dx=dx, dy=dy, contcheck=contcheck)
        if alg == 3:
            dm = np.ascontiguousarray(v["dm"])
            lib.emu_set_dm(dm.ctypes.data, C.c_float(-9999.0))
            w = v["w"] if usew else None
            return [(name, test_emu._run(lib, True, 12, 0, ang, w, contcheck, seed, dx=dx, dy=dy), port.dinfdecayaccum(ang, dm, weights=w, **kw))]
        if alg == 7:
            dm, dg = np.ascontiguousarray(v["dm"]), np.ascontiguousarray(v["dg"])
            lib.emu_set_dm(dm.ctypes.data, C.c_float(-9999.0))
            lib.emu_set_extra(dg.ctypes.data, C.c_float(1.5), None, C.c_float(0.0), None, None)
            return [(name, test_emu._run(lib, True, 16, 0, ang, v["q"], contcheck, seed, dx=dx, dy=dy), port.dinfconclimaccum(ang, dm, v["q"], dg, csol=1.5, **kw))]
        tc, cs = np.ascontiguousarray(v["tc"]), np.ascontiguousarray(v["cs"])
        dep, cout = np.empty((ny, nx), np.float32), np.empty((ny, nx), np.float32)
        lib.emu_set_dm(tc.ctypes.data, C.c_float(-9999.0))
        if alg == 8:
            lib.emu_set_extra(None, C.c_float(0.0), None, C.c_float(0.0), dep.ctypes.data, None)
        else:
            lib.emu_set_extra(None, C.c_float(0.0), cs.ctypes.data, C.c_float(-9999.0), dep.ctypes.data, cout.ctypes.data)
        tla = test_emu._run(lib, True, 9 + alg, 0, ang, v["q"], contcheck, seed, dx=dx, dy=dy)
        rt, rd, rc = port.dinftranslimaccum(ang, v["q"], tc, cs=cs if alg == 9 else None, **kw)
        return [(name + " tla", tla, rt), (name + " tdep", dep, rd)] + ([(name + " ctpt", cout, rc)] if alg == 9 else [])
    finally:
        lib.emu_set_dm(None, C.c_float(0.0))
        lib.emu_set_extra(None, C.c_float(0.0), None, C.c_float(0.0), None, None)


lib=test_emu._build()
t0=time.time(); bad=0; n=0; algruns=[0]*10
first = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
count = int(sys.argv[2]) if len(sys.argv) > 2 else 100
budget = float(sys.argv[3]) if len(sys.argv) > 3 else 1500.0
for seed in range(first, first + count):
    rng=np.random.default_rng(seed)
    ny=int(rng.integers(8,200)); nx=int(rng.integers(5,300))
    dem=synth.punch_holes(synth.gen_dem(ny,nx,hurst=float(rng.choice([0.6,0.8])),tilt=float(rng.choice([0.0,1.0,4.0])),seed=seed),seed=seed)
    if rng.random()<0.4:
        q=(dem.max()-dem.min())/8; m=dem!=-9999.0; dem=np.where(m,(np.round(dem/q)*q),dem).astype(np.float32)
    fel=port.pitremove(dem); p,_=port.d8flowdir(fel); ang,_=port.dinfflowdir(fel)
    w=synth.gen_weights(ny,nx,seed=seed)
    ad8=port.aread8(p); sca=port.areadinf(ang); ad8w=port.aread8(p,weights=w,contcheck=False); scaw=port.areadinf(ang,weights=w,contcheck=False)
    strips=int(rng.integers(1,4))
    checks=[('ad8',test_emu._run(lib,False,0,0,p,None,True,seed,strips),ad8),
            ('sca',test_emu._run(lib,True,0,0,ang,None,True,seed+1,strips),sca),
            ('ad8w',test_emu._run(lib,False,0,0,p,w,False,seed+2,strips),ad8w),
            ('scaw',test_emu._run(lib,True,0,0,ang,w,False,seed+3,strips),scaw),
            ('ad8 1 strip',test_emu._run(lib,False,0,0,p,None,True,seed+4),ad8),
            ('sca 1 strip',test_emu._run(lib,True,0,0,ang,None,True,seed+5),sca)]
    # flats over strips
    p0,_=port.d8flowdir(fel,flats=False); a0,_=port.dinfflowdir(fel,flats=False)
    fs=int(rng.integers(1,5))
    if ny//fs>=1:
        checks+= [('p strips',test_emu._flats(lib,False,fel,p0,fs,seed+6)[0],p),('ang strips',test_emu._flats(lib,True,fel,a0,fs,seed+7)[0],ang)]
    # sibling algebras (single strip), cells square or oblong
    ra=np.random.default_rng(seed+1000003)
    v=sibling_values(ra,(ny,nx)); sdx,sdy=((30.0,30.0),(20.0,30.0))[int(ra.integers(0,2))]
    for alg in sorted({seed%9+1, int(ra.integers(1,10))}):
        algruns[alg]+=1
        checks+=run_algebra(lib,alg,p,ang,v,bool(ra.integers(0,2)),seed+8+alg,sdx,sdy,usew=bool(ra.integers(0,2)))
    for name,a,b in checks:
        n+=1
        if not np.array_equal(np.ascontiguousarray(a).view(np.int32 if a.dtype==np.float32 else a.dtype), np.ascontiguousarray(b).view(np.int32 if b.dtype==np.float32 else b.dtype)):
            bad+=1; print('MISMATCH',seed,name,ny,nx,strips,flush=True)
    if time.time()-t0>budget: break
print('checks',n,'bad',bad,'seeds up to',seed,'time',round(time.time()-t0),'algebra runs',','.join(map(str,algruns[1:])))
sys.exit(1 if bad else 0)
