"""slopeavedown end to end on a synthetic n x n DEM (filled and given D8 directions on the device): td_slopeavedown_host's compute
time at dn = 50 and dx = dy = 30, 10 and 1 (niter = 2, 6 and 51), split into the D8 sweep that marks the processed cells
(td_aread8_host on the same directions) and the passes (the rest), best of several runs.
   python scripts/slopeavedown_bench.py [n=16384] [reps=3]"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import taudem_b200 as td  # noqa: E402
from taudem_b200.device import DeviceStrip, Tools  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    T = Tools(); s = DeviceStrip(n, n); dxc = s.rows(30.0)
    fel = T.pitremove(s, T.gen_dem(s, hurst=0.8, tilt=1.0))
    p, _, _ = T.d8_slopes(s, fel, dxc, dxc)
    T.d8_flats(s, fel.clone(), p, dxc, dxc)
    fel_h = s.owned(fel).cpu().numpy().copy(); p_h = s.owned(p).cpu().numpy().copy()
    del fel, p; T.close(); torch.cuda.empty_cache()
    ad8 = np.empty((n, n), np.float32)
    sweep = []
    for _ in range(reps + 1):
        td.aread8_grid(p_h, out=ad8, contcheck=False)
        sweep.append(td.last_compute_seconds() * 1e3)
    sweep = min(sweep[1:])
    out = {"n": n, "d8_sweep_ms": round(sweep, 2), "runs": []}
    for d in (30.0, 10.0, 1.0):
        ts = []
        for _ in range(reps + 1):
            slpd = td.slopeavedown_grid(fel_h, p_h, dn=50.0, dx=d, dy=d)
            ts.append(td.last_compute_seconds() * 1e3)
        best = min(ts[1:])
        niter = int(50.0 / d + 1)
        out["runs"].append({"dx": d, "niter": niter, "total_ms": round(best, 2), "passes_ms": round(best - sweep, 2),
                            "ms_per_pass": round((best - sweep) / niter, 3), "cells_set": int((slpd > -3.0e38).sum())})
        print(out["runs"][-1])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
