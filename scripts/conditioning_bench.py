"""flowdircond and retlimflow against their sibling sweeps on the same directions: td_flowdircond_host (algebra 11) against
td_aread8_host with z as weights, on a synthetic n x n DEM whose D8 directions come from the filled DEM and whose raw elevations
are conditioned; td_retlimflow_host (algebra 12) against td_areadinf_host with wg as weights, on the D-infinity angles of the same
filled DEM (wg uniform in [0, 1), rc in [0, 0.5)).  Both calls report the
device time from the dependency stencil to the end of the sweep (td_last_compute_seconds); the runs alternate, the first of each is
a warm-up, and the result is the median [min .. max] of the rest, with the card's name and power limit read in the same process.
   python scripts/conditioning_bench.py [n=16384] [reps=7]"""
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import taudem_b200 as td  # noqa: E402
from taudem_b200.device import DeviceStrip, Tools  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip()


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 7
    T = Tools(); s = DeviceStrip(n, n); dxc = s.rows(30.0)
    dem = T.gen_dem(s, hurst=0.8, tilt=1.0)
    fel = T.pitremove(s, dem.clone())
    p, _, _ = T.d8_slopes(s, fel, dxc, dxc)
    T.d8_flats(s, fel.clone(), p, dxc, dxc)
    z_h = s.owned(dem).cpu().numpy().copy(); p_h = s.owned(p).cpu().numpy().copy()
    fel_h = s.owned(fel).cpu().numpy().copy()
    del dem, fel, p; T.close(); torch.cuda.empty_cache()
    ang_h, _ = td.dinfflowdir_grid(fel_h)
    ad8 = np.empty((n, n), np.float32)
    t = {"aread8 -wg": [], "flowdircond": [], "areadinf -wg": [], "retlimflow": []}
    rng = np.random.default_rng(1)
    wg = rng.random((n, n), dtype=np.float32); rc = (rng.random((n, n), dtype=np.float32) * np.float32(0.5))
    sca = np.empty((n, n), np.float32)
    for _ in range(reps + 1):
        td.aread8_grid(p_h, weights=z_h, out=ad8, contcheck=False)
        t["aread8 -wg"].append(td.last_compute_seconds() * 1e3)
        zfdc = td.flowdircond_grid(p_h, z_h)
        t["flowdircond"].append(td.last_compute_seconds() * 1e3)
        td.areadinf_grid(ang_h, weights=wg, out=sca, contcheck=False)
        t["areadinf -wg"].append(td.last_compute_seconds() * 1e3)
        td.retlimflow_grid(ang_h, wg, rc)
        t["retlimflow"].append(td.last_compute_seconds() * 1e3)
    out = {"n": n, "card": card(), "reps": reps, "cells_lowered": int((zfdc < z_h).sum())}
    for k, v in t.items():
        v = v[1:]
        out[k] = f"{statistics.median(v):.1f} [{min(v):.1f} .. {max(v):.1f}] ms"
    out["flowdircond / aread8 -wg"] = round(statistics.median(t["flowdircond"][1:]) / statistics.median(t["aread8 -wg"][1:]), 3)
    out["retlimflow / areadinf -wg"] = round(statistics.median(t["retlimflow"][1:]) / statistics.median(t["areadinf -wg"][1:]), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
