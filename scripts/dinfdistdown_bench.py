"""dinfdistdown (ave h, ave v, ave p) against td_areadinf_host and td_d8hdisttostrm_host on the same DEM: a synthetic n x n DEM,
filled, its D8 and D-infinity directions, and src = its D8 contributing area >= thresh (the HAND workflow's stream raster).  Every
call reports the device time after its uploads (td_last_compute_seconds); the calls alternate, the first round is a warm-up, and each
result is the median [min .. max] of the rest, with the card's name and power limit read in the same process.  Also reported: the
stream cells, dinfdistdown's level count L (td_dinfdistdown_last_levels), the kernel launches of one call (about L: one per level,
plus a batch's tail of empty levels) and the cells that get a value.
   python scripts/dinfdistdown_bench.py [n=16384] [reps=5] [thresh=1000]"""
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
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    thresh = int(sys.argv[3]) if len(sys.argv) > 3 else 1000
    T = Tools(); s = DeviceStrip(n, n); dxc = s.rows(30.0)
    dem = T.gen_dem(s, hurst=0.8, tilt=1.0)
    fel = T.pitremove(s, dem.clone())
    p, _, _ = T.d8_slopes(s, fel, dxc, dxc)
    T.d8_flats(s, fel.clone(), p, dxc, dxc)
    ang, _, _ = T.dinf_slopes(s, fel, dxc, dxc)
    T.dinf_flats(s, fel.clone(), ang, dxc, dxc)
    p_h = s.owned(p).cpu().numpy().copy(); fel_h = s.owned(fel).cpu().numpy().copy(); ang_h = s.owned(ang).cpu().numpy().copy()
    del dem, fel, p, ang; T.close(); torch.cuda.empty_cache()
    ad8 = np.empty((n, n), np.float32)
    td.aread8_grid(p_h, out=ad8, contcheck=False)
    src32 = np.where(ad8 >= thresh, 1, 0).astype(np.int32)
    src16 = src32.astype(np.int16)
    del ad8
    sca = np.empty((n, n), np.float32)
    rows = np.full(n, 30.0)
    calls = {
        "areadinf": lambda: td.areadinf_grid(ang_h, out=sca),
        "d8hdisttostrm": lambda: td.d8hdisttostrm_grid(p_h, src32, thresh=1, dxc=rows, dyc=rows, src_nodata=-1),
    }
    for m in ("h", "v", "p"):
        calls[f"dinfdistdown ave {m}"] = (lambda m=m: td.dinfdistdown_grid(ang_h, src16, fel=fel_h, method=m, stat="ave"))
    t = {k: [] for k in calls}
    info = {"stream_cells": int(src16.sum())}
    for _ in range(reps + 1):
        for k, f in calls.items():
            td.reset_launch_count()
            out = f()
            t[k].append(td.last_compute_seconds() * 1e3)
            if k.startswith("dinfdistdown"):
                info[k] = {"L": int(td.lib().td_dinfdistdown_last_levels()), "launches": int(td.launch_count()),
                           "cells_with_a_value": int((out != td.api.MISSINGFLOAT).sum())}
    res = {"n": n, "card": card(), "reps": reps, "thresh": thresh, "info": info}
    for k, v in t.items():
        v = v[1:]
        res[k] = f"{statistics.median(v):.1f} [{min(v):.1f} .. {max(v):.1f}] ms"
    for m in ("h", "v", "p"):
        res[f"dinfdistdown ave {m} / areadinf"] = round(statistics.median(t[f"dinfdistdown ave {m}"][1:]) / statistics.median(t["areadinf"][1:]), 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
