"""d8hdisttostrm and d8vdisttostrm against td_aread8_host on the same directions: a synthetic n x n DEM, filled, its D8 directions,
and src = its D8 contributing area, at a low and a high stream threshold.  Every call reports the device time after its uploads
(td_last_compute_seconds); the calls alternate, the first round is a warm-up, and each result is the median [min .. max] of the rest,
with the card's name and power limit read in the same process.  Also reported per threshold: the stream cells, the BFS level count
L (td_disttostrm_last_levels), the kernel launches of one call (about L: one per level, plus a batch's tail of empty levels) and the
levels per host read-back.
   python scripts/disttostrm_bench.py [n=16384] [reps=5] [low=100] [high=10000]"""
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

BATCH = 64      # DTS_BATCH in taudem_b200/csrc/kernels.h


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip()


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    threshs = [int(sys.argv[3]) if len(sys.argv) > 3 else 100, int(sys.argv[4]) if len(sys.argv) > 4 else 10000]
    T = Tools(); s = DeviceStrip(n, n); dxc = s.rows(30.0)
    dem = T.gen_dem(s, hurst=0.8, tilt=1.0)
    fel = T.pitremove(s, dem.clone())
    p, _, _ = T.d8_slopes(s, fel, dxc, dxc)
    T.d8_flats(s, fel.clone(), p, dxc, dxc)
    p_h = s.owned(p).cpu().numpy().copy(); fel_h = s.owned(fel).cpu().numpy().copy()
    del dem, fel, p; T.close(); torch.cuda.empty_cache()
    ad8 = np.empty((n, n), np.float32)
    td.aread8_grid(p_h, out=ad8, contcheck=False)
    src = np.where(ad8 < 0, -1, ad8).astype(np.int32)
    rows = np.full(n, 30.0)
    t = {"aread8": []}
    info = {}
    for th in threshs:
        t[f"d8hdisttostrm thresh={th}"] = []
        t[f"d8vdisttostrm thresh={th}"] = []
        info[th] = {"stream_cells": int((src >= th).sum())}
    for _ in range(reps + 1):
        td.aread8_grid(p_h, out=ad8, contcheck=False)
        t["aread8"].append(td.last_compute_seconds() * 1e3)
        for th in threshs:
            for tool in ("d8hdisttostrm", "d8vdisttostrm"):
                td.reset_launch_count()
                if tool == "d8hdisttostrm":
                    td.d8hdisttostrm_grid(p_h, src, thresh=th, dxc=rows, dyc=rows, src_nodata=-1)
                else:
                    td.d8vdisttostrm_grid(p_h, fel_h, src, thresh=th, src_nodata=-1)
                t[f"{tool} thresh={th}"].append(td.last_compute_seconds() * 1e3)
                L = int(td.lib().td_disttostrm_last_levels())
                info[th].update({"L": L, "launches": int(td.launch_count()), "levels_per_readback": round(L / max(1, -(-L // BATCH)), 1)})
    out = {"n": n, "card": card(), "reps": reps, "thresholds": info}
    for k, v in t.items():
        v = v[1:]
        out[k] = f"{statistics.median(v):.1f} [{min(v):.1f} .. {max(v):.1f}] ms"
    for th in threshs:
        for tool in ("d8hdisttostrm", "d8vdisttostrm"):
            out[f"{tool} thresh={th} / aread8"] = round(statistics.median(t[f"{tool} thresh={th}"][1:]) / statistics.median(t["aread8"][1:]), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
