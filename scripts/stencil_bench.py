"""CUDA-event timings of the stencil / streaming kernels of the path (SURVEY.md 8(d): the kernels the 70 % HBM target names)
on a synthetic DEM: best and median of several launches, algorithmic bytes per cell, fraction of the measured HBM peak.
   python scripts/stencil_bench.py [n=16384] [reps=7]"""
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from taudem_b200.device import DeviceStrip, Tools, _p  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 7
    only = set(sys.argv[3].split(",")) if len(sys.argv) > 3 else None        # e.g. k_deps_dinf,k_deps_d8
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        peak = 6650.0
    T = Tools(); s = DeviceStrip(n, n); dxc, dyc = s.rows(30.0), s.rows(30.0)
    mc = n * n / 1e6
    out = {}

    def run(name, bytes_per_cell, fn):
        if only is not None and name.split(" ")[0] not in only:
            fn()                                 # later kernels need its outputs
            torch.cuda.synchronize()
            return
        ts = []
        for _ in range(reps + 1):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize(); a.record(); fn(); b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ts = sorted(ts[1:])                      # the first launch pays module load / tensor map / occupancy query
        best, med = ts[0], ts[len(ts) // 2]
        out[name] = {"ms_best": round(best, 3), "ms_median": round(med, 3), "alg_B_per_cell": bytes_per_cell,
                     "GB_per_s": round(bytes_per_cell * mc / med, 1), "frac_of_hbm_peak": round(bytes_per_cell * mc / med / peak, 3),
                     "frac_of_3350_gbs": round(bytes_per_cell * mc / med / 3350.0, 3)}
        print(f"{name:18s} best {best:8.3f} ms  median {med:8.3f} ms  {bytes_per_cell:2d} B/cell  {bytes_per_cell * mc / med:7.1f} GB/s  {100 * bytes_per_cell * mc / med / peak:5.1f} % of {peak:.0f} GB/s")

    dem = T.gen_dem(s, hurst=0.8, tilt=1.0)
    w = s.empty(torch.float32)
    run("k_fill_init", 8, lambda: T.l.td_flood_init_dev(T.ctx, _p(dem), None, _p(w), s.c, C.c_float(-9999.0), 0, T._stream()))
    fel = T.pitremove(s, dem)
    del dem, w
    p = s.empty(torch.int16); sd8 = s.empty(torch.float32)
    run("k_d8_stencil", 10, lambda: T.d8_slopes(s, fel, dxc, dyc, p=p, sd8=sd8))
    ang = s.empty(torch.float32); slp = s.empty(torch.float32)
    run("k_dinf_stencil", 12, lambda: T.dinf_slopes(s, fel, dxc, dyc, ang=ang, slp=slp))
    T.d8_flats(s, fel.clone(), p, dxc, dyc)
    felw = fel.clone(); T.dinf_flats(s, felw, ang, dxc, dyc); del felw
    ad8 = s.empty(torch.float32)
    run("k_deps_d8", 2, lambda: T.aread8_deps(s, p, ad8))
    run("k_deps_d8 (+7 scratch)", 9, lambda: T.aread8_deps(s, p, ad8))
    sca = s.empty(torch.float32)
    run("k_deps_dinf", 4, lambda: T.areadinf_deps(s, ang, sca, dxc, dyc))
    run("k_deps_dinf (+7 scratch)", 11, lambda: T.areadinf_deps(s, ang, sca, dxc, dyc))
    if only is not None and not (only & {"k_threshold", "k_twi", "k_slopearea", "k_slopearearatio", "k_pd_smooth", "k_pd_mark", "k_lengtharea", "k_sad_pass"}):
        print(json.dumps({"n": n, "hbm_peak_gbs": peak, "kernels": out}))
        return
    # point-wise consumers on the rasters of the path
    T.aread8_sweep(s, ad8); T.areadinf_deps(s, ang, sca, dxc, dyc); T.areadinf_sweep(s, ang, sca, dxc)
    src = s.empty(torch.int16); o = s.empty(torch.float32)
    run("k_threshold", 6, lambda: T.l.td_threshold_dev(T.ctx, _p(ad8), None, _p(src), s.c, C.c_float(100.0), C.c_float(-1.0), T._stream()))
    run("k_twi", 12, lambda: T.l.td_twi_dev(T.ctx, _p(slp), _p(sca), _p(o), s.c, C.c_float(-1.0), C.c_float(-1.0), T._stream()))
    run("k_slopearea", 12, lambda: T.l.td_slopearea_dev(T.ctx, _p(slp), _p(sca), _p(o), s.c, C.c_float(2.0), C.c_float(1.0), T._stream()))
    run("k_slopearearatio", 12, lambda: T.l.td_slopearearatio_dev(T.ctx, _p(slp), _p(sca), _p(o), s.c, C.c_float(-1.0), T._stream()))
    # the stream definitions: Peuker-Douglas's two passes on fel, length-area on a path length (the D8 area stands in) and ad8 as int32
    sm = s.empty(torch.float32); ss = s.empty(torch.int16)
    wts = torch.tensor([0.4, 0.1, 0.05], dtype=torch.float32)
    B = lambda *ts: sum(t.element_size() for t in ts)      # noqa: E731  (bytes per cell from the rasters read and written)
    run("k_pd_smooth", B(fel, sm), lambda: T.l.td_peukerdouglas_smooth_dev(T.ctx, _p(fel), _p(sm), s.c, C.c_float(-3.0e38), wts.data_ptr(), T._stream()))
    run("k_pd_mark", B(sm, ss), lambda: T.l.td_peukerdouglas_mark_dev(T.ctx, _p(sm), _p(ss), s.c, C.c_float(-3.0e38), T._stream()))
    ad8i = ad8.round().to(torch.int32)
    run("k_lengtharea", B(ad8, ad8i, ss), lambda: T.l.td_lengtharea_dev(T.ctx, _p(ad8), _p(ad8i), _p(ss), s.c, C.c_float(0.03), C.c_float(1.3), T._stream()))
    # slopeavedown: the D8 sweep's counts mark the processed cells, then one pass at dn = 50 (the first pass: no slope is due yet, so
    # per cell the code byte, the state pair in and out and the slope's nodata test; sd is written in place only where a slope is due)
    T.aread8_deps(s, p, ad8); T.aread8_sweep(s, ad8)
    code = s.empty(torch.uint8); sd = s.empty(torch.float32)
    st0 = torch.empty((s.ny + 2, 2 * s.pitch), dtype=torch.float32, device="cuda"); st1 = torch.empty_like(st0)
    T.l.td_slopeavedown_init_dev(T.ctx, _p(p), _p(fel), _p(code), _p(st0), _p(st1), _p(sd), s.c, -32768, C.c_float(-3.0e38), T._stream())
    dist = torch.tensor([30.0, 900.0 ** 0.5 * 2 ** 0.5] * 4, dtype=torch.float32).repeat(s.ny).cuda()
    run("k_sad_pass", 21, lambda: T.l.td_slopeavedown_pass_dev(T.ctx, _p(code), _p(fel), _p(st0), _p(st1), _p(sd), s.c, _p(dist), C.c_double(50.0), None,
                                                               T._stream()))
    print(json.dumps({"n": n, "hbm_peak_gbs": peak, "kernels": out}))


if __name__ == "__main__":
    main()
