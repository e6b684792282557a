"""CUDA-event timings and per-visit statistics of the contributing-area sweeps alone (deps excluded).

  TAUDEM_B200_TIMING=1 python scripts/sweep_stats.py [n=16384] [reps=2]

With TAUDEM_B200_TIMING=1 the kernel records, per tile visit, the cycles lane 0 spent waiting for a ticket, loading,
running the wavefront and writing back, the cells evaluated and the wavefront iterations, and counts the visits of carried
tiles (claimed by the worker that made them ready, without a ticket: their wait is zero).
TAUDEM_B200_WORKERS=<n> (fewer workers per SM), TAUDEM_B200_POLL=1 (plain nanosleep polling) and TAUDEM_B200_EXP=16 (no carried
tiles) are experiment knobs of the kernel."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from taudem_b200.device import DeviceStrip, Tools


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record(); r = fn(); b.record(); torch.cuda.synchronize()
    return r, a.elapsed_time(b)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    T = Tools()
    s, dxc, dyc, p, ang, info, pipe = bench.build_inputs(T, n, torch)
    print("inputs", info, pipe, flush=True)
    for tool in ("aread8", "areadinf"):
        out = s.empty(torch.float32)
        best = 1e30
        for _ in range(reps):
            if tool == "aread8":
                T.aread8_deps(s, p, out); _, t = timed(lambda: T.aread8_sweep(s, out))
            else:
                T.areadinf_deps(s, ang, out, dxc, dyc); _, t = timed(lambda: T.areadinf_sweep(s, ang, out, dxc))
            best = min(best, t)
        own = s.owned(out)
        line = f"{tool:9s} sweep {best:9.2f} ms  {n * n / best / 1e3:9.1f} Mcells/s  max {float(own.max()):.6g}  hash {bench.raster_hash(torch, own, 0, n):016x}"
        if os.environ.get("TAUDEM_B200_TIMING"):
            c = [T.l.td_ctx_counter(T.ctx, 24 + i) for i in range(8)]
            v = max(c[3], 1)
            line += f"\n    visits {c[3]} ({c[3] / ((n + 31) // 32) ** 2:.2f} per tile), carried {c[0]} ({100 * c[0] / v:.1f} %); cycles per visit: wait {c[4]//v} load {c[5]//v} wavefront {c[6]//v} write-back {c[7]//v}"
            line += f"; cells/visit {c[1] / v:.0f}, wavefront iterations/visit {c[2] / v:.1f}, cycles/iteration {c[6] / max(c[2], 1):.0f}"
        print(line, flush=True)
        del out


if __name__ == "__main__":
    main()
