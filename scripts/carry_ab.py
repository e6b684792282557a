"""Carry on / off comparison of the contributing-area sweep: bench.py alternately with and without TAUDEM_B200_EXP=16 (no
carried tiles), the median and spread of ms_per_step and of both sweeps' per-kernel times, and whether the results agree.

  python scripts/carry_ab.py [reps=5] [size ...=16384 32768]"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("ms_per_step", "k_sweep_warp<d8>", "k_sweep_warp<dinf>")


def run(size, carry):
    env = dict(os.environ)
    env.pop("TAUDEM_B200_EXP", None)
    if not carry:
        env["TAUDEM_B200_EXP"] = "16"
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu", "--no-same-config", "--size", str(size)],
                         env=env, check=True, stdout=subprocess.PIPE, text=True).stdout
    r = json.loads(out.strip().splitlines()[-1])
    pk = r["roofline"]["per_kernel_ms"]
    h = out.split('"hash_ad8": "')[1][:16], out.split('"hash_sca": "')[1][:16]
    return {"ms_per_step": r["ms_per_step"], "k_sweep_warp<d8>": pk["k_sweep_warp<d8>"], "k_sweep_warp<dinf>": pk["k_sweep_warp<dinf>"]}, h


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    sizes = [int(s) for s in sys.argv[2:]] or [16384, 32768]
    for size in sizes:
        res = {True: [], False: []}
        hashes = set()
        for i in range(reps):
            for carry in ((True, False) if i % 2 == 0 else (False, True)):
                m, h = run(size, carry)
                res[carry].append(m)
                hashes.add(h)
                print(size, "carry" if carry else "no-carry", json.dumps(m), h, flush=True)
        print(f"== {size}^2, {reps} runs each; results identical: {len(hashes) == 1} {sorted(hashes)}")
        for k in KEYS:
            on = [m[k] for m in res[True]]; off = [m[k] for m in res[False]]
            mon, moff = statistics.median(on), statistics.median(off)
            print(f"   {k:20s} carry {mon:8.2f} [{min(on):.2f} .. {max(on):.2f}]   no carry {moff:8.2f} [{min(off):.2f} .. {max(off):.2f}]"
                  f"   {100 * (moff - mon) / moff:+.1f} %", flush=True)


if __name__ == "__main__":
    main()
