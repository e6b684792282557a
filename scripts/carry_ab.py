"""A/B comparison of the contributing-area sweep: bench.py alternately in two arms, the median and spread of ms_per_step and of
both sweeps' per-kernel times, and whether the results agree.  The default arms are this tree with and without
TAUDEM_B200_EXP=16 (no carried tiles); with --other DIR they are this tree and the built tree DIR (another version of the
project, e.g. a copy of the parent commit), both as they are.

  python scripts/carry_ab.py [--other DIR] [reps=5] [size ...=16384 32768]"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("ms_per_step", "k_sweep_warp<d8>", "k_sweep_warp<dinf>")


def run(size, arm, other):
    """arm True: this tree as it is; False: the other arm (no carry, or the tree `other`)."""
    env = dict(os.environ)
    env.pop("TAUDEM_B200_EXP", None)
    root = ROOT
    if not arm:
        if other:
            root = other
        else:
            env["TAUDEM_B200_EXP"] = "16"
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--no-cpu", "--no-same-config", "--size", str(size)],
                         env=env, cwd=root, check=True, stdout=subprocess.PIPE, text=True).stdout
    r = json.loads(out.strip().splitlines()[-1])
    pk = r["roofline"]["per_kernel_ms"]
    h = out.split('"hash_ad8": "')[1][:16], out.split('"hash_sca": "')[1][:16]
    return {"ms_per_step": r["ms_per_step"], "k_sweep_warp<d8>": pk["k_sweep_warp<d8>"], "k_sweep_warp<dinf>": pk["k_sweep_warp<dinf>"]}, h


def main():
    args = sys.argv[1:]
    other = ""
    if args[:1] == ["--other"]:
        other = os.path.abspath(args[1])
        args = args[2:]
    reps = int(args[0]) if args else 5
    sizes = [int(s) for s in args[1:]] or [16384, 32768]
    names = ("this", "other") if other else ("carry", "no carry")
    for size in sizes:
        res = {True: [], False: []}
        hashes = set()
        for i in range(reps):
            for arm in ((True, False) if i % 2 == 0 else (False, True)):
                m, h = run(size, arm, other)
                res[arm].append(m)
                hashes.add(h)
                print(size, names[0] if arm else names[1], json.dumps(m), h, flush=True)
        print(f"== {size}^2, {reps} runs each; results identical: {len(hashes) == 1} {sorted(hashes)}")
        for k in KEYS:
            a = [m[k] for m in res[True]]; b = [m[k] for m in res[False]]
            ma, mb = statistics.median(a), statistics.median(b)
            print(f"   {k:20s} {names[0]} {ma:8.2f} [{min(a):.2f} .. {max(a):.2f}]   {names[1]} {mb:8.2f} [{min(b):.2f} .. {max(b):.2f}]"
                  f"   {100 * (mb - ma) / mb:+.1f} %", flush=True)


if __name__ == "__main__":
    main()
