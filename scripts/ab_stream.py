"""A/B of two builds of libkgx.so on the flagship workload, in one process tree on one GPU.

  python scripts/ab_stream.py --base results/base/libkgx.so [--runs 5] [--sweep]

Runs `bench.py --no-cpu-baseline` alternately against the baseline library (loaded through KGX_LIB_OVERRIDE, which is
never rebuilt) and the tree's own build, `--runs` times each; the first run of each dumps its outputs (`--dump-outputs`)
and the two dumps are compared array for array.  The baseline's sha256 is checked before and after, so a baseline that
changed under the runs is reported, not compared.  `--sweep` adds scripts/sweep2.py on the default herd for the L2
prefetch distances 0-4 and the 3-CTA variant of the tree's build, and the baseline at its default.  The card, its power
limit and its maximum SM clock are read with nvidia-smi queries (read-only).  Everything goes to results/ab_stream.json."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sha256(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(cmd, base=None):
    env = dict(os.environ)
    env.pop("KGX_LIB_OVERRIDE", None)
    if base:
        env["KGX_LIB_OVERRIDE"] = base
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        raise SystemExit("%s failed (%d):\n%s" % (" ".join(cmd), p.returncode, (p.stdout + p.stderr)[-3000:]))
    return p.stdout


def bench(base, dump):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--no-cpu-baseline"] + (["--dump-outputs", dump] if dump else [])
    r = json.loads([ln for ln in run(cmd, base).splitlines() if ln.startswith("{")][-1])
    return dict(value=r["value"], kernel=r["kernel_only"]["value"], sm_mhz=r["clocks"]["sm_mhz"], reasons=r["clocks"]["reasons"])


def same_outputs(a, b):
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    if names != sorted(f for f in os.listdir(b) if f.endswith(".npy")):
        return {"equal": False, "why": "different array sets"}
    diff = [n for n in names if not np.array_equal(np.load(os.path.join(a, n)), np.load(os.path.join(b, n)))]
    return {"equal": not diff, "arrays": len(names), "differing": diff}


def stats(vals):
    return {"median": statistics.median(vals), "min": min(vals), "max": max(vals), "all": vals}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="baseline libkgx.so")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--grid", default="264,128", help="sweep grid gx,gy (default: bench.py's default grid on a 132-SM H100 SXM)")
    args = ap.parse_args()
    base = os.path.abspath(args.base)
    out_dir = os.path.join(ROOT, "results")
    os.makedirs(out_dir, exist_ok=True)
    res = {"card": card(), "base_sha256": sha256(base), "new_sha256": sha256(os.path.join(ROOT, "kangaroo_b200", "csrc", "libkgx.so"))}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    runs = {"base": [], "new": []}
    for i in range(args.runs):
        for label in (("base", "new") if i % 2 == 0 else ("new", "base")):
            dump = os.path.join(out_dir, "dump_" + label) if i == 0 else None
            r = bench(base if label == "base" else None, dump)
            runs[label].append(r)
            print("run %d %-4s value %8.1f MJump/s  kernel %8.1f  SM %s MHz %s" % (i, label, r["value"], r["kernel"], r["sm_mhz"], r["reasons"]), flush=True)
    res["runs"] = runs
    res["base_sha256_after"] = sha256(base)
    res["base_unchanged"] = res["base_sha256_after"] == res["base_sha256"]
    res["outputs"] = same_outputs(os.path.join(out_dir, "dump_base"), os.path.join(out_dir, "dump_new"))
    for key in ("value", "kernel"):
        b, n = stats([r[key] for r in runs["base"]]), stats([r[key] for r in runs["new"]])
        res[key] = {"base": b, "new": n, "median_gain": n["median"] / b["median"] - 1.0,
                    "slowest_new_beats_fastest_base": n["min"] > b["max"],
                    "spread_base": (b["max"] - b["min"]) / b["median"], "spread_new": (n["max"] - n["min"]) / n["median"]}
        print("%-6s base median %.1f [%.1f, %.1f]  new median %.1f [%.1f, %.1f]  gain %+.2f %%  slowest new > fastest base: %s"
              % (key, b["median"], b["min"], b["max"], n["median"], n["min"], n["max"], 100 * res[key]["median_gain"],
                 res[key]["slowest_new_beats_fastest_base"]), flush=True)
    print("outputs identical:", res["outputs"], " baseline unchanged:", res["base_unchanged"], flush=True)
    if args.sweep:
        grid = "|" + args.grid
        specs = ["pf%d|KGX_MODE=stream,KGX_STREAM_PF=%d%s" % (pf, pf, grid) for pf in range(5)]
        specs += ["ctas3-pf2|KGX_MODE=stream,KGX_STREAM_CTAS=3,KGX_STREAM_PF=2%s" % grid]
        res["sweep_new"] = run([sys.executable, "scripts/sweep2.py"] + specs)
        res["sweep_base"] = run([sys.executable, "scripts/sweep2.py", "base-pf2|KGX_MODE=stream,KGX_STREAM_PF=2" + grid], base)
        print(res["sweep_new"] + res["sweep_base"], flush=True)
    json.dump(res, open(os.path.join(out_dir, "ab_stream.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
