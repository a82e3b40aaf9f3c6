"""What --batch-keys saves: one seeded multi-key input solved twice on one GPU, key after key (the solver's default, like the
reference) and with --batch-keys (one tame herd for every key).  Reports for each run the total jumps in sqrt(N) units
(N = 2^range bits), the wall time, the steady jump rate and whether every key was found, with the card name and its power
limit, and writes results/multikey_cost.json.

    python scripts/multikey_cost.py --keys 32 --bits 60 --grid 16,128 --dp 8
    python scripts/multikey_cost.py --runs batch --dp-table host,device     # the batch run with each DP table, in one call

The DP bits should keep the DP overhead, kangaroos * 2^dp jumps per key, well below sqrt(N), and the DPs of one launch
(kangaroos * 64 / 2^dp) below the engine's 2^17 slots: the default grid (4.3 M kangaroos on an H100) needs a range of
2^80 or more for both, where one sequential key takes minutes."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.golden import make_multikey  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run(args):
    """the solver's output is echoed as it comes"""
    t0 = time.perf_counter()
    p = subprocess.Popen([sys.executable, "-m", "kangaroo_b200.solver"] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, cwd=ROOT)
    lines = []
    for line in p.stdout:
        lines.append(line)
        print("  | " + line, end="", flush=True)
    return p.wait(), "".join(lines), time.perf_counter() - t0


def measure(out, privs, rp):
    """jumps, steady rate and keys found from one solver output (sequential: one block per key; batch: one block)"""
    kang = [int(v) for v in re.findall(r"kangaroos/GPU: (\d+)\s+GPUs: \d+", out)]
    gpus = [int(v) for v in re.findall(r"GPUs: (\d+)", out)]
    rates = re.findall(r"Solver rate: (\d+) MJump/s steady state .*?, \d+ MJump/s over all (\d+) steps \(([\d.]+) s\)", out)
    table_ms = [float(v) for v in re.findall(r"rank-0 (?:ingest|device table) ([\d.]+) ms/step", out)]
    close = re.search(r"close ([\d.]+) s \(engine and table freed\)", out)
    jumps = sum(kang[i] * gpus[i] * 64 * int(r[1]) for i, r in enumerate(rates))
    loop_s = sum(float(r[2]) for r in rates)
    found = {int(i): int(v, 16) for i, v in re.findall(r"Key#\s*(\d+) Pub:\s+0x[0-9A-F]+\s+Priv: 0x([0-9A-F]+)", out)}
    ok = sum(1 for i, k in enumerate(privs) if found.get(i) == k)
    return dict(keys_found=ok, jumps=jumps, jumps_sqrtN=jumps / 2.0 ** (rp / 2), jumps_sqrtN_per_key=jumps / len(privs) / 2.0 ** (rp / 2),
                loop_seconds=loop_s, steady_MJump_s=(jumps / loop_s / 1e6) if loop_s else 0.0,
                steady_rates_MJump_s=[int(r[0]) for r in rates], table_ms_per_step=table_ms,
                close_seconds=float(close.group(1)) if close else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=32)
    ap.add_argument("--bits", type=int, default=60)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--grid", default="16,128")
    ap.add_argument("--dp", type=int, default=8)
    ap.add_argument("--dp-table", default="host", help="comma-separated solver --dp-table values, each run in turn")
    ap.add_argument("--runs", default="batch,sequential", help="batch, sequential or both")
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "multikey_cost.json"))
    a = ap.parse_args()
    start, end, privs = make_multikey.make(a.keys, a.bits, a.seed)
    tmp = tempfile.mkdtemp()
    cfg = os.path.join(tmp, "keys.txt")
    make_multikey.write(cfg, os.path.join(tmp, "keys.answers.txt"), start, end, privs)
    common = ["--dp", str(a.dp), "--grid", a.grid, "--seed", str(a.seed)]
    res = dict(card=card(), keys=a.keys, range_bits=a.bits, grid=a.grid, dp=a.dp, seed=a.seed,
               model_sequential_sqrtN=2.08 * a.keys, model_batch_sqrtN=2.08 * a.keys ** 0.5)
    runs = [(n, e) for n, e in (("batch", ["--batch-keys"]), ("sequential", [])) if n in a.runs.split(",")]
    tables = a.dp_table.split(",")
    for table in tables:
        for name, extra in runs:
            key = name if len(tables) == 1 and table == "host" else "%s/%s" % (name, table)
            rc, out, wall = run([cfg] + common + extra + ["--dp-table", table])
            m = measure(out, privs, a.bits)
            m.update(returncode=rc, wall_seconds=wall, dp_table=table)
            res[key] = m
            print("%-16s keys %d/%d  jumps %.3g = %.2f sqrt(N) (%.3f per key)  wall %.1f s  steady %.0f MJump/s  table %s ms/step  "
                  "close %s s  rc %d" % (key, m["keys_found"], a.keys, m["jumps"], m["jumps_sqrtN"], m["jumps_sqrtN_per_key"], wall,
                                         m["steady_MJump_s"], ",".join("%.2f" % v for v in m["table_ms_per_step"][:4]),
                                         m["close_seconds"], rc), flush=True)
            if rc not in (0, 1):
                print(out[-3000:])
    for table in tables:
        sfx = "" if len(tables) == 1 and table == "host" else "/" + table
        s, b = res.get("sequential" + sfx), res.get("batch" + sfx)
        if s and b:
            res["jump_ratio_batch_over_sequential" + sfx] = b["jumps"] / s["jumps"] if s["jumps"] else None
            res["wall_ratio_batch_over_sequential" + sfx] = b["wall_seconds"] / s["wall_seconds"]
            print("%s%s: batch/sequential jumps %.3f (model 1/sqrt(K) = %.3f), wall time %.3f" %
                  (res["card"], sfx, res["jump_ratio_batch_over_sequential" + sfx] or 0, a.keys ** -0.5,
                   res["wall_ratio_batch_over_sequential" + sfx]))
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
