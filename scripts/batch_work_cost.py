"""Cost of batch work files (solver --batch-keys --batch-save / --batch-resume, worktool check) on one GPU, default grid, the
64-key 2^56 fixture: the save's size and time and the longest step beside it against the median step, the import-and-verify
time of a resume, and the time of `worktool check` on the file.  One run each; prints the card and its power limit first.

    python scripts/batch_work_cost.py
"""
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "tests", "golden", "in56_64keys.txt")


def run(args):
    t = time.perf_counter()
    p = subprocess.run([sys.executable, "-m"] + args, capture_output=True, text=True, cwd=ROOT)
    return p.stdout + p.stderr, time.perf_counter() - t


def main():
    path = os.path.join(tempfile.mkdtemp(), "batch64.work")
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    out, _ = run(["kangaroo_b200.solver", CFG, "--batch-keys", "--dp", "8", "--seed", "3", "--max-steps", "60",
                  "--batch-save", path, "--batch-save-interval", "0.2"])
    for line in out.splitlines():
        if line.startswith(("Range width", "SaveWork", "Batch:", "work file")):
            print(line)
    print("file: %.1f MB" % (os.path.getsize(path) / 1048576.0))
    out, _ = run(["kangaroo_b200.solver", "--batch-keys", "--batch-resume", path, "--max-steps", "1"])
    for line in out.splitlines():
        if line.startswith(("Resume", "rank")):
            print(line)
    out, dt = run(["kangaroo_b200.worktool", "check", path])
    print(out.strip())
    print("worktool check: %.2f s wall (process start, library load and check)" % dt)
    # the same file without its batch block (a plain HEADW file of key 0): the check's cost of the other 63 keys
    sys.path.insert(0, ROOT)
    from kangaroo_b200 import worktool
    plain = path + ".plain"
    with open(path, "rb") as src, open(plain, "wb") as dst:
        dst.write(src.read(worktool.read_batch(path).offset))
    worktool.check(plain)                                       # warm-up: library load, module load
    times = {}
    for name, f in (("plain", plain), ("batch", path), ("plain", plain), ("batch", path)):
        t = time.perf_counter()
        r = worktool.check(f)
        times.setdefault(name, []).append(time.perf_counter() - t)
    print("check in process (two runs each, alternating): plain HEADW %s s, batch file of %d keys %s s" %
          (["%.2f" % v for v in times["plain"]], r.n_keys, ["%.2f" % v for v in times["batch"]]))


if __name__ == "__main__":
    main()
