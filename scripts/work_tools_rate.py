"""Rates of the GPU work-file tools (python -m kangaroo_b200.worktool check / merge) next to the reference's CPU -wcheck / -wm /
-wmdir (oracle/_ref/kangaroo_ref_cpu, where it was built) on the same files.

Makes two work files with the solver (--dp-table device, default grid, --dp DP, --max-steps STEPS, two seeds) in a temporary
directory, then times:
  - check: the check kernels alone (torch.profiler, CUDA activity: wt_check_entries_kernel + wt_check_walks_kernel) and end to
    end (host clock around the synchronous call);
  - merge of the 2 files and of 8 inputs (the 2 files 4 times over, so 3/4 of the entries are duplicates);
  - the reference's -wcheck, -wm and -wmdir on the same files (with --ref-timeout seconds each; "not measured" past it).
Prints one JSON line with the card's name and power limit.

    python scripts/work_tools_rate.py [--dp 8] [--steps 60] [--ref-timeout 600]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REFBIN = os.path.join(ROOT, "oracle", "_ref", "kangaroo_ref_cpu")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=60).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                         # noqa: BLE001
        return "unknown (%s)" % e


def timed(cmd, timeout):
    t0 = time.perf_counter()
    try:
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired:
        return None, ""
    return time.perf_counter() - t0, p.stdout


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dp", type=int, default=8)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--ref-timeout", type=float, default=600)
    ap.add_argument("--keep", default="", help="directory to keep the work files in (default: a temporary one)")
    a = ap.parse_args()
    import torch
    from kangaroo_b200 import worktool as wt
    res = {"card": card()}
    tmp = a.keep or tempfile.mkdtemp(prefix="kgx_wt_")
    try:
        files = []
        for seed in (1, 2):
            path = os.path.join(tmp, "s%d.work" % seed)
            t0 = time.perf_counter()
            subprocess.run([sys.executable, "-m", "kangaroo_b200.solver", os.path.join(ROOT, "tests", "golden", "in80.txt"), "--dp", str(a.dp),
                            "--max-steps", str(a.steps), "--seed", str(seed), "--dp-table", "device", "--save-work", path,
                            "--save-kangaroos"], capture_output=True, text=True, timeout=3600, cwd=ROOT)
            res["solver_s%d" % seed] = round(time.perf_counter() - t0, 2)
            files.append(path)
        res["file_bytes"] = os.path.getsize(files[0])
        wt.check(files[0])                                               # warm-up: module load, comb
        t0 = time.perf_counter()
        r = wt.check(files[0])
        res["check_e2e_s"] = time.perf_counter() - t0
        res["entries"], res["walks"], res["wrong"] = r.entries, r.walks, r.wrong_entries + r.wrong_walks
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            wt.check(files[0])
        kern = {}
        for ev in prof.events():
            if ev.name.startswith("_ZN6kgx_wt") or "wt_check" in ev.name:
                name = "entries" if "entries" in ev.name else "walks" if "walks" in ev.name else None
                if name:
                    kern[name] = kern.get(name, 0.0) + ev.device_time_total * 1e-6
        res["check_kernel_entries_s"] = kern.get("entries")
        res["check_kernel_walks_s"] = kern.get("walks")
        if kern.get("entries"):
            res["check_kernel_entries_per_s"] = r.entries / kern["entries"]
        res["check_e2e_entries_per_s"] = r.entries / res["check_e2e_s"]
        for name, inputs in (("merge2", files), ("merge8", files * 4)):
            dest = os.path.join(tmp, name + ".work")
            t0 = time.perf_counter()
            m = wt.merge_files(inputs, dest)
            dt = time.perf_counter() - t0
            res[name + "_s"] = dt
            res[name + "_out_entries"] = m.entries
            res[name + "_dups"] = m.duplicates
        ins = sum(r.entries for r in [wt.check(f) for f in files])
        res["merge2_input_entries_per_s"] = ins / res["merge2_s"]
        res["merge8_input_entries_per_s"] = 4 * ins / res["merge8_s"]
        if os.path.exists(REFBIN):
            dt, out = timed([REFBIN, "-t", str(os.cpu_count()), "-wcheck", files[0]], a.ref_timeout)
            res["ref_wcheck_s"] = dt if dt is not None else "not measured (timeout)"
            res["ref_threads"] = os.cpu_count()
            dt, _ = timed([REFBIN, "-wm", files[0], files[1], os.path.join(tmp, "ref_m2.work")], a.ref_timeout)
            res["ref_wm_s"] = dt if dt is not None else "not measured (timeout)"
            d = os.path.join(tmp, "dir8")
            os.makedirs(d, exist_ok=True)
            for i in range(8):
                shutil.copy(files[i % 2], os.path.join(d, "f%d.work" % i))
            dt, _ = timed([REFBIN, "-wmdir", d, os.path.join(tmp, "ref_m8.work")], a.ref_timeout)
            res["ref_wmdir8_s"] = dt if dt is not None else "not measured (timeout)"
        else:
            res["ref"] = "not measured (oracle/_ref/kangaroo_ref_cpu not built)"
    finally:
        if not a.keep:
            shutil.rmtree(tmp, ignore_errors=True)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
