"""Cost of merging batch work files (python -m kangaroo_b200.worktool merge on --batch-keys --batch-save files).

Makes two batch work files with the solver (the 64-key 2^56 fixture, default grid, --dp DP, --max-steps STEPS, two seeds) in
a temporary directory, then measures:
  - the merge of the two files (kgx_work_merge_batch, host clock around the synchronous call, --runs times) and the number of
    collisions in each class;
  - the resolver alone: kgx_work_resolve on N collisions against 1, 64, 1024 and 65535 keys (host clock around the C call on
    arrays prepared before, so it includes the key index, the comb and the copies), next to the host's kgi_resolve_multi
    (build/libkgx_ingest.so) on a sample of them, per collision.
Prints one JSON line with the card's name and power limit.

    python scripts/batch_merge_rate.py [--dp 8] [--steps 60] [--runs 3] [--n 262144]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CFG64 = os.path.join(ROOT, "tests", "golden", "in56_64keys.txt")
TYPE_BIT = 1 << 126


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:                         # noqa: BLE001
        return "unknown (%s)" % e


def keys_of(n, rng):
    """n keys K = k*G with consecutive scalars from a random one (one point addition each)"""
    from kangaroo_b200 import ecmath as ec
    k0 = int(rng.integers(1, 1 << 62)) << 60
    p, out, ks = ec.mul(k0), [], []
    for i in range(n):
        out.append(p)
        ks.append(k0 + i)
        p = ec.add(p, ec.G)
    return ks, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dp", type=int, default=8)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--n", type=int, default=1 << 18, help="collisions per resolver call")
    ap.add_argument("--host-sample", type=int, default=2000, help="collisions resolved on the host per key count")
    a = ap.parse_args()
    import ctypes
    from kangaroo_b200 import worktool as wt
    from kangaroo_b200._lib import load_library
    from kangaroo_b200.ingest import DPTable, _limbs4
    u64p = ctypes.POINTER(ctypes.c_uint64)
    res = {"gpu": card(), "runs": a.runs}
    with tempfile.TemporaryDirectory() as d:
        files = []
        for seed in (1, 2):
            p = os.path.join(d, "run%d.work" % seed)
            out = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver", CFG64, "--batch-keys", "--dp", str(a.dp), "--seed", str(seed),
                                  "--max-steps", str(a.steps), "--batch-save", p], capture_output=True, text=True, cwd=ROOT)
            if not os.path.exists(p):
                raise SystemExit(out.stdout[-2000:] + out.stderr[-2000:])
            files.append(p)
        res["file_mb"] = [round(os.path.getsize(p) / 2**20, 1) for p in files]
        times = []
        for i in range(a.runs + 1):                 # the first call loads the module: not timed
            t0 = time.perf_counter()
            r = wt.merge_batch_files(files, os.path.join(d, "m%d.work" % i))
            if i:
                times.append(time.perf_counter() - t0)
        res["merge_s"] = [round(t, 3) for t in times]
        res.update(entries=r.entries, duplicates=r.duplicates, collisions=r.collisions, solving=r.solving,
                   already_solved=r.already_solved, no_key=r.no_key, same_herd=r.same_herd, solved_in_inputs=r.solved_in_inputs,
                   solved_by_merge=r.solved_by_merge, left=r.left)
    rng = np.random.default_rng(5)
    start = 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD00000000000000
    host = DPTable(threads=1)
    limbs = lambda v: (v & 0xFFFFFFFFFFFFFFFF, v >> 64)
    rates = {}
    for nk in (1, 64, 1024, 65535):
        ks, pts = keys_of(nk, rng)
        pick = rng.integers(0, nk, a.n)
        w = [int(v) << 40 for v in rng.integers(1, 1 << 62, a.n)]
        tame = [ks[int(j)] + x for j, x in zip(pick, w)]    # every collision hits a key
        wild = [x | TYPE_BIT for x in w]
        got = wt.resolve(tame[:a.host_sample], wild[:a.host_sample], pts, start)
        kt_dev = np.ascontiguousarray(np.hstack([wt._limbs([p[0] for p in pts], 4), wt._limbs([p[1] for p in pts], 4)]))
        da, db = np.ascontiguousarray(wt._limbs(tame, 2)), np.ascontiguousarray(wt._limbs(wild, 2))
        idx, priv = np.zeros(a.n, dtype=np.uint32), np.zeros((a.n, 4), dtype=np.uint64)
        lib = load_library()
        args = (0, da.ctypes.data_as(u64p), db.ctypes.data_as(u64p), a.n, kt_dev.ctypes.data_as(u64p), nk, _limbs4(start),
                idx.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), priv.ctypes.data_as(u64p))
        calls = []
        for _ in range(a.runs):
            t0 = time.perf_counter()
            assert lib.kgx_work_resolve(*args) == 0
            calls.append(time.perf_counter() - t0)
        dev = min(calls) / a.n
        assert all(idx[:a.host_sample] == [g[0] for g in got])
        kt = DPTable.key_table(pts)
        m = a.host_sample
        t0 = time.perf_counter()
        want = [host.resolve_multi(limbs(x), limbs(y), kt, start) for x, y in zip(tame[:m], wild[:m])]
        hst = (time.perf_counter() - t0) / m
        assert got[:m] == want
        rates[nk] = {"device_us": round(dev * 1e6, 4), "device_calls_s": [round(c, 4) for c in calls], "host_us": round(hst * 1e6, 2),
                     "speedup": round(hst / dev, 1)}
    host.close()
    res["resolve_per_collision"] = rates
    res["resolve_collisions_per_call"] = a.n
    print(json.dumps(res))


if __name__ == "__main__":
    main()
