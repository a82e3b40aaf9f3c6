"""Insert rate of rank 0's two DP tables, in one process: the device table (kgx_dptable_add, records already in GPU memory,
time to the returned events) and the host table (kgi_add, the reference's HashTable with 8 bucket-sharded workers, records in
host memory).  Both tables grow together through size steps 2^20 .. 2^MAX entries: at each step they are grown to 2^k less
room for the timed batches, then batches of 2^16 and 2^20 records are inserted into both, alternating device and host, and
timed.  Each row reports the entries the tables held when its batches started (below 2^22 the timed batches alone outgrow
the step, so those rows start away from 2^k).  Each batch carries 5 % exact duplicates and 5 %
same-x records with another distance (half of them from the other herd) of entries already stored.  Prints the card name
and its power limit, one line per measurement, and writes results/dp_table_rate.json.

    python scripts/dp_table_rate.py                 # 2^20 .. 2^28 entries (the host table then holds ~16 GB of host RAM)
    python scripts/dp_table_rate.py --max-log2 26"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NB = 1 << 18
TYPE = np.uint64(1 << 62)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def random_recs(rng, n):
    a = rng.integers(0, 1 << 63, size=(n, 5), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 5), dtype=np.uint64)
    a[:, 0] = (a[:, 0] & np.uint64(0xFFFFFFFF)) | (rng.integers(0, NB, size=n, dtype=np.uint64) << np.uint64(32))
    return a


def batch(rng, n, stored):
    """n records: 90 % new, 5 % copies of stored ones, 5 % stored x with another distance (half of them the other herd)"""
    a = random_recs(rng, n)
    k = n // 20
    if len(stored):
        a[:k] = stored[rng.integers(0, len(stored), size=k)]
        c = stored[rng.integers(0, len(stored), size=k)].copy()
        c[:, 3] = rng.integers(0, 1 << 63, size=k, dtype=np.uint64)
        c[k // 2:, 4] ^= TYPE
        c[:k // 2, 3] ^= np.uint64(1)
        a[k:2 * k] = c
    return a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-log2", type=int, default=28)
    ap.add_argument("--reps", type=int, default=3, help="timed batches per table, size and batch size")
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "dp_table_rate.json"))
    a = ap.parse_args()
    import torch
    from kangaroo_b200.ingest import DPTable, DeviceDPTable
    rng = np.random.default_rng(1)
    top = 1 << a.max_log2
    host = DPTable(threads=8, max_events=1 << 20)
    dev = DeviceDPTable(top + (4 << 20), max_events=1 << 20)
    res = dict(card=card(), host_threads=host.threads, device_table_bytes=dev.memory_bytes(), rows=[])
    print("%s  host workers %d  device table %.2f GB" % (res["card"], host.threads, dev.memory_bytes() / 1e9), flush=True)
    ne = ctypes.c_uint32(0)
    stored_ = [np.zeros((0, 5), np.uint64)]                   # a sample of stored records to plant duplicates from
    keep = 1 << 16

    def insert(recs, timed):
        d = torch.from_numpy(recs.view(np.uint8).reshape(-1)).cuda()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rc, nd, _ = dev.add_raw(d.data_ptr(), [len(recs)], len(recs))
        t1 = time.perf_counter()
        rh = host._lib.kgi_add(host._h, recs.ctypes.data_as(ctypes.c_void_p), len(recs), 0, host._ev, host._cap, ctypes.byref(ne))
        t2 = time.perf_counter()
        assert rc == 0 and rh == 0 and nd == ne.value and len(dev) == len(host)
        stored = np.concatenate([stored_[0], recs[rng.integers(0, len(recs), size=keep // 16)]])[-keep:]
        stored_[0] = stored
        return t1 - t0, t2 - t1, nd

    for lg in range(20, a.max_log2 + 1):
        while len(dev) < (1 << lg) - (1 << 20) * a.reps * 1.1:  # grow both tables to just below the size
            insert(batch(rng, 1 << 20, stored_[0]), False)
        for bl in (16, 20):
            td, th, ev = [], [], 0
            for _ in range(a.reps):
                x, y, n_ev = insert(batch(rng, 1 << bl, stored_[0]), True)
                td.append(x); th.append(y); ev += n_ev
            row = dict(table_entries=len(dev), table_log2=lg, batch=1 << bl, device_records_per_s=(1 << bl) / float(np.median(td)),
                       host_records_per_s=(1 << bl) / float(np.median(th)), events=ev, reps=a.reps)
            row["speedup"] = row["device_records_per_s"] / row["host_records_per_s"]
            res["rows"].append(row)
            print("table 2^%d (%d entries)  batch 2^%d  device %.1f M rec/s  host %.2f M rec/s  x%.0f  (%d events)" %
                  (lg, row["table_entries"], bl, row["device_records_per_s"] / 1e6, row["host_records_per_s"] / 1e6, row["speedup"], ev),
                  flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    t0 = time.perf_counter()
    dev.close()
    t1 = time.perf_counter()
    host.close()
    print("close: device table %.2f s, host table %.2f s (%d entries)" % (t1 - t0, time.perf_counter() - t1, res["rows"][-1]["table_entries"]))


if __name__ == "__main__":
    main()
