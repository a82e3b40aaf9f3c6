"""Work-file save and load times of rank 0's device DP table (DeviceDPTable.save_work / load_work_ex: the bucket sort on the
GPU, then the file through pinned chunks), with the host table's save_work (the reference's HashTable::SaveTable) on the same
entries as a control.  Both tables are filled with 2^LOG2 random records of distinct x; the file goes to a temporary
directory and is removed at the end.  Prints the card's name and power limit and one JSON line of times in seconds.

    python scripts/dp_table_save_rate.py [--log2 26] [--reps 3]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NB = 1 << 18
HDR = dict(dp_bits=12, range_start=1 << 70, range_end=(1 << 70) + (1 << 66), pubkey=(0xABCDEF << 100, 0x777 << 50),
           total_count=123456789, total_time=42.5)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2", type=int, default=26)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch-log2", type=int, default=22)
    a = ap.parse_args()
    import torch
    from kangaroo_b200.ingest import DPTable, DeviceDPTable
    n, b = 1 << a.log2, 1 << a.batch_log2
    dev = DeviceDPTable(n, max_events=1 << 16)
    host = DPTable(threads=8, max_events=1 << 16)
    ne = ctypes.c_uint32(0)
    rng = np.random.default_rng(3)
    for i in range(0, n, b):                                 # records {kidx | h << 32, x lo, x hi, d lo, d hi}, x random
        r = rng.integers(0, 1 << 63, size=(b, 5), dtype=np.uint64) * np.uint64(2)
        r[:, 0] = np.arange(i, i + b, dtype=np.uint64) | (rng.integers(0, NB, size=b, dtype=np.uint64) << np.uint64(32))
        r[:, 4] &= np.uint64(0x7FFFFFFFFFFFFFFF)
        d = torch.from_numpy(r.view(np.uint8).reshape(-1)).cuda()
        assert dev.add_raw(d.data_ptr(), [b], b)[0] == 0
        assert host._lib.kgi_add(host._h, r.ctypes.data_as(ctypes.c_void_p), b, 0, host._ev, host._cap, ctypes.byref(ne)) == 0
    torch.cuda.synchronize()
    assert len(dev) == len(host)
    out = dict(card=card(), entries=len(dev), save_device=[], load_device=[], save_host=[])
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "t.work")
        for _ in range(a.reps):
            t0 = time.perf_counter()
            dev.save_work(path, **HDR)
            t1 = time.perf_counter()
            w = dev.load_work_ex(path)
            t2 = time.perf_counter()
            host.save_work(path, **HDR)
            t3 = time.perf_counter()
            assert len(dev) == out["entries"] and w.dp_bits == HDR["dp_bits"]
            out["save_device"].append(round(t1 - t0, 3))
            out["load_device"].append(round(t2 - t1, 3))
            out["save_host"].append(round(t3 - t2, 3))
    print(json.dumps(out), flush=True)
    dev.close()
    host.close()


if __name__ == "__main__":
    main()
