"""The device DP table's two layouts side by side, in one process: entries in GPU memory (entries="device") and entries in
mapped, pinned host memory (entries="host", KGX_DPT_HOST_ENTRIES).
  1. insert rate: both tables grow together through size steps 2^20 .. 2^MAX entries; at each step batches of 2^16 and 2^20
     records (records already in GPU memory, time to the returned events) go into both, alternating the layouts.  Each batch
     carries 5 % exact duplicates and 5 % same-x records with another distance of entries already stored, as
     scripts/dp_table_rate.py's do.
  2. save and load of the full tables (2^MAX entries less the timed batches) to a temporary directory, each layout's file
     loaded back into the other layout; the files are compared byte for byte.
  3. the capacity the solver's default rule gives with --dp-table-entries host on this machine (GPU free memory, MemAvailable,
     one table), and the time to create a table of that capacity (its pinned buffer); the table is freed at once.
Prints the card name and its power limit, one line per measurement, and writes results/host_entries_rate.json.

    python scripts/host_entries_rate.py                 # 2^20 .. 2^27 entries
    python scripts/host_entries_rate.py --max-log2 24 --no-default"""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from dp_table_rate import batch, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-log2", type=int, default=27)
    ap.add_argument("--reps", type=int, default=3, help="timed batches per layout, size and batch size")
    ap.add_argument("--no-default", action="store_true", help="skip step 3 (it pins most of the host's available RAM)")
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "host_entries_rate.json"))
    a = ap.parse_args()
    import torch
    from kangaroo_b200 import solver as S
    from kangaroo_b200.ingest import DeviceDPTable
    rng = np.random.default_rng(1)
    top = 1 << a.max_log2
    t0 = time.perf_counter()
    dev = DeviceDPTable(top + (4 << 20), max_events=1 << 20)
    t1 = time.perf_counter()
    host = DeviceDPTable(top + (4 << 20), max_events=1 << 20, entries="host")
    t2 = time.perf_counter()
    tables = dict(device=dev, host=host)
    res = dict(card=card(), capacity=dev.capacity, create_s=dict(device=t1 - t0, host=t2 - t1),
               gpu_bytes=dict(device=dev.memory_bytes(), host=host.memory_bytes()), pinned_bytes=host.host_bytes(), rows=[])
    print("%s  capacity %d: device layout %.2f GB GPU (created in %.2f s), host layout %.2f GB GPU + %.2f GB pinned (%.2f s)" %
          (res["card"], dev.capacity, dev.memory_bytes() / 1e9, t1 - t0, host.memory_bytes() / 1e9, host.host_bytes() / 1e9, t2 - t1),
          flush=True)
    stored_ = [np.zeros((0, 5), np.uint64)]
    keep = 1 << 16

    def insert(recs):
        d = torch.from_numpy(recs.view(np.uint8).reshape(-1)).cuda()
        torch.cuda.synchronize()
        out = {}
        for name in ("device", "host"):
            t = time.perf_counter()
            rc, ne, _ = tables[name].add_raw(d.data_ptr(), [len(recs)], len(recs))
            out[name] = (time.perf_counter() - t, ne)
            assert rc == 0
        assert out["device"][1] == out["host"][1] and len(dev) == len(host)
        stored_[0] = np.concatenate([stored_[0], recs[rng.integers(0, len(recs), size=keep // 16)]])[-keep:]
        return out

    for lg in range(20, a.max_log2 + 1):
        while len(dev) < (1 << lg) - (1 << 20) * a.reps * 1.1:
            insert(batch(rng, 1 << 20, stored_[0]))
        for bl in (16, 20):
            times = dict(device=[], host=[])
            for _ in range(a.reps):
                for name, (dt, _) in insert(batch(rng, 1 << bl, stored_[0])).items():
                    times[name].append(dt)
            row = dict(table_entries=len(dev), table_log2=lg, batch=1 << bl, reps=a.reps,
                       device_records_per_s=(1 << bl) / float(np.median(times["device"])),
                       host_records_per_s=(1 << bl) / float(np.median(times["host"])))
            res["rows"].append(row)
            print("table 2^%d (%d entries)  batch 2^%d  device entries %.1f M rec/s  host entries %.1f M rec/s  (host/device %.2f)" %
                  (lg, row["table_entries"], bl, row["device_records_per_s"] / 1e6, row["host_records_per_s"] / 1e6,
                   row["host_records_per_s"] / row["device_records_per_s"]), flush=True)

    hdr = dict(dp_bits=20, range_start=1 << 100, range_end=(1 << 100) + (1 << 120), pubkey=(3, 5), total_count=1, total_time=1.0)
    with tempfile.TemporaryDirectory() as tmp:
        files, io = {}, {}
        for name, t in tables.items():
            files[name] = os.path.join(tmp, name + ".work")
            t0 = time.perf_counter()
            t.save_work(files[name], **hdr)
            io["save_" + name] = time.perf_counter() - t0
        same = filecmp.cmp(files["device"], files["host"], shallow=False)
        n = len(dev)
        for name, src in (("device", "host"), ("host", "device")):     # each layout loads the other's file
            t0 = time.perf_counter()
            tables[name].load_work_ex(files[src])
            io["load_" + name] = time.perf_counter() - t0
            assert len(tables[name]) == n
        res["save_load"] = dict(entries=n, file_bytes=os.path.getsize(files["device"]), files_equal=same, **io)
        print("save / load of %d entries (%.2f GB file, files equal: %s): save device %.2f s, host %.2f s; load device %.2f s, "
              "host %.2f s" % (n, os.path.getsize(files["device"]) / 1e9, same, io["save_device"], io["save_host"],
                               io["load_device"], io["load_host"]), flush=True)
    dev.close()
    host.close()

    if not a.no_default:
        free = torch.cuda.mem_get_info(0)[0]
        avail = S.mem_available()
        cap = S.default_table_capacity(free - S.scratch_bytes(1 << 17), entries="host", host_limit=S.host_entries_limit(avail, 1))
        t0 = time.perf_counter()
        t = DeviceDPTable(cap, entries="host")
        dt = time.perf_counter() - t0
        res["default"] = dict(gpu_free=free, mem_available=avail, capacity=cap, gpu_bytes=t.memory_bytes(), pinned_bytes=t.host_bytes(),
                              create_s=dt)
        t0 = time.perf_counter()
        t.close()
        res["default"]["destroy_s"] = time.perf_counter() - t0
        print("default rule here: GPU free %.1f GB, MemAvailable %.1f GB -> capacity %d entries (%.2f GB GPU, %.2f GB pinned), "
              "created in %.2f s, freed in %.2f s" % (free / 1e9, avail / 1e9, cap, res["default"]["gpu_bytes"] / 1e9,
                                                     res["default"]["pinned_bytes"] / 1e9, dt, res["default"]["destroy_s"]), flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
