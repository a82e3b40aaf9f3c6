"""Cost of resolving tame/wild collisions on the device (kgx_resolver_*, kgx_dptable_add_resolve) against the host resolver.

Measures, on one GPU:
  - the resolver per collision at 1, 64, 1024 and 65535 keys: the run call (host clock around kgx_resolver_run and a
    synchronise of its stream, --n collisions per call, median of --reps calls after a warm-up) and the kernel alone
    (wt_resolve_pairs_kernel's device time in a torch.profiler trace of its own, median); half the collisions hit a key;
    next to the host's kgi_resolve_multi per collision (build/libkgx_ingest.so, where it was built) on a sample;
  - the device table's add of one step of records (--records, with --events collisions among them) plain and resolving,
    alternated, median ms per call: what resolving costs a step;
  - the rank-0 ingest thread's ms/step (the solver's rate line) of a --batch-keys run of the 64-key 2^56 fixture over
    --steps steps, with --dp-table device (resolved with the insert) and, where the library exists, --dp-table host
    (kgi_resolve_multi per collision).
Prints the card's name, power limit and SM clocks, then one JSON line.

    python scripts/resolver_rate.py [--n 65536] [--reps 20] [--steps 300]"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CFG64 = os.path.join(ROOT, "tests", "golden", "in56_64keys.txt")
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
TYPE_BIT = 1 << 126
M64 = (1 << 64) - 1


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
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


def pairs_of(n, ks, rng):
    """n (tame, wild) tagged-distance pairs; the even ones hit a key (tame = k + w, wild = w), the odd ones none"""
    out = []
    for i in range(n):
        w = int(rng.integers(0, 1 << 62)) << 40
        k = ks[int(rng.integers(0, len(ks)))] + (0 if i % 2 == 0 else 1 << 100)
        out.append((k + w, w | TYPE_BIT))
    return out


def limbs(vals):
    return np.array([[v & M64, v >> 64] for v in vals], dtype=np.uint64)


def resolver_rates(n_keys, n, reps, rng, torch):
    from torch.profiler import ProfilerActivity, profile
    from kangaroo_b200.ingest import DeviceResolver
    ks, pts = keys_of(n_keys, rng)
    pairs = pairs_of(n, ks, rng)
    dev = torch.device("cuda", 0)
    p = torch.from_numpy(np.hstack([limbs([a for a, _ in pairs]), limbs([b for _, b in pairs])]).view(np.int64)).to(dev)
    key = torch.empty(n, dtype=torch.int32, device=dev)
    priv = torch.empty((n, 4), dtype=torch.int64, device=dev)
    t0 = time.perf_counter()
    r = DeviceResolver(pts, 0)
    t_create = time.perf_counter() - t0
    st = torch.cuda.current_stream(dev)
    try:
        def call():
            r.run_raw(p.data_ptr(), n, key.data_ptr(), priv.data_ptr(), st.cuda_stream)
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        times = []
        for _ in range(reps):
            t0 = time.perf_counter()
            call()
            st.synchronize()
            times.append(time.perf_counter() - t0)
        hits = int((key.cpu().numpy().view(np.uint32) != 0xFFFFFFFF).sum())
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
        ks_us = [e.device_time for e in prof.events() if "wt_resolve_pairs_kernel" in e.name]
    finally:
        r.close()
    host_us = None
    if os.path.exists(INGEST):
        from kangaroo_b200.ingest import DPTable
        t = DPTable(threads=1)
        kt = DPTable.key_table(pts)
        sample = pairs[:max(200, min(2000, 200000 // n_keys))]
        t0 = time.perf_counter()
        for a, b in sample:
            t.resolve_multi((a & M64, a >> 64), (b & M64, b >> 64), kt, 0)
        host_us = 1e6 * (time.perf_counter() - t0) / len(sample)
        t.close()
    return dict(keys=n_keys, collisions=n, hits=hits, create_ms=round(1e3 * t_create, 2),
                call_us_per_collision=round(1e6 * statistics.median(times) / n, 4),
                kernel_us_per_collision=round(statistics.median(ks_us) / n, 4) if ks_us else None,
                kernel_launches_traced=len(ks_us), host_us_per_collision=None if host_us is None else round(host_us, 2))


def add_rates(n_keys, records, events, reps, rng, torch):
    """one step's add, plain and resolving, alternated on a fresh pair of tables per repetition"""
    from kangaroo_b200.ingest import DeviceDPTable, DeviceResolver
    ks, pts = keys_of(n_keys, rng)
    pairs = pairs_of(events, ks, rng)
    h = rng.integers(0, 1 << 18, size=records).astype(np.uint64)
    base = np.zeros((records, 5), dtype=np.uint64)
    base[:, 0] = np.arange(records, dtype=np.uint64) | (h << np.uint64(32))
    base[:, 1] = rng.integers(0, 1 << 63, size=records, dtype=np.uint64)
    base[:, 2] = rng.integers(0, 1 << 63, size=records, dtype=np.uint64)
    step = base.copy()                           # the step: the first `events` records collide with the table's entries
    step[:, 1] ^= np.uint64(1)
    step[:events, 1] = base[:events, 1]
    for i, (a, b) in enumerate(pairs):
        base[i, 3], base[i, 4] = a & M64, a >> 64
        step[i, 3], step[i, 4] = b & M64, b >> 64
    dev = torch.device("cuda", 0)
    bufs = [torch.from_numpy(x.view(np.uint8).reshape(-1)).to(dev) for x in (base, step)]
    r = DeviceResolver(pts, 0)
    s = torch.cuda.Stream(device=dev)
    times = {"plain": [], "resolve": []}
    try:
        for rep in range(reps + 2):
            for kind in ("plain", "resolve") if rep % 2 == 0 else ("resolve", "plain"):
                t = DeviceDPTable(4 * records, max_events=4096)
                t.reserve(records)
                t.add(bufs[0].data_ptr(), [records], records, s.cuda_stream)
                res = r if kind == "resolve" else None
                t0 = time.perf_counter()
                ev = t.add(bufs[1].data_ptr(), [records], records, s.cuda_stream, resolver=res)
                dt = time.perf_counter() - t0
                t.close()
                assert len(ev) == min(events, 4096)
                if rep >= 2:
                    times[kind].append(dt)
    finally:
        r.close()
    return dict(keys=n_keys, records=records, collision_events=events,
                plain_ms=round(1e3 * statistics.median(times["plain"]), 3), resolve_ms=round(1e3 * statistics.median(times["resolve"]), 3))


def ingest_ms(table, steps):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver", CFG64, "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "3",
                        "--max-steps", str(steps), "--dp-table", table], capture_output=True, text=True, timeout=1800, cwd=ROOT)
    out = p.stdout + p.stderr
    m = re.search(r"rank-0 [a-z ]+ ([0-9.]+) ms/step", out)
    b = re.search(r"Batch: (\d+)/(\d+) keys solved", out)
    return dict(table=table, rc=p.returncode, ingest_ms_per_step=float(m.group(1)) if m else None,
                keys_solved=int(b.group(1)) if b else None, tail=None if m else out[-600:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 16, help="collisions per resolver call")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--records", type=int, default=1 << 17, help="records of one step's add")
    ap.add_argument("--events", type=int, default=1024, help="collision events of that add")
    ap.add_argument("--steps", type=int, default=300, help="--max-steps of the solver runs (0: skip them)")
    a = ap.parse_args()
    import torch
    print("card: %s" % card(), flush=True)
    rng = np.random.default_rng(1)
    res = dict(card=card(), resolver=[], add=[], ingest=[])
    for n_keys in (1, 64, 1024, 65535):
        res["resolver"].append(resolver_rates(n_keys, a.n, a.reps, rng, torch))
        print(json.dumps(res["resolver"][-1]), flush=True)
    for n_keys in (1, 64):
        res["add"].append(add_rates(n_keys, a.records, a.events, a.reps, rng, torch))
        print(json.dumps(res["add"][-1]), flush=True)
    if a.steps:
        for table in ("device", "host") if os.path.exists(INGEST) else ("device",):
            res["ingest"].append(ingest_ms(table, a.steps))
            print(json.dumps(res["ingest"][-1]), flush=True)
    res["card_after"] = card()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
