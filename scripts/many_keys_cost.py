"""Cost per solved key of --batch-keys at up to 65535 keys, on one GPU and the default herd:
  - kgx_retarget with n_to = 1k, 4k, 16k and 65534 destinations: the call's host time (it returns without waiting for the
    device), call + sync with nothing else queued, and the device time of its kernels (retarget_delta_kernel, one launch per
    1024 destinations, and retarget_kernel, one pass over the herd) from torch.profiler in a pass of its own;
  - the host mirror of one retarget (solver.retarget_targets) on the same herd;
  - BatchSolver._claim of one 4-key class through solver.class_members at 65535 keys, against the scan over all keys;
  - worktool check of a batch file whose wild entries match no key (every key is tried) against the number of keys.
Prints the card and its power limit first, then one JSON line per measurement.

    python scripts/many_keys_cost.py [--reps 5]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NK = 65535
RP = 64
WDIV2 = ((1 << RP) - 1) >> 1


def emit(**kw):
    print(json.dumps(kw), flush=True)


def retarget_costs(orc, keys, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from kangaroo_b200 import GPUEngine, random_herd_arrays
    from kangaroo_b200.solver import assign_targets, retarget_targets
    gx, gy = GPUEngine.GetGridSize(0, 0, 0)
    eng = GPUEngine(gx, gy, 0, 1 << 16)
    n = eng.nbKangaroo
    eng.SetWildOffset(WDIV2)
    eng.SetParams(orc.dp_mask(16), *orc.create_jump_table(RP))
    sc, d128 = random_herd_arrays(n, RP, WDIV2, np.random.default_rng(1))
    live = list(range(NK))
    targets = assign_targets(n, live)
    eng.CreateHerdMulti(sc, d128, keys, targets)
    emit(what="herd", grid=[gx, gy], kangaroos=n, kernel=eng.kernel, keys=NK, wilds_per_key=n // 2 / NK)
    frm = 0
    for n_to in (1024, 4096, 16384, NK - 1):
        to = [k for k in range(1, n_to + 1)]
        call, total, mirror = [], [], []
        for r in range(reps + 1):                      # the first is a warm-up
            eng.sync()
            t = time.perf_counter()
            eng.Retarget(frm, to)
            t1 = time.perf_counter()
            eng.sync()
            t2 = time.perf_counter()
            tt = time.perf_counter()
            targets = retarget_targets(targets, frm, to)  # the mirror follows the engine, as the solver keeps it
            t3 = time.perf_counter()
            if r:
                call.append(t1 - t)
                total.append(t2 - t)
                mirror.append(t3 - tt)
            frm, to = to[0], [frm] + to[1:]            # move the wilds back and forth: every call moves a key's wilds
        assert np.array_equal(eng.Targets(), targets)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                eng.Retarget(frm, to)
                targets = retarget_targets(targets, frm, to)
                frm, to = to[0], [frm] + to[1:]
            eng.sync()
            torch.cuda.synchronize()
        dev = {}
        for ev in prof.key_averages():
            if "retarget" in ev.key:
                dev[ev.key.split("(")[0].split("<")[0].strip()] = (ev.count, ev.device_time_total / 1e3)
        emit(what="kgx_retarget", n_to=n_to, call_ms=1e3 * float(np.median(call)), call_sync_ms=1e3 * float(np.median(total)),
             device_ms_per_call={k: c_ms[1] / reps for k, c_ms in dev.items()}, launches_per_call={k: c[0] / reps for k, c in dev.items()},
             host_mirror_ms=1e3 * float(np.median(mirror)), reps=reps)
    eng.close()


def claim_cost(reps):
    """_claim of one class of 4 keys (two copies and a negative) at 65535 keys through the member list, against the scan over
    every key that it replaced, both giving the 4 keys their private keys; median of reps each"""
    from kangaroo_b200.solver import BatchSolver, class_members, class_privs, key_classes
    p = (1 << 256) - 0x1000003D1
    keys = [(i + 1, 2 * i + 3) for i in range(NK)]
    r0 = 1000
    for i in (20000, 40000, NK - 1):
        keys[i] = keys[r0] if i != 40000 else (keys[r0][0], p - keys[r0][1])
    rep, neg = key_classes(keys)
    s = BatchSolver.__new__(BatchSolver)
    s.start, s.rep, s.neg, s.members = 1, rep, neg, class_members(rep)
    assert len(s.members[r0]) == 4
    member, scan = [], []
    for _ in range(reps):
        s.priv, s._announce = [None] * NK, []
        t = time.perf_counter()
        s._claim([(r0, 5, 0, 1)], [])
        member.append(time.perf_counter() - t)
        priv = [None] * NK
        t = time.perf_counter()
        priv[r0] = class_privs(1, 5, False)
        for i in range(NK):
            if rep[i] == r0:
                priv[i] = class_privs(1, priv[r0], neg[i])
        scan.append(time.perf_counter() - t)
        assert priv == s.priv
    emit(what="claim_one_class", keys=NK, class_keys=4, member_list_us=1e6 * float(np.median(member)),
         full_scan_us=1e6 * float(np.median(scan)), reps=reps)


def headw(start, end, pub, buckets):
    """a HEADW work file (dp 16, no kangaroos): header, then the 2^18 buckets {count, maxItem, entries sorted by x}"""
    l4 = lambda v: int(v).to_bytes(32, "little")
    out = [struct.pack("<III", 0xFA6A8001, 0, 16), l4(start), l4(end), l4(pub[0]), l4(pub[1]), struct.pack("<Qd", 0, 0.0)]
    for h in range(1 << 18):
        b = sorted(buckets.get(h, []))
        out.append(struct.pack("<II", len(b), (len(b) + 3) // 4 * 4))
        out.extend(x.to_bytes(16, "little") + d.to_bytes(16, "little") for x, d in b)
    out.append(struct.pack("<Q", 0))
    return b"".join(out)


def check_costs(orc, reps):
    from kangaroo_b200 import worktool as wt
    rng = np.random.default_rng(7)
    pubs_all = [orc.ec_mul_g(int(v)) for v in rng.integers(1 << 40, 1 << 62, size=NK)]
    n_ent = 1024
    # wild entries {x lo 128, d tagged wild (bit 126), both signs (bit 127)} at random points: none matches a key
    ents = {}
    for i in range(n_ent):
        d = int(rng.integers(1, 1 << 62)) | (1 << 126) | ((i & 1) << 127)
        ents.setdefault(int(rng.integers(0, 1 << 18)), []).append((int(rng.integers(1, 1 << 62)) << 64 | i, d))
    tmp = tempfile.mkdtemp()
    for nk in (1, 64, 1024, 8192, NK):
        plain = headw(1, 1 << 64, pubs_all[0], ents)
        path = os.path.join(tmp, "k%d.work" % nk)
        with open(path, "wb") as f:
            f.write(plain + wt.batch_block(wt.BatchBlock(pubs_all[:nk], [False] * nk, [None] * nk, []), len(plain)).tobytes())
        wt.check(path)                                 # warm-up
        times = []
        for _ in range(reps):
            t = time.perf_counter()
            r = wt.check(path)
            times.append(time.perf_counter() - t)
        assert r.n_keys == nk and r.wrong_entries == n_ent
        s = float(np.median(times))
        emit(what="worktool_check", keys=nk, wild_entries=n_ent, seconds=s, entry_keys_per_s=n_ent * nk / s, reps=reps)
        os.remove(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    from oracle import kgo
    orc = kgo.Oracle()
    rng = np.random.default_rng(3)
    t = time.perf_counter()
    keys = [orc.ec_mul_g(int(v) | (1 << 62)) for v in rng.integers(1, 1 << 62, size=NK)]
    emit(what="keys", keys=NK, seconds=time.perf_counter() - t)
    retarget_costs(orc, keys, a.reps)
    claim_cost(a.reps)
    check_costs(orc, a.reps)


if __name__ == "__main__":
    main()
