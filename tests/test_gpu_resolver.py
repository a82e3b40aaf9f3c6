"""-m gpu: the persistent collision resolver (kgx_resolver_*, ingest.DeviceResolver), the device table's resolving add
(kgx_dptable_add_resolve) and the solver and worktool without build/libkgx_ingest.so.

The resolver is checked against a model on ecmath (the first key in input order that +-m1*G or +-m2*G hits, m1 = |Td| + |Wd|,
m2 = ||Td| - |Wd||, and its private key), against kgx_work_resolve and, where the library exists, against the host's
kgi_resolve_multi, at 1 to 65535 keys with known scalars.  The solver runs point KGX_INGEST_LIB at a path that does not exist,
as a checkout built without the reference sources, and must find the same keys as the runs with the library."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200 import worktool as wt
from tests.ranks_util import ROOT, run_ranks
from tests.test_gpu_batch_merge import M126, SIGN, collisions, key_table
from tests.test_gpu_dp_table import ev_tuple, random_recs, same_x
from tests.worktool_util import TYPE_BIT, crafted_pair

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
has_ingest = os.path.exists(INGEST)
NO_LIB = dict(os.environ, KGX_INGEST_LIB=os.path.join(ROOT, "build", "no_such_libkgx_ingest.so"))
PRIV56 = "Priv: 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD612C0F05F3DA03"
M64 = (1 << 64) - 1


def limbs(v):
    return (v & M64, v >> 64)


# ---- the model ------------------------------------------------------------------------------------------------------------
def keys_for(n, rng):
    """n keys with known scalars: tests.test_gpu_batch_merge.key_table's, whose specials (a key listed twice, a negative, the
    point at infinity, 2^126 + 5) start at 64 keys, and past 64 keys key 5 again next to last and a key of its own last; below
    that, for 7 to 63 keys, the same specials at indices 3 to 6 -- key 1 again, the negative of key 2, the point at infinity,
    2^126 + 5"""
    ks, pts = key_table(n, rng)
    if n > 64:
        ks[n - 2], pts[n - 2] = ks[5], pts[5]
        ks[n - 1], pts[n - 1] = ks[n - 3] + 2, ec.add(pts[n - 3], ec.mul(2))
    if 7 <= n < 64:
        ks[3], pts[3] = ks[1], pts[1]
        ks[4], pts[4] = ec.N - ks[2], ec.neg(pts[2])
        ks[5], pts[5] = 0, None
        ks[6], pts[6] = (1 << 126) + 5, ec.mul((1 << 126) + 5)
    return ks, pts


def model(pairs, pts, start):
    """the expected [(key index, private key) or None] of each (d_first, d_other) pair"""
    by_x = {}
    for i, p in enumerate(pts):
        by_x.setdefault(None if p is None else p[0], []).append(i)
    cache = {}

    def mul(m):
        if m not in cache:
            cache[m] = ec.mul(m) if m % ec.N else None
        return cache[m]

    out = []
    for a, b in pairs:
        if not ((a ^ b) >> 126) & 1:
            out.append(None)                                         # one herd
            continue
        t, w = a & M126, b & M126
        best = None
        for m in (t + w, abs(t - w)):
            P = mul(m)
            for i in by_x.get(None if P is None else P[0], []):
                s = m if pts[i] == P else ec.N - m                   # K = P or K = -P (the same x)
                if best is None or i < best[0]:
                    best = (i, (s + start) % ec.N)
                break                                                # the first key of that x in input order
        out.append(best)
    return out


def device_resolve(pts, start, pairs, stream=None):
    from kangaroo_b200.ingest import DeviceResolver
    r = DeviceResolver(pts, start)
    try:
        return r.resolve([a for a, _ in pairs], [b for _, b in pairs], stream=stream)
    finally:
        r.close()


@pytest.mark.parametrize("n", [1, 7, 8, 9, 64, 1024, 65535])
def test_resolver_equals_the_model_and_the_one_call_resolver(n):
    rng = np.random.default_rng(100 + n)
    ks, pts = keys_for(n, rng)
    pairs = collisions(ks, rng)
    t = w = (1 << 125) + 77                                          # m1 = 2^126 + 154 and m2 = 0 on the wild side too
    pairs += [(t | TYPE_BIT, w), (t | SIGN, w | TYPE_BIT | SIGN), (0, TYPE_BIT), (TYPE_BIT, 0)]
    pairs += [(ks[j] + 999, 999 | TYPE_BIT) for j in range(min(n, 4))]   # keys 1 to 3 below 64 keys: 3 is key 1 again
    for start in ((0x1234 << 120) + 99, ec.N - 3, 0):
        want = model(pairs, pts, start)
        got = device_resolve(pts, start, pairs)
        assert got == want
        assert wt.resolve([a for a, _ in pairs], [b for _, b in pairs], pts, start) == want
        hits = [g for g in want if g is not None]
        assert len(hits) >= 12 and len(hits) < len(pairs)           # pairs that match no key are there too
        for i, priv in hits:
            assert (priv - start) % ec.N == ks[i] % ec.N
        found = {i for i, _ in hits}
        assert n - 1 in found                                        # the last key
        if 7 <= n < 64:
            assert {0, 1, 2, 5, 6} <= found and not found & {3, 4}  # the point at infinity, 2^126 + 5; later copies never
        if n >= 64:
            assert {0, 3, 4, 5, 11, 12, 63} <= found and not found & {9, 10, n - 2 if n > 64 else 9}
        if has_ingest:
            from kangaroo_b200.ingest import DPTable
            h = DPTable(threads=1)
            try:
                kt = DPTable.key_table(pts)
                assert [h.resolve_multi(limbs(a), limbs(b), kt, start) for a, b in pairs] == want
            finally:
                h.close()


def test_a_run_behind_other_work_on_a_side_stream():
    """the pairs are written on a side stream behind a long kernel, and the run is queued on that stream right behind them:
    a run on any other stream would read the zeros the buffer held before"""
    import torch
    from kangaroo_b200.ingest import DeviceResolver, _limbs_u64
    rng = np.random.default_rng(5)
    ks, pts = keys_for(64, rng)
    pairs = collisions(ks, rng)
    start = 12345
    want = model(pairs, pts, start)
    n = len(pairs)
    host = torch.from_numpy(np.hstack([_limbs_u64([a for a, _ in pairs], 2), _limbs_u64([b for _, b in pairs], 2)]).view(np.int64)).pin_memory()
    dev = torch.zeros_like(host, device="cuda")
    key = torch.full((n,), 0x5A5A, dtype=torch.int32, device="cuda")
    priv = torch.full((n, 4), 0x5A5A, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    r = DeviceResolver(pts, start)
    side = torch.cuda.Stream()
    try:
        with torch.cuda.stream(side):
            torch.cuda._sleep(200_000_000)                           # about 0.1 s of spinning on the side stream
            dev.copy_(host, non_blocking=True)
            r.run_raw(dev.data_ptr(), n, key.data_ptr(), priv.data_ptr(), side.cuda_stream)
        side.synchronize()
    finally:
        r.close()
    k, p = key.cpu().numpy().view(np.uint32), priv.cpu().numpy().view(np.uint64)
    got = [None if kk == 0xFFFFFFFF else (int(kk), sum(int(v) << (64 * w) for w, v in enumerate(pp))) for kk, pp in zip(k.tolist(), p)]
    assert got == want


def test_bad_arguments_are_refused():
    from kangaroo_b200.ingest import DeviceResolver
    with pytest.raises(RuntimeError, match="not below n"):
        DeviceResolver([ec.G], ec.N)
    with pytest.raises(RuntimeError, match="n_keys"):
        DeviceResolver(np.zeros((0, 8), dtype=np.uint64), 0)
    assert device_resolve([ec.G], 0, []) == []


# ---- the resolving add -----------------------------------------------------------------------------------------------------
def hitting(rng, ks, n, h_pool):
    """n pairs of records at one x: a tame one at d = k + w, then a wild one at w (and some the other way round, and some that
    match no key), each pair in a bucket of h_pool"""
    first, later = [], []
    for i in range(n):
        j = int(rng.integers(0, len(ks)))
        w = int(rng.integers(0, 1 << 62)) << 40
        k = ks[j] if ks[j] < 1 << 125 else 12345
        if i % 5 == 4:
            k += 1 << 100                                            # matches no key (almost surely)
        a, b = (k + w) | (SIGN if i % 3 == 0 else 0), w | TYPE_BIT | (SIGN if i % 2 else 0)
        if i % 4 == 1:
            a, b = b, a
        h = int(rng.choice(h_pool))
        x0, x1 = int(rng.integers(0, 1 << 63)), (int(rng.integers(0, 1 << 31)) << 32) | h
        first.append([i | (h << 32), x0, x1, a & M64, a >> 64])
        later.append([(i + 1000) | (h << 32), x0, x1, b & M64, b >> 64])
    return np.array(first, dtype=np.uint64), np.array(later, dtype=np.uint64)


def test_resolving_add_equals_the_plain_add(tmp_path):
    """the crafted records of tests/test_gpu_dp_table.py (new entries, same-herd and cross-herd copies, duplicates, several
    rank segments, more events than the cap), plus pairs that hit keys: the same events, counts and saved bytes as the plain
    add, and every collision's key and private key the resolver's"""
    import torch
    from kangaroo_b200.ingest import DeviceDPTable, DeviceResolver, EV_COLLISION
    rng = np.random.default_rng(11)
    ks, pts = keys_for(64, rng)
    start = (0x77 << 100) + 5
    cap = 1 << 11
    plain, fused = DeviceDPTable(1 << 22, max_events=cap), DeviceDPTable(1 << 22, max_events=cap)
    r = DeviceResolver(pts, start)
    pool = rng.integers(0, 1 << 18, size=64)
    base = random_recs(rng, 20000)
    f1, l1 = hitting(rng, ks, 300, pool)
    batches = [[base[:7000], f1], [base[7000:], same_x(base[:1000], rng, True), same_x(base[1000:2500], rng, False)],
               [l1[:150], base[:500], random_recs(rng, 2000, pool)], [l1[150:], same_x(base[10000:14500], rng, False)]]
    seen_hits = 0
    try:
        for segs in batches:
            stride = max(len(s) for s in segs) + 3
            flat = np.zeros((len(segs) * stride, 5), dtype=np.uint64)
            for k, s in enumerate(segs):
                flat[k * stride:k * stride + len(s)] = s
            buf = torch.from_numpy(flat.view(np.uint8).reshape(-1)).cuda()
            counts = [len(s) for s in segs]
            rc_p, n_p, ev_p = plain.add_raw(buf.data_ptr(), counts, stride)
            rc_f, n_f, ev_f = fused.add_raw(buf.data_ptr(), counts, stride, resolver=r)
            assert (rc_f, n_f, len(fused)) == (rc_p, n_p, len(plain))
            m = min(n_p, cap)
            assert [ev_tuple(ev_f[i].ev) for i in range(m)] == [ev_tuple(ev_p[i]) for i in range(m)]
            coll = [i for i in range(m) if ev_p[i].kind == EV_COLLISION]
            pairs = [(int(ev_p[i].d_old[0]) | int(ev_p[i].d_old[1]) << 64, int(ev_p[i].d_new[0]) | int(ev_p[i].d_new[1]) << 64) for i in coll]
            want = dict(zip(coll, r.resolve([a for a, _ in pairs], [b for _, b in pairs])))
            for i in range(m):
                e = ev_f[i]
                got = None if e.key == 0xFFFFFFFF else (int(e.key), sum(int(e.priv[w]) << (64 * w) for w in range(4)))
                assert got == want.get(i), i
            hits = [(a, b, want[i]) for (a, b), i in zip(pairs, coll) if want[i] is not None]
            assert [h for _, _, h in hits] == model([(a, b) for a, b, _ in hits], pts, start)
            seen_hits += len(hits)
        assert seen_hits >= 200 and n_p > cap
        hdr = dict(dp_bits=9, range_start=start, range_end=start + (1 << 60), pubkey=ec.G, total_count=7, total_time=1.5, total_walk=0)
        a, b = str(tmp_path / "plain.work"), str(tmp_path / "fused.work")
        plain.save_work(a, **hdr)
        fused.save_work(b, **hdr)
        assert open(a, "rb").read() == open(b, "rb").read()
        evs = fused.add(buf.data_ptr(), counts, stride, resolver=r)          # the tuples the solver reads (the last batch again)
        assert len(evs) == min(sum(counts), cap) and all(len(e) == 6 for e in evs)
        coll = [e for e in evs if e[0] == EV_COLLISION]
        assert all(e[5] is None for e in evs if e[0] != EV_COLLISION)
        assert [e[5] for e in coll] == r.resolve([e[3][0] | e[3][1] << 64 for e in coll], [e[4][0] | e[4][1] << 64 for e in coll])
        assert sum(e[5] is not None for e in coll) >= 100
    finally:
        plain.close()
        fused.close()
        r.close()


def test_more_events_than_the_cap():
    """a call with more events than the cap returns the first cap of them, each resolved"""
    import torch
    from kangaroo_b200.ingest import DeviceDPTable, DeviceResolver
    rng = np.random.default_rng(12)
    ks, pts = keys_for(8, rng)
    cap = 100
    plain, fused = DeviceDPTable(1 << 20, max_events=cap), DeviceDPTable(1 << 20, max_events=cap)
    r = DeviceResolver(pts, 0)
    first, later = hitting(rng, ks, 700, rng.integers(0, 1 << 18, size=8))
    try:
        for segs in ([first], [later]):
            buf = torch.from_numpy(np.ascontiguousarray(segs[0]).view(np.uint8).reshape(-1)).cuda()
            rc_p, n_p, ev_p = plain.add_raw(buf.data_ptr(), [len(segs[0])], len(segs[0]))
            rc_f, n_f, ev_f = fused.add_raw(buf.data_ptr(), [len(segs[0])], len(segs[0]), resolver=r)
            assert (rc_f, n_f) == (rc_p, n_p)
            m = min(n_p, cap)
            assert [ev_tuple(ev_f[i].ev) for i in range(m)] == [ev_tuple(ev_p[i]) for i in range(m)]
        assert n_p == 700
        pairs = [(int(e.ev.d_old[0]) | int(e.ev.d_old[1]) << 64, int(e.ev.d_new[0]) | int(e.ev.d_new[1]) << 64) for e in ev_f[:cap]]
        got = [None if e.key == 0xFFFFFFFF else (int(e.key), sum(int(e.priv[w]) << (64 * w) for w in range(4))) for e in ev_f[:cap]]
        assert got == model(pairs, pts, 0) and sum(g is not None for g in got) >= 40
    finally:
        plain.close()
        fused.close()
        r.close()


# ---- the solver and worktool without the library ---------------------------------------------------------------------------
def solver(args, env, timeout=900):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT,
                       env=env)
    return p.returncode, p.stdout + p.stderr


def privs(out):
    return re.findall(r"Priv: 0x[0-9A-F]+", out)


IN56 = [os.path.join(GOLD, "in56.txt"), "--dp", "8", "--grid", "32,128", "--seed", "7"]


@pytest.mark.parametrize("table", ["device", "sharded"])
def test_solver_in56_without_the_ingest_library(table):
    rc, out = solver(IN56 + ["--dp-table", table, "--dp-table-capacity", str(1 << 24)], NO_LIB)
    assert rc == 0 and PRIV56 in out, out[-2000:]
    if has_ingest and table == "device":                             # the same run with the library: the same key, exit code
        rc2, out2 = solver(IN56 + ["--dp-table", table, "--dp-table-capacity", str(1 << 24)], os.environ)
        assert (rc2, privs(out2)) == (rc, privs(out))


def test_host_table_without_the_library_names_the_device_tables():
    rc, out = solver(IN56 + ["--dp-table", "host"], NO_LIB, timeout=300)
    assert rc == 2 and "--dp-table device" in out and "--dp-table sharded" in out and "no_such_libkgx_ingest.so" in out, out[-2000:]


def test_batch_keys_without_the_ingest_library():
    answers = [int(v, 16) for v in open(os.path.join(GOLD, "in56_64keys.answers.txt")).read().split()]
    rc, out = solver([os.path.join(GOLD, "in56_64keys.txt"), "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "3",
                      "--dp-table", "device"], NO_LIB)
    assert rc == 0, out[-3000:]
    got = {int(i): int(v, 16) for i, v in re.findall(r"Key#\s*(\d+) Pub:\s+0x[0-9A-F]+\s+Priv: 0x([0-9A-F]+)", out)}
    assert got == dict(enumerate(answers)), out[-3000:]


def test_resume_of_a_host_table_file_under_the_device_table(tmp_path):
    """ref_work48: a file the reference's own HashTable wrote"""
    import gzip
    import shutil
    from tests.golden import make_work_golden as g
    path = str(tmp_path / "ref.work")
    with gzip.open(os.path.join(GOLD, "ref_work48.work.gz"), "rb") as src, open(path, "wb") as dst:
        shutil.copyfileobj(src, dst)
    rc, out = solver(["--resume", path, "--grid", "8,32", "--seed", "1", "--dp", "10", "--max-steps", "20000", "--dp-table", "device",
                      "--dp-table-capacity", str(1 << 22)], NO_LIB, timeout=600)
    assert "1024 kangaroos imported and verified" in out, out[-2000:]
    assert rc == 0 and "Priv: 0x%X" % g.PRIV in out, out[-2000:]


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_ranks_without_the_ingest_library(world, monkeypatch):
    monkeypatch.setenv("KGX_INGEST_LIB", NO_LIB["KGX_INGEST_LIB"])
    rcs, outs = run_ranks(world, IN56[:-1] + [str(7 + world), "--dp-table", "sharded", "--dp-table-capacity", str(1 << 23)], timeout=600)
    assert rcs == [0] * world, "".join(o[-2000:] for o in outs)
    assert PRIV56 in outs[0] and "GPUs: %d" % world in outs[0], outs[0][-2000:]
    assert all("Traceback" not in o for o in outs)


def test_worktool_merge_without_the_ingest_library(tmp_path):
    from tests.golden import make_work_golden as g
    pa, pb = crafted_pair(tmp_path)
    runs = []
    for env in ([NO_LIB, os.environ] if has_ingest else [NO_LIB]):
        dest = str(tmp_path / "found.work")
        p = subprocess.run([sys.executable, "-m", "kangaroo_b200.worktool", "merge", pa, pb, "-o", dest], capture_output=True, text=True,
                           timeout=600, cwd=ROOT, env=env)
        assert p.returncode == 0 and "Priv: 0x%X" % g.PRIV in p.stdout, p.stdout + p.stderr
        assert not os.path.exists(dest)
        runs.append(p.stdout.replace(str(tmp_path), ""))
    assert len(set(runs)) == 1
