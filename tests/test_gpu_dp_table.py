"""-m gpu: the device-resident DP table (kgx_dptable_*, ingest.DeviceDPTable) against the host table of the reference's
HashTable (kgi_add, ingest.DPTable) fed the same records in the same order -- events, counts and work files byte for byte --
and the solver's --dp-table device end to end."""
import ctypes
import gzip
import hashlib
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests.worktool_util import Work

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
DROPIN = os.path.join(ROOT, "build", "kangaroo_b200")
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")

NB = 1 << 18
TYPE = np.uint64(1 << 62)
HDR = dict(dp_bits=9, range_start=0x1234 << 70, range_end=(0x1234 << 70) + (1 << 60), pubkey=(0xABCDEF << 100, 0x777 << 50),
           total_count=123456789, total_time=42.5, total_walk=0)
PRIV56 = "Priv: 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD612C0F05F3DA03"


# ---- records and the two tables --------------------------------------------------------------------------------------
def random_recs(rng, n, buckets=None):
    """n x 5 uint64 = n 40-byte DP records {u32 kIdx, u32 h, x[2], d[2]} with random content (d's b126 = herd type)"""
    a = rng.integers(0, 1 << 63, size=(n, 5), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 5), dtype=np.uint64)
    h = rng.integers(0, NB, size=n, dtype=np.uint64) if buckets is None else rng.choice(np.asarray(buckets, np.uint64), size=n)
    a[:, 0] = (a[:, 0] & np.uint64(0xFFFFFFFF)) | (h << np.uint64(32))
    return a


def same_x(recs, rng, same_type):
    """copies of recs with another distance: same herd (-> reset) or the other herd (-> collision)"""
    out = recs.copy()
    out[:, 3] = rng.integers(0, 1 << 63, size=len(out), dtype=np.uint64)
    out[:, 4] = (rng.integers(0, 1 << 62, size=len(out), dtype=np.uint64) & ~TYPE) | (recs[:, 4] & TYPE)
    if not same_type:
        out[:, 4] ^= TYPE
    return out


def ev_tuple(e):
    return (int(e.kind), int(e.rank), int(e.kidx), int(e.h), (int(e.d_old[0]), int(e.d_old[1])), (int(e.d_new[0]), int(e.d_new[1])))


class Pair:
    """a host table and a device table fed the same batches"""

    def __init__(self, capacity=1 << 22, cap=1 << 16, threads=8):
        from kangaroo_b200.ingest import DPTable, DeviceDPTable
        self.host = DPTable(threads=threads, max_events=1 << 20)
        self.dev = DeviceDPTable(capacity, max_events=cap)
        self.cap = cap

    def add(self, segments, first=None):
        """segments: one record array per rank (one step of a gather).  Checks events and counts, returns the events.
        first: the events the call must return, in arrival order, when it makes more than cap."""
        import torch
        host_ev, host_bad = [], False
        for r, seg in enumerate(segments):
            if len(seg) == 0:
                continue
            ne = ctypes.c_uint32(0)
            a = np.ascontiguousarray(seg)
            rc = self.host._lib.kgi_add(self.host._h, a.ctypes.data_as(ctypes.c_void_p), len(a), r, self.host._ev, self.host._cap, ctypes.byref(ne))
            host_bad |= rc != 0
            host_ev += [ev_tuple(self.host._ev[i]) for i in range(ne.value)]
        stride = max([len(s) for s in segments] + [1]) + 3          # a gather buffer: every rank at a multiple of the stride
        flat = np.zeros((len(segments) * stride, 5), dtype=np.uint64)
        for r, seg in enumerate(segments):
            flat[r * stride:r * stride + len(seg)] = seg
        buf = torch.from_numpy(flat.view(np.uint8).reshape(-1)).cuda()
        rc, n, evs = self.dev.add_raw(buf.data_ptr(), [len(s) for s in segments], stride)
        dev_ev = [ev_tuple(evs[i]) for i in range(min(n, self.cap))]
        assert rc == (-1 if host_bad else 0)
        assert n == len(host_ev)
        assert len(self.dev) == len(self.host)
        if n <= self.cap:
            assert sorted(dev_ev) == sorted(host_ev)
        else:                                                       # the first cap events (arrival order) of the same multiset
            assert len(dev_ev) == self.cap
            left = sorted(host_ev)
            for e in dev_ev:
                left.remove(e)
        if first is not None:
            assert dev_ev == first[:self.cap]
        # arrival order: the records whose (rank, kIdx, d) is unique in the call come back in the order they were sent
        order, seen = {}, set()
        for r, seg in enumerate(segments):
            for i, rec in enumerate(seg):
                k = (r, int(rec[0]) & 0xFFFFFFFF, int(rec[3]), int(rec[4]))
                order[k] = None if k in seen else (r, i)
                seen.add(k)
        idx = [order[(e[1], e[2], e[5][0], e[5][1])] for e in dev_ev]
        idx = [i for i in idx if i is not None]
        assert idx == sorted(idx)
        return host_ev

    def saves(self, tmp_path, **hdr):
        h, d = str(tmp_path / "host.work"), str(tmp_path / "dev.work")
        kw = dict(HDR, **hdr)
        self.host.save_work(h, **kw)
        self.dev.save_work(d, **kw)
        return h, d

    def close(self):
        self.host.close()
        self.dev.close()


def digest(path):
    m = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            m.update(blk)
    return m.hexdigest()


def table_entries(path):
    """(h, x0, x1, d0, d1) of every entry of a work file's table (a small file: parsed in Python)"""
    m64 = (1 << 64) - 1
    return [(h, x & m64, x >> 64, d & m64, d >> 64) for h, bucket in enumerate(Work.read(path).table) for x, d in bucket]


def as_recs(entries, rng, kidx0=0):
    a = np.zeros((len(entries), 5), dtype=np.uint64)
    for i, (h, x0, x1, d0, d1) in enumerate(entries):
        a[i] = [(kidx0 + i) | (h << 32), x0, x1, d0, d1]
    return a


# ---- 1, 2: semantics batch by batch, then the save ---------------------------------------------------------------------
@needs_ingest
def test_batches_match_the_host_table_and_the_saves_are_identical(tmp_path):
    rng = np.random.default_rng(11)
    p = Pair(cap=1 << 16)
    base = random_recs(rng, 30000)
    p.add([base[:10000], base[10000:20000], np.zeros((0, 5), np.uint64), base[20000:]])            # 4 ranks, one empty
    # planted exact duplicates (old and within the call), same-herd and tame/wild collisions, across and within calls
    fresh = random_recs(rng, 5000)
    ev = p.add([np.concatenate([base[:500], fresh[:2000]]),
                np.concatenate([same_x(base[500:900], rng, True), same_x(base[900:1300], rng, False), fresh[:300]]),
                np.concatenate([fresh[2000:], same_x(fresh[2000:2400], rng, False), same_x(fresh[2400:2600], rng, True)])])
    kinds = [e[0] for e in ev]
    assert kinds.count(2) == 400 + 400 and kinds.count(1) == 500 + 400 + 300 + 200
    # many records of one (h, x) in one call: the first is stored, every later one compared with it
    one = random_recs(rng, 1)
    many = np.repeat(one, 300, axis=0)
    many[1:] = same_x(many[1:], rng, True)
    many[100:200] = same_x(many[100:200], rng, False)
    many[250:] = many[0]
    p.add([many[:120], random_recs(rng, 50), many[120:]])
    # one bucket pushed past several maxItem reallocations: 16 + 4k, stored or not
    hot = int(rng.integers(0, NB))
    b1 = random_recs(rng, 70, buckets=[hot])
    p.add([b1[:40]])
    p.add([b1[40:], b1[:30], same_x(b1[5:25], rng, False)])
    p.add([random_recs(rng, 33, buckets=[hot]), b1[60:]])
    # a malformed h: skipped, the others inserted, the call returns -1 on both tables
    bad = random_recs(rng, 200)
    bad[17, 0] = (bad[17, 0] & np.uint64(0xFFFFFFFF)) | (np.uint64(NB + 5) << np.uint64(32))
    p.add([random_recs(rng, 10), bad])
    # more events than cap: 70000 duplicates of the first batch, each a reset with no d_old, returned in arrival order
    segs = [base[:25000], base[25000:30000], np.concatenate([base[:20000], base[:20000]])]
    first = [(1, r, int(rec[0]) & 0xFFFFFFFF, int(rec[0]) >> 32, (0, 0), (int(rec[3]), int(rec[4]))) for r, seg in enumerate(segs) for rec in seg]
    p.add(segs, first=first)
    assert len(p.dev) == len(p.host) > 35000
    h, d = p.saves(tmp_path)
    assert open(h, "rb").read() == open(d, "rb").read()
    # the saved buckets carry the reference's maxItem: the hot bucket's went past 16 several times
    w = Work.read(d)
    nb, mx = len(w.table[hot]), w.maxitem[hot]
    assert nb >= 103 and mx > nb and (mx - 16) % 4 == 0             # (a random record of another batch may share the bucket)
    p.close()


# ---- 3: a file the reference wrote ---------------------------------------------------------------------------------------
@needs_ingest
def test_load_the_reference_written_fixture(tmp_path):
    path = str(tmp_path / "ref.work")
    with gzip.open(os.path.join(GOLD, "ref_work48.work.gz"), "rb") as src, open(path, "wb") as dst:
        shutil.copyfileobj(src, dst)
    p = Pair(capacity=1 << 20)
    wh = p.host.load_work_ex(path)
    wd = p.dev.load_work_ex(path)
    assert len(p.dev) == len(p.host) > 0
    assert (wd.dp_bits, wd.range_start, wd.range_end, wd.key, wd.total_count, wd.total_time, wd.nb_walk, wd.walk_offset) == \
        (wh.dp_bits, wh.range_start, wh.range_end, wh.key, wh.total_count, wh.total_time, wh.nb_walk, wh.walk_offset)
    h, d = p.saves(tmp_path, total_walk=5)
    assert open(h, "rb").read() == open(d, "rb").read()
    # the same new batch: duplicates and both kinds of collision with the loaded entries, and new entries in their buckets
    rng = np.random.default_rng(5)
    loaded = table_entries(h)
    pick = [loaded[i] for i in rng.choice(len(loaded), size=min(600, len(loaded)), replace=False)]
    old = as_recs(pick, rng)
    ev = p.add([old[:200], same_x(old[200:400], rng, True), same_x(old[400:], rng, False),
                random_recs(rng, 3000, buckets=[e[0] for e in pick])])
    assert len(ev) == len(pick)                                    # one event per planted record
    h2, d2 = p.saves(tmp_path)
    assert open(h2, "rb").read() == open(d2, "rb").read()
    p.close()


# ---- 4: capacity -------------------------------------------------------------------------------------------------------
@needs_ingest
def test_a_full_table_refuses_the_call_and_changes_nothing(tmp_path):
    from kangaroo_b200.ingest import DPTable, TableFull
    rng = np.random.default_rng(3)
    p = Pair(capacity=1000)
    recs = random_recs(rng, 1100)
    p.add([recs[:600], recs[600:900]])
    before = open(p.saves(tmp_path)[1], "rb").read()
    with pytest.raises(TableFull, match="full"):
        p.dev.add_dp40(__import__("torch").from_numpy(recs[900:1100].view(np.uint8).reshape(-1)).cuda())
    assert len(p.dev) == 900
    assert open(p.saves(tmp_path)[1], "rb").read() == before       # nothing of the refused call went in
    p.add([recs[900:1000]])                                        # exactly to capacity
    assert len(p.dev) == 1000
    h, d = p.saves(tmp_path)
    assert open(h, "rb").read() == open(d, "rb").read()
    t = DPTable(threads=1)                                         # the host table reads the device table's file
    t.load_work_ex(d)
    assert len(t) == 1000
    t.close()
    # a file of more entries than the capacity is refused, and the table is left empty like any failed load
    from kangaroo_b200.ingest import DeviceDPTable
    small = DeviceDPTable(999)
    with pytest.raises(TableFull, match="capacity of 999"):
        small.load_work_ex(d)
    assert len(small) == 0
    small.close()
    p.close()


# ---- 5: scale ----------------------------------------------------------------------------------------------------------
@needs_ingest
def test_2p26_entries_save_like_the_host_table(tmp_path):
    rng = np.random.default_rng(26)
    n, batch = 1 << 26, 1 << 20
    p = Pair(capacity=n + (1 << 16), cap=4096)
    for i in range(n // batch):
        recs = random_recs(rng, batch)
        if i:
            recs[:1000] = prev[:1000]                              # a few duplicates per batch: 1000 fewer entries each time
        host = p.host
        ne = ctypes.c_uint32(0)
        assert host._lib.kgi_add(host._h, recs.ctypes.data_as(ctypes.c_void_p), batch, 0, host._ev, host._cap, ctypes.byref(ne)) == 0
        import torch
        rc, nev, _ = p.dev.add_raw(torch.from_numpy(recs.view(np.uint8).reshape(-1)).cuda().data_ptr(), [batch], batch)
        assert rc == 0 and nev == ne.value and len(p.dev) == len(host)
        prev = recs
    assert len(p.dev) == n - 1000 * (n // batch - 1)
    h, d = p.saves(tmp_path)
    assert os.path.getsize(h) == os.path.getsize(d) and digest(h) == digest(d)
    p.close()


# ---- 6: the solver -----------------------------------------------------------------------------------------------------
def solver(args, timeout=900, prefix=None):
    p = subprocess.run((prefix or [sys.executable]) + ["-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT)
    return p.returncode, p.stdout + p.stderr


DEV = ["--dp-table", "device", "--dp-table-capacity", str(1 << 24)]


@needs_ingest
def test_solver_device_table_in56_and_puzzle110_window():
    rc, out = solver([os.path.join(GOLD, "in56.txt"), "--dp", "8", "--grid", "32,128", "--seed", "7"] + DEV)
    assert rc == 0 and PRIV56 in out, out[-2000:]
    assert "dp table: device, capacity 16777216 entries" in out and "rank-0 device table" in out, out[-2000:]
    rc, out = solver([os.path.join(GOLD, "puzzle110_window56.txt"), "--dp", "8", "--grid", "32,128", "--seed", "11", "--dp-table", "device"])
    assert rc == 0 and "Priv: 0x35C0D7234DF7DEB0F20CF7062444" in out, out[-2000:]


@needs_ingest
def test_solver_device_table_batch_keys():
    answers = [int(v, 16) for v in open(os.path.join(GOLD, "in56_64keys.answers.txt")).read().split()]
    rc, out = solver([os.path.join(GOLD, "in56_64keys.txt"), "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "3",
                      "--dp-table", "device"])                      # ~26 M DPs: the default capacity
    assert rc == 0, out[-3000:]
    privs = {int(i): int(v, 16) for i, v in re.findall(r"Key#\s*(\d+) Pub:\s+0x[0-9A-F]+\s+Priv: 0x([0-9A-F]+)", out)}
    assert privs == dict(enumerate(answers)), out[-3000:]
    m = re.search(r"Batch: (\d+)/(\d+) keys solved, (\d+) jumps", out)
    assert m and int(m.group(1)) == int(m.group(2)) == 64, out[-3000:]
    assert int(m.group(3)) < 0.5 * 64 * 2.08 * 2 ** 28            # under half of 64 single-key runs


@needs_ingest
def test_solver_device_table_on_two_gpus():
    """two GPUs, or two ranks sharing one over gloo"""
    from tests.ranks_util import solver_on
    rc, out = solver_on(2, [os.path.join(GOLD, "in56.txt"), "--dp", "8", "--grid", "32,128", "--seed", "8"] + DEV)
    assert rc == 0 and PRIV56 in out and "GPUs: 2" in out, out[-3000:]


COMMON = ["--dp", "8", "--grid", "8,32", "--seed", "5", "--save-kangaroos"]


@needs_ingest
def test_work_files_cross_between_the_tables(tmp_path):
    """device save -> host resume and host save -> device resume both solve; the same straight run saves the same file with
    either table; the drop-in binary's checker accepts the device table's file"""
    cfg = os.path.join(GOLD, "in56.txt")
    a, b = str(tmp_path / "dev.work"), str(tmp_path / "host.work")
    rc, out = solver([cfg, "--max-steps", "4", "--save-work", a] + COMMON + DEV)
    assert os.path.exists(a) and "work file written" in out, out[-2000:]
    rc, out2 = solver([cfg, "--max-steps", "4", "--save-work", b] + COMMON)
    assert os.path.exists(b), out2[-2000:]
    ra, rb = open(a, "rb").read(), open(b, "rb").read()
    if " 0 dead kangaroos re-created" in out and " 0 dead kangaroos re-created" in out2:
        assert ra[:148] == rb[:148] and ra[156:] == rb[156:]       # all but the header's run time
    else:                                                          # re-created kangaroos draw in event order: the tables still agree
        assert ra[:140] == rb[:140]
    rc, out = solver(["--resume", a, "--grid", "16,32", "--seed", "2"])
    assert "imported and verified" in out and PRIV56 in out, out[-2000:]
    rc, out = solver(["--resume", b, "--grid", "16,32", "--seed", "2"] + DEV)
    assert "imported and verified" in out and PRIV56 in out, out[-2000:]
    if os.path.exists(DROPIN):
        chk = subprocess.run([DROPIN, "-wcheck", a], capture_output=True, text=True, timeout=600, cwd=ROOT).stdout
        assert "[100.000% OK]" in chk and "Wrong" not in chk, chk[-1500:]


@needs_ingest
def test_resume_file_larger_than_the_capacity_is_refused(tmp_path):
    cfg = os.path.join(GOLD, "in80.txt")
    a = str(tmp_path / "a.work")
    solver([cfg, "--max-steps", "3", "--save-work", a] + COMMON)
    from kangaroo_b200.ingest import DPTable
    t = DPTable(threads=1)
    t.load_work_ex(a)
    n = len(t)
    t.close()
    rc, out = solver(["--resume", a, "--grid", "8,32", "--seed", "2", "--max-steps", "5", "--dp-table", "device",
                      "--dp-table-capacity", str(n - 1)])
    assert rc != 0 and "holds more than the table's capacity of %d entries" % (n - 1) in out, out[-2000:]
    assert "imported and verified" not in out and "MJump/s" not in out


@needs_ingest
def test_a_full_table_stops_the_run_with_a_resumable_cut(tmp_path):
    """capacity for about 4 launches' DPs: the run stops with a message and writes the table of the launches it holds, with
    their count and no kangaroos; the host table resumes it"""
    cfg = os.path.join(GOLD, "in80.txt")
    a = str(tmp_path / "full.work")
    per_launch = 8 * 32 * 128 * 64 // 256                          # DPs of one launch at dp 8, on average
    rc, out = solver([cfg, "--dp", "8", "--grid", "8,32", "--seed", "5", "--save-work", a, "--dp-table", "device",
                      "--dp-table-capacity", str(4 * per_launch)])
    assert rc == 1 and "DP table full, run stopped" in out and "resume it with --dp-table host" in out, out[-2000:]
    from kangaroo_b200.ingest import DPTable
    t = DPTable(threads=1)
    w = t.load_work_ex(a)
    launches = w.total_count // (8 * 32 * 128 * 64)
    assert w.total_count % (8 * 32 * 128 * 64) == 0 and 2 <= launches <= 5 and w.nb_walk == 0
    assert 0 < len(t) <= 4 * per_launch
    t.close()
    t = DPTable(threads=1)
    t.load_work_ex(a)
    rc, out = solver(["--resume", a, "--grid", "8,32", "--seed", "2", "--max-steps", "3"])
    assert ("Resume %s: %d DPs" % (a, len(t))) in out and "0 kangaroos in the file" in out, out[-2000:]


@needs_ingest
def test_steps_behind_a_save_wait_in_host_ram_and_give_the_same_files(tmp_path):
    """--save-interval on every step keeps the ingest thread busy with saves, so steps queue behind them: those wait in host
    RAM, not on the GPU, and come back to the GPU to be inserted.  A mid-run save equals the end-of-run save of a straight run
    with the host table stopped at that file's count, byte for byte past the header's time."""
    from kangaroo_b200 import ecmath as ec
    from kangaroo_b200 import solver as S
    start, end, pubs = ec.parse_config(os.path.join(GOLD, "in80.txt"))
    path = str(tmp_path / "m.work")
    copies = []

    class Keep(S.Solver):
        def _on_saved(self, p, mb, seconds, err):
            assert err is None
            copies.append(open(p, "rb").read())

    s = Keep(start, end, pubs[0], 8, (8, 32), seed=9, save_work=path, save_interval=1e-6, save_kangaroos=True, dp_table="device",
             dp_table_capacity=1 << 22)
    s.run(12, verbose=False)
    parked = s.parked
    s.close()
    assert len(copies) >= 3 and s.same_herd == 0 and not s.table_stopped
    assert parked > 0
    mid = copies[len(copies) // 2]
    cm = int.from_bytes(mid[140:148], "little")
    straight = str(tmp_path / "s.work")
    rc, out = solver([os.path.join(GOLD, "in80.txt"), "--max-steps", str(cm // (8 * 32 * 128 * 64) - 1), "--save-work", straight,
                      "--dp", "8", "--grid", "8,32", "--seed", "9", "--save-kangaroos"])
    assert " 0 dead kangaroos re-created" in out, out[-2000:]
    raw = open(straight, "rb").read()
    assert raw[:148] == mid[:148] and raw[156:] == mid[156:]


@needs_ingest
def test_a_failing_insert_stops_the_run(tmp_path):
    """an insert that raises (a CUDA error, say) stops the run with a message instead of leaving the main loop waiting"""
    from kangaroo_b200 import ecmath as ec
    from kangaroo_b200 import solver as S
    start, end, pubs = ec.parse_config(os.path.join(GOLD, "in80.txt"))
    s = S.Solver(start, end, pubs[0], 8, (8, 32), seed=9, dp_table="device", dp_table_capacity=1 << 22)
    add, calls = s.dps.add, []

    def failing(*args):
        calls.append(1)
        if len(calls) == 3:
            raise RuntimeError("kgx_dptable_add: injected")
        return add(*args)

    s.dps.add = failing
    assert s.run(50, verbose=False) is None
    assert s.table_stopped and s.table_kind == "error" and "injected" in s.table_msg
    assert s.steps < 10
    s.close()
