"""-m gpu: the device DP table (kgx_dptable_*), its bucket sort and the work-file merge (kgx_work_merge) at the keys random
records never produce -- shared x.hi or x.lo, one x in several buckets, one tag and home slot, probe chains that wrap, one home
slot over hundreds of buckets, copies of earlier records -- against tests/dptable_model.py's model of the reference's
HashTable: its events in arrival order, its count and its saved bytes.  Where build/libkgx_ingest.so is built the reference's
own HashTable (the host table) is fed the same records and checked too."""
import ctypes
import os

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200 import worktool as wt
from tests import dptable_model as dm
from tests.worktool_util import NB, ROOT, Work, merge_model

pytestmark = pytest.mark.gpu
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
CAP = 4096                           # the capacity the index classes are searched for: nslots = 6208


def events_of(evs, n):
    """the first n kgx_dp_event of a ctypes Event array as (kind, rank, kidx, h, d_old, d_new) tuples"""
    raw = ctypes.string_at(ctypes.addressof(evs), 48 * n)
    w32, w64 = np.frombuffer(raw, np.uint32).reshape(n, 12).tolist(), np.frombuffer(raw, np.uint64).reshape(n, 6).tolist()
    return [(a[0], a[1], a[2], a[3], (b[2], b[3]), (b[4], b[5])) for a, b in zip(w32, w64)]


def upload(segments, stride):
    """the segments as one gather buffer on the GPU: rank r's records at r * stride"""
    import torch
    flat = np.zeros((max(1, len(segments) * stride), 5), np.uint64)
    for r, seg in enumerate(segments):
        flat[r * stride:r * stride + len(seg)] = seg
    return torch.from_numpy(flat.view(np.uint8).reshape(-1)).cuda()


class Checked:
    """a device table and the model (and the host table where it is built) fed the same calls"""

    def __init__(self, capacity=CAP, max_events=1 << 14):
        from kangaroo_b200.ingest import DPTable, DeviceDPTable
        self.dev = DeviceDPTable(capacity, max_events=max_events)
        self.model = dm.HashTableModel()
        self.host = DPTable(threads=8, max_events=1 << 16) if os.path.exists(INGEST) else None
        self.cap = max_events

    def add(self, segments, stride=None):
        """one call: the device's events are the model's, element for element; the counts agree"""
        want, skipped = self.model.add(segments)
        stride = stride or max(len(s) for s in segments) + 3
        buf = upload(segments, stride)
        rc, n, evs = self.dev.add_raw(buf.data_ptr(), [len(s) for s in segments], stride)
        assert n == len(want) <= self.cap
        assert rc == (-1 if skipped else 0)
        assert events_of(evs, n) == want
        assert len(self.dev) == len(self.model)
        if self.host is not None:
            got, bad = dm.host_add(self.host, segments)
            assert sorted(got) == sorted(want) and bad == (skipped > 0) and len(self.host) == len(self.model)
        return want

    def check_save(self, tmp_path):
        path = str(tmp_path / "dev.work")
        self.dev.save_work(path, **dm.save_args())
        raw = open(path, "rb").read()
        assert raw == self.model.to_work().to_bytes()
        if self.host is not None:
            self.host.save_work(str(tmp_path / "host.work"), **dm.save_args())
            assert open(str(tmp_path / "host.work"), "rb").read() == raw
        return raw

    def close(self):
        self.dev.close()
        if self.host is not None:
            self.host.close()


# ---- 1: every class in calls of its own, then all of them in one table -----------------------------------------------------
def test_each_class_alone_then_all_together(tmp_path):
    adv = dm.Adversary(31)
    classes = adv.classes()
    kinds = set()
    for name, recs in classes:
        t = Checked()
        for segs in adv.calls(recs):
            kinds |= {e[0] for e in t.add(segs)}
            t.check_save(tmp_path)
        t.close()
    assert kinds == {dm.EV_RESET, dm.EV_COLLISION}
    t = Checked()
    everything = np.concatenate([r for _, r in classes])
    everything = everything[adv.rng.permutation(len(everything))]
    for segs in adv.calls(everything, ncalls=4, nsegs=6):
        t.add(segs)
        t.check_save(tmp_path)
    # every class again as copies of the full table's records, in one call
    t.add([adv.copies(r) for _, r in classes])
    t.check_save(tmp_path)
    t.close()


# ---- 2: rank segments --------------------------------------------------------------------------------------------------------
def test_256_rank_segments_then_257_refused(tmp_path):
    """256 segments: the first and last empty, runs of empty ones between, one of exactly the stride; records of every class and
    their copies spread over them.  The events name each record's rank, in arrival order."""
    adv = dm.Adversary(41)
    stride = 24
    counts = adv.rng.integers(1, 16, size=256)
    counts[[0, 255]] = 0
    counts[10:20] = 0
    counts[100:140] = 0
    counts[254] = 0
    counts[200] = stride
    base = np.concatenate([adv.shared_hi(), adv.shared_lo(), adv.one_x(), adv.same_home(), adv.wrapping(), adv.contention(200)])
    recs = np.concatenate([base, adv.copies(base, 500)])
    total = int(counts.sum())
    if total > len(recs):
        recs = np.concatenate([recs, adv.random(total - len(recs))])
    recs = recs[adv.rng.permutation(len(recs))][:total]
    segments = np.split(recs, np.cumsum(counts)[:-1])
    t = Checked()
    ev = t.add(segments, stride=stride)
    ranks = {e[1] for e in ev}
    assert len(ev) > 100 and 200 in ranks and min(ranks) > 0 and max(ranks) < 254
    before = t.check_save(tmp_path)
    import torch
    buf = torch.zeros(257 * 40, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="257 ranks"):
        t.dev.add_raw(buf.data_ptr(), [1] * 257, 1)
    assert len(t.dev) == len(t.model)
    assert t.check_save(tmp_path) == before
    t.close()


# ---- 3: a load in chunks, at exactly the capacity ----------------------------------------------------------------------------
def test_load_in_chunks_at_exact_capacity(tmp_path):
    """A table a little over three save chunks (2^21 entries), saved to A, loads into a table of exactly A's entry count: four
    flushes, buckets across their boundaries.  It saves A again; any further record is refused and changes nothing.  Loaded
    with room for one more call, every entry of A added again is a duplicate."""
    from kangaroo_b200.ingest import DeviceDPTable, TableFull
    adv = dm.Adversary(53)
    C = dm.SAVE_CHUNK
    t = DeviceDPTable(3 * C + (1 << 16), max_events=1 << 12)
    host = None
    if os.path.exists(INGEST):
        from kangaroo_b200.ingest import DPTable
        host = DPTable(threads=8, max_events=1 << 16)
    crafted = np.concatenate([adv.shared_hi(8), adv.shared_lo(8)])
    batches = [adv.random(1 << 20) for _ in range(6)] + [adv.random(30000)]
    batches[1] = np.concatenate([batches[1], crafted[:len(crafted) // 2], adv.copies(crafted[:len(crafted) // 2])])
    batches[4] = np.concatenate([batches[4], crafted[len(crafted) // 2:], adv.copies(crafted), adv.copies(batches[0], 5000)])
    for b in batches:
        b = b[adv.rng.permutation(len(b))]
        buf = upload([b], len(b))
        rc, n, _ = t.add_raw(buf.data_ptr(), [len(b)], len(b))
        assert rc == 0
        if host is not None:
            ev, _ = dm.host_add(host, [b])
            assert len(ev) == n and len(host) == len(t)
    count = len(t)
    assert 3 * C < count <= t.capacity
    a = str(tmp_path / "a.work")
    t.save_work(a, **dm.save_args())
    t.close()
    raw = open(a, "rb").read()
    if host is not None:
        host.save_work(str(tmp_path / "h.work"), **dm.save_args())
        assert open(str(tmp_path / "h.work"), "rb").read() == raw
        host.close()
    nb, _, _ = dm.bucket_heads(raw)
    assert int(nb.sum()) == count and int(nb.max()) >= 30
    end = np.cumsum(nb)
    straddle = [k for k in range(1, count // C + 1) if np.any((end - nb < k * C) & (end > k * C))]
    assert straddle, "no bucket crosses a flush boundary"

    exact = DeviceDPTable(count, max_events=1 << 12)
    exact.load_work_ex(a)
    assert len(exact) == count
    b = str(tmp_path / "b.work")
    exact.save_work(b, **dm.save_args())
    assert open(b, "rb").read() == raw
    buf = upload([adv.random(1)], 1)
    with pytest.raises(TableFull, match="full"):
        exact.add_raw(buf.data_ptr(), [1], 1)
    assert len(exact) == count
    exact.save_work(b, **dm.save_args())
    assert open(b, "rb").read() == raw
    exact.close()

    recs = dm.file_records(raw)
    step = 1 << 21
    room = DeviceDPTable(count + step, max_events=1 << 12)
    room.load_work_ex(a)
    for i in range(0, len(recs), step):
        part = recs[i:i + step]
        buf = upload([part], len(part))
        rc, n, evs = room.add_raw(buf.data_ptr(), [len(part)], len(part))
        assert rc == 0 and n == len(part), "records of A not found after the load: %d of %d" % (len(part) - n, len(part))
        assert all(e[0] == dm.EV_RESET and e[4] == (0, 0) for e in events_of(evs, min(n, 1 << 12)))
        assert len(room) == count
    room.close()


# ---- 4: the merge -------------------------------------------------------------------------------------------------------------
def blocks(sums, C):
    """kgx_work_merge's blocks of whole buckets for a block of C entries: [(last bucket, entries)]"""
    out, fill, last = [], 0, None
    for h in np.nonzero(sums)[0].tolist():
        if fill + sums[h] > C:
            out.append((last, fill))
            fill = 0
        fill += sums[h]
        last = h
    return out + [(last, fill)]


def test_merge_at_adversarial_buckets(tmp_path):
    """four inputs holding classes (a), (b) and (c), with runs of equal x over three or four inputs whose d are equal or not;
    blocks of the default size, of exactly the largest bucket and of a size an adversarial bucket ends exactly"""
    from tests.golden import make_work_golden as g
    works = dm.Adversary(61).merge_inputs(4, g.START, g.START + (1 << g.RANGE_BITS) - 1, ec.mul(g.PRIV))
    paths = [w.write(str(tmp_path / ("in%d.work" % i))) for i, w in enumerate(works)]
    want, dup, coll = merge_model(works)
    runs = {}
    for i, w in enumerate(works):
        for h in range(NB):
            for x, d in w.table[h]:
                runs.setdefault((h, x), []).append(d)
    long = [ds for ds in runs.values() if len(ds) >= 3]
    assert sum(1 for ds in long if len(set(ds)) < len(ds) and len(set(ds)) > 1) >= 10
    assert dup > 20 and len(coll) > 40
    sums = np.array([sum(len(w.table[h]) for w in works) for h in range(NB)])
    big = int(sums.max())
    adversarial = set(np.nonzero(sums >= 30)[0].tolist())
    small = next(C for C in range(big + 1, 4 * big) if any(h in adversarial and f == C for h, f in blocks(sums, C)[:-1]))
    assert any(f == big for _, f in blocks(sums, big))
    for block in (0, big, small):
        dest = str(tmp_path / ("m%d.work" % block))
        r = wt.merge_files(paths, dest, block_entries=block)
        assert open(dest, "rb").read() == want.to_bytes(), block
        assert (r.entries, r.duplicates, r.collisions) == (want.entries(), dup, len(coll))
        assert [(h, d1[0] | d1[1] << 64, d2[0] | d2[1] << 64) for h, d1, d2 in r.collision_list] == coll
        if block:
            assert r.blocks == len(blocks(sums, block))


# ---- 5: the bucket sort on x.lo alone ------------------------------------------------------------------------------------------
def test_one_bucket_ordered_by_x_lo_alone(tmp_path):
    """12000 entries of one bucket share x.hi (2^63: its sign bit set), so the save orders them by x.lo alone"""
    adv = dm.Adversary(71, capacity=16384)
    n = 12000
    recs = adv.recs(4321, adv._words(n), np.full(n, 1 << 63, np.uint64))
    t = Checked(capacity=16384)
    t.add([recs[:5000], recs[5000:7000]])
    t.add([recs[7000:], adv.copies(recs, 3000)])
    raw = t.check_save(tmp_path)
    assert len(t.dev) == n and Work.read(str(tmp_path / "dev.work")).maxitem[4321] > n
    t.close()
    assert len(raw) == 156 + 8 * NB + 32 * n + 8
