"""A plain model of the reference's HashTable (HashTable::Add record by record, the events kgx_ingest.cpp's add_one maps its
results to, SaveTable's bytes), a mirror of the device table's index hash (kgx_dptable.cuh: slot_tag, slot_home, slots_for),
and a seeded generator of DP records at the keys random records never produce: shared x.hi, shared x.lo, one x in several
buckets, one tag and home slot, probe chains that wrap past the last slot, one home slot over hundreds of buckets, and
copies of earlier records."""
import ctypes
import struct

import numpy as np

from tests.worktool_util import NB, Work

M64 = (1 << 64) - 1
TYPE = 1 << 62                       # b126 of the tagged distance (its high word's bit 62): the herd
EV_RESET, EV_COLLISION = 1, 2
SAVE_CHUNK = 1 << 21                 # kgx_dptable.cuh: entries per host<->device chunk of a save or a load
HOME_MUL_X1 = 0x9E3779B97F4A7C15     # slot_home's multipliers
HOME_MUL = 0xD6E8FEB86659FD93
HDR = dict(dp=9, start=0x1234 << 70, end=(0x1234 << 70) + (1 << 60), key=(0xABCDEF << 100, 0x777 << 50), count=123456789, time=42.5)


# ---- the device table's index hash ------------------------------------------------------------------------------------
def slots_for(capacity):
    return capacity + capacity // 2 + 64


def slot_tag(h, x1):
    return (h + 1) | ((x1 >> 51) << 19)


def slot_home(h, x0, x1, nslots):
    k = ((x0 ^ ((x1 * HOME_MUL_X1) & M64) ^ (h << 40)) * HOME_MUL) & M64
    k ^= k >> 32
    return (k * nslots) >> 64


def slot_homes(h, x0, x1, nslots):
    """slot_home over uint64 arrays (numpy multiplies mod 2^64; the high word of k * nslots from 32-bit halves, nslots < 2^32)"""
    assert nslots < 1 << 32
    with np.errstate(over="ignore"):
        k = (x0 ^ (x1 * np.uint64(HOME_MUL_X1)) ^ (h << np.uint64(40))) * np.uint64(HOME_MUL)
    k ^= k >> np.uint64(32)
    n = np.uint64(nslots)
    return ((k >> np.uint64(32)) * n + (((k & np.uint64(0xFFFFFFFF)) * n) >> np.uint64(32))) >> np.uint64(32)


# ---- HashTable ----------------------------------------------------------------------------------------------------------
class HashTableModel:
    """HashTable::Add (HashTable.cpp:262-307) per record in arrival order: maxItem 16 on a bucket's first Add, +4 on every later
    Add that finds nbItem >= maxItem - 1, stored or not; an x already in the bucket is a duplicate (equal d: RESET, d_old 0),
    a same-herd collision (RESET, d_old = the stored d) or a collision between herds (COLLISION)."""

    def __init__(self):
        self.ent = {}                # h -> {x: d}, x and d 128-bit ints (low word first in a record)
        self.mx = {}

    def __len__(self):
        return sum(len(b) for b in self.ent.values())

    def add(self, segments):
        """segments: one (n, 5) uint64 record array per rank -> (events in arrival order, records skipped for h >= 2^18).
        An event is (kind, rank, kidx, h, (d_old lo, hi), (d_new lo, hi))."""
        events, skipped = [], 0
        for r, seg in enumerate(segments):
            for w0, x0, x1, d0, d1 in np.asarray(seg, dtype=np.uint64).reshape(-1, 5).tolist():
                h = w0 >> 32
                if h >= NB:
                    skipped += 1
                    continue
                b = self.ent.setdefault(h, {})
                mx = self.mx.get(h, 0) or 16
                if b and len(b) >= mx - 1:
                    mx += 4
                self.mx[h] = mx
                x, d = x0 | x1 << 64, d0 | d1 << 64
                old = b.get(x)
                if old is None:
                    b[x] = d
                    continue
                if old == d:
                    kind, old = EV_RESET, 0
                else:
                    kind = EV_COLLISION if (old ^ d) & (TYPE << 64) else EV_RESET
                events.append((kind, r, w0 & 0xFFFFFFFF, h, (old & M64, old >> 64), (d0, d1)))
        return events, skipped

    def to_work(self, **hdr):
        """the table as HashTable::SaveTable writes it: buckets in order, entries by unsigned 128-bit x"""
        a = dict(HDR, **hdr)
        w = Work(a["dp"], a["start"], a["end"], a["key"], a["count"], a["time"])
        for h, b in self.ent.items():
            w.table[h] = sorted(b.items())
            w.maxitem[h] = self.mx[h]
        return w


def save_args(**hdr):
    """the keyword arguments of DPTable.save_work / DeviceDPTable.save_work that write HashTableModel.to_work(**hdr)'s header"""
    a = dict(HDR, **hdr)
    return dict(dp_bits=a["dp"], range_start=a["start"], range_end=a["end"], pubkey=a["key"], total_count=a["count"],
                total_time=a["time"], total_walk=0)


def host_add(table, segments):
    """segments into a DPTable (the reference's HashTable through kgi_add), one call per rank -> (events, any record skipped).
    The host table returns each call's events in worker-shard order."""
    out, bad = [], False
    for r, seg in enumerate(segments):
        if len(seg) == 0:
            continue
        a = np.ascontiguousarray(seg, dtype=np.uint64)
        ne = ctypes.c_uint32(0)
        rc = table._lib.kgi_add(table._h, a.ctypes.data_as(ctypes.c_void_p), len(a), r, table._ev, table._cap, ctypes.byref(ne))
        assert ne.value <= table._cap
        bad |= rc != 0
        out += [(int(e.kind), int(e.rank), int(e.kidx), int(e.h), (int(e.d_old[0]), int(e.d_old[1])), (int(e.d_new[0]), int(e.d_new[1])))
                for e in table._ev[:ne.value]]
    return out, bad


def bucket_heads(raw):
    """(nbItem, maxItem) of every bucket of a HEADW file's bytes, and the offset of each bucket's first entry"""
    nb, mx, off = np.zeros(NB, np.int64), np.zeros(NB, np.int64), np.zeros(NB, np.int64)
    o = 156
    for h in range(NB):
        nb[h], mx[h] = struct.unpack_from("<II", raw, o)
        off[h] = o + 8
        o += 8 + 32 * int(nb[h])
    return nb, mx, off


def file_records(raw):
    """every entry of a HEADW file's table as a record (kIdx = its position in the file)"""
    nb, _, off = bucket_heads(raw)
    full = np.nonzero(nb)[0]
    ent = np.concatenate([np.frombuffer(raw, np.uint64, count=4 * int(nb[h]), offset=int(off[h])) for h in full]).reshape(-1, 4)
    h = np.repeat(full.astype(np.uint64), nb[full])
    rec = np.empty((len(ent), 5), np.uint64)
    rec[:, 0] = (h << np.uint64(32)) | np.arange(len(ent), dtype=np.uint64)
    rec[:, 1:] = ent
    return rec


# ---- records at the edges ------------------------------------------------------------------------------------------------
SPECIAL = [0, 1, (1 << 63) - 1, 1 << 63, M64]


class Adversary:
    """Seeded 40-byte DP records ((n, 5) uint64: {u32 kIdx, u32 h}, x lo, x hi, d lo, d hi).  Every record gets a new kIdx, so
    each event names its record.  capacity: the device table the index classes (d), (e), (f) are built for."""

    def __init__(self, seed, capacity=4096):
        self.rng = np.random.default_rng(seed)
        self.capacity = capacity
        self.nslots = slots_for(capacity)
        self.kidx = 0

    def u64(self, n):
        return self.rng.integers(0, 1 << 63, size=n, dtype=np.uint64) * np.uint64(2) + self.rng.integers(0, 2, size=n, dtype=np.uint64)

    def recs(self, h, x0, x1, d0=None, d1=None):
        n = len(x0)
        out = np.empty((n, 5), np.uint64)
        out[:, 0] = (np.broadcast_to(np.asarray(h, np.uint64), (n,)) << np.uint64(32)) | np.arange(self.kidx, self.kidx + n, dtype=np.uint64)
        self.kidx += n
        out[:, 1], out[:, 2] = x0, x1
        out[:, 3] = self.u64(n) if d0 is None else d0
        out[:, 4] = self.u64(n) if d1 is None else d1
        return out

    def random(self, n, buckets=None):
        h = self.rng.integers(0, NB, size=n, dtype=np.uint64) if buckets is None else self.rng.choice(np.asarray(buckets, np.uint64), size=n)
        return self.recs(h, self.u64(n), self.u64(n))

    def buckets(self, n):
        return [int(h) for h in self.rng.choice(NB, size=n, replace=False)]

    def _words(self, n):
        """n distinct 64-bit words: SPECIAL, pairs one bit apart, the rest random"""
        v = list(SPECIAL)
        for b in self.rng.choice(64, size=4, replace=False):
            w = int(self.u64(1)[0])
            v += [w, w ^ (1 << int(b))]
        v = list(dict.fromkeys(v))
        while len(v) < n:
            v = list(dict.fromkeys(v + [int(w) for w in self.u64(n - len(v))]))
        v = np.array(v[:n], np.uint64)
        self.rng.shuffle(v)
        return v

    def shared_hi(self, nbuckets=3):
        """(a) buckets of 30 to 60 entries that share x.hi and differ in x.lo only"""
        out = []
        for i, h in enumerate(self.buckets(nbuckets)):
            n = int(self.rng.integers(30, 61))
            hi = [0, M64, 1 << 63][i] if i < 3 else int(self.u64(1)[0])
            out.append(self.recs(h, self._words(n), np.full(n, hi, np.uint64)))
        return np.concatenate(out)

    def shared_lo(self, nbuckets=3):
        """(b) buckets of 30 to 60 entries that share x.lo and differ in x.hi only"""
        out = []
        for i, h in enumerate(self.buckets(nbuckets)):
            n = int(self.rng.integers(30, 61))
            lo = [M64, 0, 1 << 63][i] if i < 3 else int(self.u64(1)[0])
            out.append(self.recs(h, np.full(n, lo, np.uint64), self._words(n)))
        return np.concatenate(out)

    def one_x(self, nx=6, per=5):
        """(c) one 128-bit x under several buckets (the first two x: (0, 0) and (2^64-1, 2^64-1)); the same d in some of them"""
        out = []
        for i in range(nx):
            x0, x1 = (0, 0) if i == 0 else (M64, M64) if i == 1 else (int(self.u64(1)[0]), int(self.u64(1)[0]))
            d0, d1 = self.u64(per), self.u64(per)
            d0[1::2], d1[1::2] = d0[0], d1[0]
            out.append(self.recs(np.array(self.buckets(per), np.uint64), np.full(per, x0, np.uint64), np.full(per, x1, np.uint64), d0, d1))
        return np.concatenate(out)

    def _search(self, want, h, x0=None, x1=None, top=None, unique_h=False):
        """records of bucket(s) h whose home slot is in `want` (a set of slots): x0 / x1 fixed where given, else random; top
        fixes x1 >> 51.  h may be None (random buckets)."""
        found, hs = [], set()
        while len(found) < want["n"]:
            m = 1 << 20
            H = self.rng.integers(0, NB, size=m, dtype=np.uint64) if h is None else np.full(m, h, np.uint64)
            X0 = self.u64(m) if x0 is None else np.full(m, x0, np.uint64)
            X1 = self.u64(m) if x1 is None else np.full(m, x1, np.uint64)
            if top is not None:
                X1 = (X1 & np.uint64((1 << 51) - 1)) | np.uint64(top << 51)
            home = slot_homes(H, X0, X1, self.nslots)
            for i in np.nonzero((home >= np.uint64(want["lo"])) & (home < np.uint64(want["hi"])))[0]:
                if unique_h and int(H[i]) in hs:
                    continue
                hs.add(int(H[i]))
                found.append((int(H[i]), int(X0[i]), int(X1[i])))
                if len(found) == want["n"]:
                    break
        a = np.array(found, np.uint64).reshape(-1, 3)
        return self.recs(a[:, 0], a[:, 1], a[:, 2])

    def same_home(self, n=8):
        """(d) one bucket, one x1 >> 51 (the 13 bits of x.hi in the tag) and one home slot, different x: n sharing x.hi that
        differ in x.lo, and n sharing x.lo that differ in the low 51 bits of x.hi"""
        h = self.buckets(1)[0]
        home = int(self.rng.integers(0, self.nslots - 256))
        top = int(self.rng.integers(0, 1 << 13))
        x1 = (top << 51) | int(self.u64(1)[0] >> np.uint64(13))
        slot = dict(n=n, lo=home, hi=home + 1)
        return np.concatenate([self._search(slot, h, x1=x1), self._search(slot, h, x0=int(self.u64(1)[0]), top=top)])

    def wrapping(self, window=4, n=10):
        """(e) n records whose home is one of the last `window` slots: more records than slots, so chains wrap to slot 0.  Half
        of them in one bucket."""
        slot = dict(n=n // 2, lo=self.nslots - window, hi=self.nslots)
        return np.concatenate([self._search(slot, self.buckets(1)[0]), self._search(slot, None)])

    def contention(self, n=300):
        """(f) one record in each of n distinct buckets, all with one home slot"""
        home = int(self.rng.integers(self.nslots // 4, self.nslots // 2))
        return self._search(dict(n=n, lo=home, hi=home + 1), None, unique_h=True)

    def copies(self, recs, n=None):
        """(g) copies of records: a third exact (new kIdx, same x and d), a third with another d of the same herd, a third with
        a d of the other herd"""
        recs = np.asarray(recs, np.uint64)
        pick = recs[self.rng.choice(len(recs), size=min(n or len(recs), len(recs)), replace=False)]
        out = self.recs(pick[:, 0] >> np.uint64(32), pick[:, 1], pick[:, 2], pick[:, 3], pick[:, 4])
        k = len(out) // 3
        t = np.uint64(TYPE)
        out[k:, 3] = self.u64(len(out) - k)
        out[k:, 4] = (self.u64(len(out) - k) & ~t) | (pick[k:, 4] & t)
        out[2 * k:, 4] ^= t
        return out[self.rng.permutation(len(out))]

    def classes(self):
        """[(name, records)] of classes (a) to (f), each shuffled"""
        out = [("shared_hi", self.shared_hi()), ("shared_lo", self.shared_lo()), ("one_x", self.one_x()),
               ("same_home", self.same_home()), ("wrapping", self.wrapping()), ("contention", self.contention())]
        return [(name, r[self.rng.permutation(len(r))]) for name, r in out]

    def merge_inputs(self, n_inputs, start, end, key):
        """n_inputs Work files holding classes (a), (b) and (c): a third of the entries in one input, the others in two to
        n_inputs of them with the first input's d, another d of its herd or of the other herd (the same variant again in some),
        and random entries so that no two inputs hold as many entries (the reference's -wmdir orders its inputs by size)"""
        works = [Work(16 + i % 3, start, end, key, 1000 * (i + 1), 0.5 * (i + 1)) for i in range(n_inputs)]
        pool = np.concatenate([self.shared_hi(), self.shared_lo(), self.one_x()])
        for w0, x0, x1, d0, d1 in pool.tolist():
            h, x, d = w0 >> 32, x0 | x1 << 64, d0 | d1 << 64
            k = 1 if self.rng.random() < 1 / 3 else int(self.rng.integers(2, n_inputs + 1))
            ds = [d]
            for _ in range(k - 1):
                c = int(self.rng.integers(0, 4))
                v = int(self.u64(1)[0]) | (int(self.u64(1)[0]) & ~(3 << 62)) << 64
                ds.append(d if c == 0 else (v | (d & (TYPE << 64))) if c == 1 else (v | (~d & (TYPE << 64))) if c == 2 else ds[-1])
            for i, dd in zip(sorted(self.rng.choice(n_inputs, size=k, replace=False).tolist()), ds):
                works[i].add(x, dd, h)
        while len({w.entries() for w in works}) < n_inputs:
            w = works[int(self.rng.integers(0, n_inputs))]
            w.add(int(self.u64(1)[0]) | int(self.u64(1)[0]) << 64, int(self.u64(1)[0]), int(self.rng.integers(0, NB)))
        return works

    def calls(self, recs, ncalls=3, nsegs=3):
        """recs over ncalls calls of nsegs rank segments (one of them empty), with copies (g) of records of the same call and
        of earlier calls mixed in -> [[segment, ...], ...]"""
        parts = np.array_split(recs, ncalls)
        out, seen = [], np.zeros((0, 5), np.uint64)
        for p in parts:
            seen = np.concatenate([seen, p])
            c = np.concatenate([p, self.copies(p, max(1, len(p) // 3)), self.copies(seen, max(1, len(seen) // 4))])
            c = c[self.rng.permutation(len(c))]
            cut = sorted(self.rng.choice(np.arange(1, len(c)), size=nsegs - 2, replace=False).tolist()) if len(c) > nsegs else []
            segs = np.split(c, cut)
            segs.insert(int(self.rng.integers(0, len(segs) + 1)), np.zeros((0, 5), np.uint64))
            out.append(segs)
        return out
