"""Shared helpers of the work-file tool tests: a HEADW reader / writer in Python and a model of the N-way merge."""
import gzip
import math
import os
import shutil
import struct

from kangaroo_b200 import ecmath as ec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
REFBIN = os.path.join(ROOT, "oracle", "_ref", "kangaroo_ref_cpu")
NB = 1 << 18
TYPE_BIT = 1 << 126


def golden(name, tmp_path, dest=None):
    path = str(tmp_path / (dest or name[:-3]))
    with gzip.open(os.path.join(GOLD, name), "rb") as src, open(path, "wb") as dst:
        shutil.copyfileobj(src, dst)
    return path


class Work:
    """A HEADW file: header fields, 2^18 buckets of (x, d) int pairs (x: the stored 128 bits, d: the tagged distance), maxItem
    per bucket, and the kangaroo block (None when the file ends after its table)."""

    def __init__(self, dp, start, end, key, count=0, time=0.0, version=0):
        self.dp, self.start, self.end, self.key, self.count, self.time, self.version = dp, start, end, key, count, time, version
        self.table = [[] for _ in range(NB)]
        self.maxitem = [0] * NB
        self.walks = b""

    @classmethod
    def read(cls, path):
        raw = open(path, "rb").read()
        assert struct.unpack_from("<I", raw)[0] == 0xFA6A8001
        val = lambda o: int.from_bytes(raw[o:o + 32], "little")
        w = cls(struct.unpack_from("<I", raw, 8)[0], val(12), val(44), (val(76), val(108)), struct.unpack_from("<Q", raw, 140)[0],
                struct.unpack_from("<d", raw, 148)[0], struct.unpack_from("<I", raw, 4)[0])
        off = 156
        for h in range(NB):
            nb, mx = struct.unpack_from("<II", raw, off)
            off += 8
            w.maxitem[h] = mx
            for i in range(nb):
                w.table[h].append((int.from_bytes(raw[off:off + 16], "little"), int.from_bytes(raw[off + 16:off + 32], "little")))
                off += 32
        w.walks = raw[off:] if off < len(raw) else None
        return w

    def entries(self):
        return sum(len(b) for b in self.table)

    def header_bytes(self):
        l4 = lambda v: int(v).to_bytes(32, "little")
        return (struct.pack("<III", 0xFA6A8001, self.version, self.dp) + l4(self.start) + l4(self.end) + l4(self.key[0]) +
                l4(self.key[1]) + struct.pack("<Qd", self.count, self.time))

    def to_bytes(self, walk_count=True):
        out = [self.header_bytes()]
        for h in range(NB):
            b = self.table[h]
            out.append(struct.pack("<II", len(b), self.maxitem[h]))
            out.extend(x.to_bytes(16, "little") + d.to_bytes(16, "little") for x, d in b)
        if walk_count:
            out.append(self.walks if self.walks else struct.pack("<Q", 0))
        return b"".join(out)

    def write(self, path, walk_count=True):
        open(path, "wb").write(self.to_bytes(walk_count))
        return path

    def add(self, x, d, h=None):
        """an entry of bucket h (default: the one x's bits 128..145 name -- pass the full 256-bit x), kept sorted"""
        if h is None:
            h = (x >> 128) & 0x3FFFF
        b = self.table[h]
        b.append((x & ((1 << 128) - 1), d))
        b.sort(key=lambda e: e[0])
        self.maxitem[h] = max(self.maxitem[h], (len(b) + 3) // 4 * 4)


def tagged(dist, wild, neg=False):
    return dist | (TYPE_BIT if wild else 0) | ((1 << 127) if neg else 0)


def search_key(w):
    return ec.add(w.key, ec.neg(ec.mul(w.start))) if w.start else w.key


def merge_model(works):
    """The N-way merge of `works` in order -> (Work, duplicates, collisions [(h, d_first, d_other)]): at equal x the earlier
    input's entry is kept, a later one with an equal tagged d is a duplicate, any other a collision (as the reference's pairwise
    MergeH calls give), listed by bucket then x.  maxItem = nbItem rounded up to 4."""
    w0 = works[0]
    out = Work(min(w.dp for w in works), w0.start, w0.end, w0.key, sum(w.count for w in works), 0.0)
    out.time = 0.0
    for w in works:
        out.time += w.time
    dup, coll = 0, []
    for h in range(NB):
        first = {}
        for w in works:
            for x, d in w.table[h]:
                if x not in first:
                    first[x] = d
                elif first[x] == d:
                    dup += 1
                else:
                    coll.append((h, x, first[x], d))
        b = sorted(first.items(), key=lambda e: e[0])
        out.table[h] = b
        out.maxitem[h] = (len(b) + 3) // 4 * 4
    out.walks = None
    coll.sort(key=lambda c: (c[0], c[1]))                  # bucket, then x (stable: input order at one x)
    return out, dup, [(h, a, b) for h, _, a, b in coll]


def log2_count(n):
    return "%.2f" % math.log2(n)


def crafted_pair(tmp_path, priv=None):
    """Two small files on ref_work48's key and range whose merge finds the key: a tame DP at d_t*G in one file and a wild DP
    at the same x (d_w = d_t - k, K + d_w*G = d_t*G with k = priv - start) in the other, among a few ordinary tame DPs."""
    from tests.golden import make_work_golden as g
    priv = g.PRIV if priv is None else priv
    pub = ec.mul(priv)
    end = g.START + (1 << g.RANGE_BITS) - 1
    k = priv - g.START
    a, b = Work(g.DP_BITS, g.START, end, pub, 1000, 1.5), Work(g.DP_BITS + 2, g.START, end, pub, 2000, 2.5)
    d_t = k + 0x1234567
    a.add(ec.mul(d_t)[0], tagged(d_t, False))
    b.add(ec.mul(d_t)[0], tagged(d_t - k, True))
    for i in range(1, 6):
        a.add(ec.mul(977 * i)[0], tagged(977 * i, False))
        b.add(ec.mul(1543 * i)[0], tagged(1543 * i, False))
    return a.write(str(tmp_path / "pair_a.work")), b.write(str(tmp_path / "pair_b.work"))
