"""Work-file tools on the GPU: check and merge HEADW work files (the reference's -wcheck and -wm / -wmdir).

    python -m kangaroo_b200.worktool check FILE [--device N]
    python -m kangaroo_b200.worktool merge FILE1 FILE2 [FILE ...] -o DEST [--device N]
    python -m kangaroo_b200.worktool merge --dir DIR -o DEST [--device N]

`check` recomputes every stored DP (d*G, or key - start*G + d*G for a wild one) and every kangaroo on the GPU
(libkgx.so, kgx_work_check) and exits 1 when anything is wrong.  It also takes the solver's batch work files (--batch-keys
--batch-save): every kangaroo is checked against its own target key, every wild DP against all keys of the file.  `merge` combines files of the same key and range in the order
given (the entry of the earlier file wins at equal x) with kgx_work_merge, resolves every tame/wild collision on the device
with the solver's resolver (kgx_work_resolve: the reference's CheckKey result), and either prints the key and writes nothing, or writes
DEST through DEST.tmp, fsync and rename.  The merged file ends with a kangaroo count of 0, so the solver's --resume and the
reference's -i take it; they start fresh herds.  Batch work files (the same keys in the same order and the same range) are
merged with kgx_work_merge_batch, which resolves every tame/wild collision against all keys on the device; DEST is always
written, with a batch block that records every key solved in an input or by the merge, so that --batch-resume continues from
it.  There is no CPU path: without a device both commands fail.

The batch block of a batch work file (its layout: kgx_workfile.h) is written and read here, through libkgx.so's
kgx_batch_block / kgx_batch_read, which the device check uses too; neither needs a device."""
import argparse
import ctypes
import math
import os
import struct
import sys

import numpy as np

from . import ecmath as ec
from ._lib import load_library
from .ingest import _limbs4, read_work_header

HEADW = 0xFA6A8001
_u64p = ctypes.POINTER(ctypes.c_uint64)
TYPE_BIT = 1 << 126                    # b126 of a tagged distance: the herd (HashTable::CalcDistAndType)


class CheckInfo(ctypes.Structure):
    """kgx_work_check_info"""
    _fields_ = [("dp_bits", ctypes.c_uint32), ("has_walk_count", ctypes.c_uint32), ("entries", ctypes.c_uint64),
                ("wrong_entries", ctypes.c_uint64), ("walks", ctypes.c_uint64), ("walks_tame", ctypes.c_uint64),
                ("walks_wild", ctypes.c_uint64), ("wrong_walks", ctypes.c_uint64), ("n_wrong_entries_listed", ctypes.c_uint32),
                ("n_wrong_walks_listed", ctypes.c_uint32), ("n_keys", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class MergeInfo(ctypes.Structure):
    """kgx_work_merge_info"""
    _fields_ = [("dp_bits", ctypes.c_uint32), ("blocks", ctypes.c_uint32), ("entries", ctypes.c_uint64),
                ("duplicates", ctypes.c_uint64), ("collisions", ctypes.c_uint64), ("total_count", ctypes.c_uint64),
                ("total_time", ctypes.c_double), ("n_listed", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class BatchMergeInfo(ctypes.Structure):
    """kgx_batch_merge_info"""
    _fields_ = [("n_keys", ctypes.c_uint32), ("solved_in_inputs", ctypes.c_uint32), ("solved_by_merge", ctypes.c_uint32),
                ("left", ctypes.c_uint32), ("same_herd", ctypes.c_uint64), ("no_key", ctypes.c_uint64),
                ("already_solved", ctypes.c_uint64), ("solving", ctypes.c_uint64)]


class BatchKeyResult(ctypes.Structure):
    """kgx_batch_key_result"""
    _fields_ = [("status", ctypes.c_uint32), ("h", ctypes.c_uint32), ("priv", ctypes.c_uint64 * 4), ("d_first", ctypes.c_uint64 * 2),
                ("d_other", ctypes.c_uint64 * 2)]


class Collision(ctypes.Structure):
    """kgx_work_collision"""
    _fields_ = [("h", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("d_first", ctypes.c_uint64 * 2),
                ("d_other", ctypes.c_uint64 * 2)]


def _err(lib):
    return lib.kgx_work_last_error().decode()


def is_work_file(path):
    """a regular file that starts with the HEADW magic (Kangaroo::ReadHeader)"""
    if not os.path.isfile(path):
        return False
    with open(path, "rb") as f:
        raw = f.read(4)
    return len(raw) == 4 and struct.unpack("<I", raw)[0] == HEADW


class BatchBlock:
    """The batch block of a batch work file: pubs [(x, y)] in input order, solved (bool per key), privs (int, or None when
    unsolved), targets (uint16 per kangaroo, file order), offset (byte where the block starts = where the records end)."""

    def __init__(self, pubs, solved, privs, targets, offset=0):
        self.pubs, self.solved, self.privs, self.offset = list(pubs), [bool(v) for v in solved], list(privs), int(offset)
        self.targets = np.ascontiguousarray(targets, dtype=np.uint16)

    @property
    def n_keys(self):
        return len(self.pubs)

    @property
    def nb_walk(self):
        return int(self.targets.size)


def _limbs(vals, n):
    return np.array([[(int(v) >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(n)] for v in vals], dtype=np.uint64).reshape(len(vals), n)


def _val(row):
    return sum(int(v) << (64 * k) for k, v in enumerate(row))


def batch_block(block, offset):
    """kgx_batch_block: the bytes that follow the kangaroo records of a batch work file whose records end at byte `offset`"""
    lib = load_library()
    n = block.n_keys
    keys = np.ascontiguousarray(np.hstack([_limbs([p[0] for p in block.pubs], 4), _limbs([p[1] for p in block.pubs], 4)]))
    privs = np.ascontiguousarray(_limbs([(p or 0) if s else 0 for p, s in zip(block.privs, block.solved)], 4))
    solved = np.ascontiguousarray(block.solved, dtype=np.uint8)
    out = np.empty(int(lib.kgx_batch_block_bytes(n, block.nb_walk)), dtype=np.uint8)
    rc = lib.kgx_batch_block(keys.ctypes.data_as(_u64p), solved.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), privs.ctypes.data_as(_u64p), n,
                             block.targets.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)), block.nb_walk, int(offset),
                             out.ctypes.data_as(ctypes.c_void_p))
    if rc != 0:
        raise ValueError(_err(lib))
    return out


def read_batch(path):
    """kgx_batch_read -> BatchBlock, or None for a plain HEADW file.  Not a HEADW file, or a batch block cut short or damaged:
    ValueError; a file that cannot be opened: OSError."""
    lib = load_library()
    nk, nw, off = ctypes.c_uint32(0), ctypes.c_uint64(0), ctypes.c_uint64(0)
    rc = lib.kgx_batch_read(os.fsencode(path), ctypes.byref(nk), ctypes.byref(nw), ctypes.byref(off), None, None, None, None)
    if rc == 0:
        return None
    if rc == 1:
        n = nk.value
        keys, privs = np.zeros((n, 8), dtype=np.uint64), np.zeros((n, 4), dtype=np.uint64)
        solved, targets = np.zeros(n, dtype=np.uint8), np.zeros(nw.value, dtype=np.uint16)
        rc = lib.kgx_batch_read(os.fsencode(path), ctypes.byref(nk), ctypes.byref(nw), ctypes.byref(off), keys.ctypes.data_as(_u64p),
                                solved.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), privs.ctypes.data_as(_u64p),
                                targets.ctypes.data_as(ctypes.POINTER(ctypes.c_uint16)))
        if rc == 1:
            return BatchBlock([(_val(k[:4]), _val(k[4:])) for k in keys], solved, [_val(p) if s else None for p, s in zip(privs, solved)],
                              targets, off.value)
    if rc == -1:
        raise ValueError(_err(lib))
    raise OSError(-rc, "%s: %s" % (path, os.strerror(-rc)))


class CheckResult:
    def __init__(self, info, wrong_entries, wrong_walks):
        for name, _ in CheckInfo._fields_:
            setattr(self, name, getattr(info, name))
        self.wrong_entry_positions = wrong_entries      # [(bucket, index in bucket)], file order
        self.wrong_walk_indices = wrong_walks

    @property
    def ok(self):
        return self.wrong_entries == 0 and self.wrong_walks == 0


def check(path, device=0, chunk=0, cap=16):
    """kgx_work_check on one file -> CheckResult.  A directory or a file that is not HEADW raises ValueError."""
    if os.path.isdir(path):
        raise ValueError("%s is a directory: partitioned work files are not supported" % path)
    lib = load_library()
    info = CheckInfo()
    we = (ctypes.c_uint32 * (2 * cap))()
    ww = (ctypes.c_uint64 * cap)()
    rc = lib.kgx_work_check(int(device), os.fsencode(path), int(chunk), ctypes.byref(info), we, ww, cap)
    if rc == -1:
        raise ValueError(_err(lib))
    if rc != 0:
        raise RuntimeError("kgx_work_check: " + _err(lib))
    return CheckResult(info, [(we[2 * i], we[2 * i + 1]) for i in range(info.n_wrong_entries_listed)],
                       [ww[i] for i in range(info.n_wrong_walks_listed)])


def check_records(kind, recs, hs, key, range_start, device=0):
    """kgx_work_check_records: kind 0 = (n, 4) uint64 table entries with their buckets hs, kind 1 = (n, 12) uint64 kangaroo
    records -> per-record uint8 results (entries: 1 = wrong; kangaroos: 0 wrong, 1 tame, 2 wild)"""
    recs = np.ascontiguousarray(recs, dtype=np.uint64)
    n = recs.shape[0]
    out = np.zeros(n, dtype=np.uint8)
    hs = np.ascontiguousarray(hs if hs is not None else np.zeros(n), dtype=np.uint32)
    lib = load_library()
    rc = lib.kgx_work_check_records(int(device), int(kind), recs.ctypes.data_as(ctypes.c_void_p), hs.ctypes.data_as(ctypes.c_void_p), n,
                                    _limbs4(key[0]), _limbs4(key[1]), _limbs4(range_start), out.ctypes.data_as(ctypes.c_void_p))
    if rc != 0:
        raise (ValueError if rc == -1 else RuntimeError)("kgx_work_check_records: " + _err(lib))
    return out


def comb_table(device=0):
    """the check's fixed-base table: {(w, j): (x, y)} = j * 2^(4w) * G"""
    lib = load_library()
    out = (ctypes.c_uint64 * (480 * 8))()
    if lib.kgx_work_comb(int(device), out) != 0:
        raise RuntimeError("kgx_work_comb: " + _err(lib))
    val = lambda o: sum(int(out[o + k]) << (64 * k) for k in range(4))
    return {(w, j): (val(8 * (w * 15 + j - 1)), val(8 * (w * 15 + j - 1) + 4)) for w in range(32) for j in range(1, 16)}


class MergeResult:
    def __init__(self, info, collisions):
        for name, _ in MergeInfo._fields_:
            setattr(self, name, getattr(info, name))
        self.collision_list = collisions                # [(h, d_first (2 limbs), d_other (2 limbs))], bucket then x order


def merge_files(paths, tmp_path, device=0, block_entries=0, cap=1 << 20):
    """kgx_work_merge: paths merged in order into tmp_path -> MergeResult.  Refusals (bad inputs, a bucket larger than a
    block) raise ValueError and leave no tmp_path."""
    lib = load_library()
    arr = (ctypes.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])
    info = MergeInfo()
    coll = (Collision * cap)()
    rc = lib.kgx_work_merge(int(device), arr, len(paths), os.fsencode(tmp_path), int(block_entries), ctypes.byref(info), coll, cap)
    if rc == -1:
        raise ValueError(_err(lib))
    if rc != 0:
        raise RuntimeError("kgx_work_merge: " + _err(lib))
    return MergeResult(info, [(c.h, (c.d_first[0], c.d_first[1]), (c.d_other[0], c.d_other[1])) for c in coll[:info.n_listed]])


class BatchMergeResult(MergeResult):
    """MergeResult of kgx_work_merge_batch (collision_list is empty) with the counts of kgx_batch_merge_info and, per key,
    status (0 unsolved, 1 solved in an input, 2 solved by the merge), priv (int or None) and, for status 2, the collision
    (h, d_first, d_other) that solved it"""

    def __init__(self, info, binfo, keys):
        super().__init__(info, [])
        for name, _ in BatchMergeInfo._fields_:
            setattr(self, name, getattr(binfo, name))
        self.status = [k.status for k in keys]
        self.privs = [_val(k.priv) if k.status else None for k in keys]
        self.solved_by = [(k.h, _val(k.d_first), _val(k.d_other)) if k.status == 2 else None for k in keys]


def merge_batch_files(paths, tmp_path, device=0, block_entries=0):
    """kgx_work_merge_batch: batch work files merged in order into tmp_path -> BatchMergeResult.  Refusals raise ValueError
    and leave no tmp_path."""
    lib = load_library()
    first = read_batch(paths[0])
    if first is None:
        raise ValueError("MergeWork: %s is a plain HEADW work file: batch work files merge only with batch work files" % paths[0])
    arr = (ctypes.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])
    info, binfo = MergeInfo(), BatchMergeInfo()
    keys = (BatchKeyResult * first.n_keys)()
    rc = lib.kgx_work_merge_batch(int(device), arr, len(paths), os.fsencode(tmp_path), int(block_entries), ctypes.byref(info),
                                  ctypes.byref(binfo), keys, first.n_keys)
    if rc == -1:
        raise ValueError(_err(lib))
    if rc != 0:
        raise RuntimeError("kgx_work_merge_batch: " + _err(lib))
    return BatchMergeResult(info, binfo, keys[:binfo.n_keys])


def resolve(d_first, d_other, keys, range_start, device=0):
    """kgx_work_resolve: collisions (two lists of tagged distances) against keys K = key - start*G (a list of (x, y), None for
    the point at infinity) -> [(key index, private key) or None], as kgi_resolve_multi gives them"""
    lib = load_library()
    n = len(d_first)
    kt = np.ascontiguousarray(np.hstack([_limbs([0 if k is None else k[0] for k in keys], 4),
                                         _limbs([0 if k is None else k[1] for k in keys], 4)]))
    a, b = np.ascontiguousarray(_limbs(d_first, 2)), np.ascontiguousarray(_limbs(d_other, 2))
    idx, priv = np.zeros(n, dtype=np.uint32), np.zeros((n, 4), dtype=np.uint64)
    rc = lib.kgx_work_resolve(int(device), a.ctypes.data_as(_u64p), b.ctypes.data_as(_u64p), n, kt.ctypes.data_as(_u64p), len(keys),
                              _limbs4(range_start), idx.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), priv.ctypes.data_as(_u64p))
    if rc != 0:
        raise (ValueError if rc == -1 else RuntimeError)("kgx_work_resolve: " + _err(lib))
    return [None if i == 0xFFFFFFFF else (int(i), _val(p)) for i, p in zip(idx.tolist(), priv)]


def dir_inputs(dirname):
    """Kangaroo::MergeDir's inputs (Merge.cpp:255-315): every regular HEADW file of the directory, largest first (equal sizes
    by name, so that the order does not depend on the directory's listing)"""
    files = [os.path.join(dirname, f) for f in os.listdir(dirname)]
    files = [f for f in files if not os.path.islink(f) and is_work_file(f)]
    return sorted(files, key=lambda f: (-os.path.getsize(f), os.path.basename(f)))


def _same_version_and_range(paths, p, h, first):
    """MergeWork's refusals of input p (header h) against paths[0] (header first): another version or range -> ValueError"""
    if h.version != first.version:
        raise ValueError("MergeWork: cannot merge workfile of different version (%s)" % p)
    if (h.range_start, h.range_end) != (first.range_start, first.range_end):
        raise ValueError("MergeWork: File range differs (%s, %s)" % (paths[0], p))


def validate(paths):
    """MergeWork's refusals (Merge.cpp:56-143), before the device is touched: fewer than two inputs, a directory, a file that
    is not HEADW, another version, a key off the curve, another range or another key -> ValueError"""
    if len(paths) < 2:
        raise ValueError("MergeWork: at least two work files are needed, %d given" % len(paths))
    first = None
    for p in paths:
        if os.path.isdir(p):
            raise ValueError("%s is a directory: partitioned work files are not supported" % p)
        if not is_work_file(p):
            raise ValueError("MergeWork: %s is not a HEADW work file" % p)
        h = read_work_header(p)
        x, y = h.key
        if not (x < ec.P and y < ec.P and (y * y - x * x * x - 7) % ec.P == 0):
            raise ValueError("MergeWork: key of %s does not lie on elliptic curve" % p)
        first = first or h
        _same_version_and_range(paths, p, h, first)
        if h.key != first.key:
            raise ValueError("MergeWork: key differs, multiple keys not yet supported (%s, %s)" % (paths[0], p))


def validate_batch(paths, blocks):
    """kgx_work_merge_batch's refusals that need no device (blocks: read_batch of every path): a plain file among batch
    files, another range or version, another key count or order, two inputs with different private keys for one key ->
    ValueError"""
    for p, b in zip(paths, blocks):
        if b is None:
            raise ValueError("MergeWork: %s is a plain HEADW work file: batch work files merge only with batch work files" % p)
    h0, b0 = read_work_header(paths[0]), blocks[0]
    for p, b in zip(paths[1:], blocks[1:]):
        _same_version_and_range(paths, p, read_work_header(p), h0)
        if b.n_keys != b0.n_keys:
            raise ValueError("MergeWork: %s holds %d keys, %s %d: the key lists differ" % (p, b.n_keys, paths[0], b0.n_keys))
        for k, (q, q0) in enumerate(zip(b.pubs, b0.pubs)):
            if q != q0:
                raise ValueError("MergeWork: key #%d of %s differs from key #%d of %s: the key lists differ" % (k, p, k, paths[0]))
    for k in range(b0.n_keys):
        recorded = {b.privs[k] for b in blocks if b.solved[k]}
        if len(recorded) > 1:
            raise ValueError("MergeWork: two inputs record different private keys for key #%d" % k)


def merge_batch(paths, blocks, dest, device=0, block_entries=0, out=print):
    """Merge batch work files into dest (always written, through DEST.tmp, fsync and rename) -> (0, {key index: private key}
    of the keys the merge solved)"""
    validate_batch(paths, blocks)
    tmp = dest + ".tmp"
    res = merge_batch_files(paths, tmp, device=device, block_entries=block_entries)
    with open(tmp, "rb+") as f:
        os.fsync(f.fileno())
    os.replace(tmp, dest)
    for p in paths:
        out("File %s: [DP%d]" % (p, read_work_header(p).dp_bits))
    found = {}
    for i, (st, priv) in enumerate(zip(res.status, res.privs)):
        if st == 2:
            found[i] = priv
            out("Key#%2d Pub:  0x%064X\n       Priv: 0x%X" % (i, blocks[0].pubs[i][0], priv))
    out("Keys: %d, %d solved in the inputs, %d solved by the merge, %d left" %
        (res.n_keys, res.solved_in_inputs, res.solved_by_merge, res.left))
    out("Collisions: %d (%d solved a key, %d on a key already solved, %d on no key, %d same-herd)" %
        (res.collisions, res.solving, res.already_solved, res.no_key, res.same_herd))
    out("Dead kangaroo: %d" % (res.duplicates + res.same_herd))
    out("Total f1+f2: DP count 2^%.2f" % (math.log2(res.entries) if res.entries else float("-inf")))
    out("Merged %d batch files into %s: %d entries, %d duplicates" % (len(paths), dest, res.entries, res.duplicates))
    return 0, found


def merge(paths, dest, device=0, block_entries=0, out=print):
    """Merge `paths` (in order) into dest -> (exit code, private key or None).  A solved key removes DEST.tmp and writes no
    file (Merge.cpp:218-229); otherwise DEST.tmp is synced and renamed over dest.  Batch work files go to merge_batch, which
    returns the keys it solved instead of a private key."""
    if len(paths) >= 2 and all(is_work_file(p) for p in paths):
        blocks = [read_batch(p) for p in paths]
        if any(b is not None for b in blocks):
            return merge_batch(paths, blocks, dest, device=device, block_entries=block_entries, out=out)
    validate(paths)
    tmp = dest + ".tmp"
    res = merge_files(paths, tmp, device=device, block_entries=block_entries)
    for p in paths:
        out("File %s: [DP%d]" % (p, read_work_header(p).dp_bits))
    h = read_work_header(tmp)
    start, pub = h.range_start, h.key
    key = ec.add(pub, ec.neg(ec.mul(start))) if start else pub          # Kangaroo::InitSearchKey
    unresolved, priv = 0, None
    cross = [c for c in res.collision_list if (c[1][1] ^ c[2][1]) & (TYPE_BIT >> 64)]
    same_herd = len(res.collision_list) - len(cross)
    if cross:                                                             # Merge.cpp's CheckKey on each, in order, on the device
        found = resolve([_val(d1) for _, d1, _ in cross], [_val(d2) for _, _, d2 in cross], [key], start, device=device)
        first = next((i for i, m in enumerate(found) if m is not None), len(found))
        unresolved, priv = first, (found[first][1] if first < len(found) else None)
    if res.n_listed < res.collisions:
        out("Warning: %d collisions, only the first %d examined" % (res.collisions, res.n_listed))
    if priv is not None and ec.mul(priv) == pub:
        os.remove(tmp)
        out("Key# 0 Pub:  0x%064X\n       Priv: 0x%X" % (pub[0], priv))
        return 0, priv
    with open(tmp, "rb+") as f:
        os.fsync(f.fileno())
    os.replace(tmp, dest)
    out("Dead kangaroo: %d" % (res.duplicates + same_herd))
    out("Total f1+f2: DP count 2^%.2f" % (math.log2(res.entries) if res.entries else float("-inf")))
    if unresolved:
        out("Unresolved tame/wild collisions: %d" % unresolved)
    out("Merged %d files into %s: %d entries, %d duplicates, %d same-herd collisions" %
        (len(paths), dest, res.entries, res.duplicates, same_herd))
    return 0, None


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m kangaroo_b200.worktool", description=__doc__.split("\n\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    c = sub.add_parser("check", help="recompute every DP and kangaroo of a work file on the GPU (-wcheck)")
    c.add_argument("file")
    c.add_argument("--device", type=int, default=0)
    m = sub.add_parser("merge", help="merge work files of the same key and range on the GPU (-wm / -wmdir)")
    m.add_argument("files", nargs="*")
    m.add_argument("--dir", default=None, help="merge every HEADW file of DIR, largest first (-wmdir); batch work files too")
    m.add_argument("-o", "--output", required=True, metavar="DEST")
    m.add_argument("--device", type=int, default=0)
    m.add_argument("--block-entries", type=int, default=0, help="entries per device block, summed over the inputs (0 = 2^22)")
    a = ap.parse_args(argv)
    try:
        if a.cmd == "check":
            r = check(a.file, device=a.device)
            pct = 100.0 * (1.0 - r.wrong_entries / r.entries) if r.entries else 100.0
            print("[%.3f%% OK]" % pct)
            if r.n_keys:
                print("Batch work file: %d keys (every kangaroo checked against its own target key)" % r.n_keys)
            print("DP: %d" % r.entries)
            print("DP Wrong: %d" % r.wrong_entries)
            for h, i in r.wrong_entry_positions:
                print("  wrong DP at bucket %06X [%d]" % (h, i))
            if r.has_walk_count:
                print("Kangaroos: %d (tame OK %d, wild OK %d, wrong %d)" % (r.walks, r.walks_tame, r.walks_wild, r.wrong_walks))
                for i in r.wrong_walk_indices:
                    print("  wrong kangaroo #%d" % i)
            else:
                print("Kangaroos: none (the file ends after its table)")
            return 0 if r.ok else 1
        if a.dir is not None:
            if a.files:
                ap.error("merge: give files or --dir, not both")
            files = dir_inputs(a.dir)
            if len(files) < 2:
                raise ValueError("MergeDir: less than 2 work files in the directory")
        else:
            files = a.files
        rc, _ = merge(files, a.output, device=a.device, block_entries=a.block_entries)
        return rc
    except ValueError as e:
        print(str(e), file=sys.stderr)
        return 2


if __name__ == "__main__":
    sys.exit(main())
