"""ctypes binding of build/libkgx_ingest.so (C ABI: include/kgx_ingest.h): the rank-0 distinguished-point table.

The table is the reference's own `class HashTable` (HashTable.{h,cpp}, compiled unmodified from the reference sources by
kangaroo_b200/csrc/build_ingest.sh); the library adds the batched, bucket-sharded multi-threaded insert that replaces the
single-mutex loop of Kangaroo::SolveKeyGPU (Kangaroo.cpp:594-612) when the DP records of all GPUs arrive on rank 0.
No Python-side fallback: without the library DPTable() raises.  KGX_INGEST_LIB in the environment names another copy of the
library (or a path that does not exist, to run as a checkout built without the reference sources).

DeviceDPTable and DeviceResolver are libkgx.so's: the device table and the collision resolver on the GPU, which need no
reference sources; nothing here loads libkgx_ingest.so for them."""
import collections
import ctypes
import os
import struct

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KGX_INGEST_LIB") or os.path.join(HERE, "..", "build", "libkgx_ingest.so")
NO_KEY = 0xFFFFFFFF

EV_RESET, EV_COLLISION = 1, 2
DP40_BYTES, ITEM_BYTES = 40, 56
_M64 = 0xFFFFFFFFFFFFFFFF


class Event(ctypes.Structure):
    """kgi_event"""
    _fields_ = [("kind", ctypes.c_uint32), ("rank", ctypes.c_uint32), ("kidx", ctypes.c_uint32), ("h", ctypes.c_uint32),
                ("d_old", ctypes.c_uint64 * 2), ("d_new", ctypes.c_uint64 * 2)]


class EventKey(ctypes.Structure):
    """kgx_dp_event_key: an event of kgx_dptable_add_resolve, with its collision's key index (NO_KEY: none) and private key"""
    _fields_ = [("ev", Event), ("key", ctypes.c_uint32), ("reserved", ctypes.c_uint32), ("priv", ctypes.c_uint64 * 4)]


_u64p = ctypes.POINTER(ctypes.c_uint64)
_SIGS = {
    "kgi_create": (ctypes.c_void_p, [ctypes.c_int]),
    "kgi_destroy": (None, [ctypes.c_void_p]),
    "kgi_reset": (None, [ctypes.c_void_p]),
    "kgi_count": (ctypes.c_uint64, [ctypes.c_void_p]),
    "kgi_threads": (ctypes.c_int, [ctypes.c_void_p]),
    "kgi_add": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(Event), ctypes.c_uint32,
                               ctypes.POINTER(ctypes.c_uint32)]),
    "kgi_add_items": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, _u64p, ctypes.POINTER(Event),
                                     ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32)]),
    "kgi_resolve": (ctypes.c_int, [ctypes.c_void_p, _u64p, _u64p, _u64p, _u64p, _u64p, _u64p]),
    "kgi_resolve_multi": (ctypes.c_int, [ctypes.c_void_p, _u64p, _u64p, _u64p, ctypes.c_uint32, _u64p, ctypes.POINTER(ctypes.c_uint32),
                                         _u64p]),
    "kgi_save_work": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32, _u64p, _u64p, _u64p, _u64p, ctypes.c_uint64,
                                     ctypes.c_double]),
    "kgi_load_work": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint32), _u64p,
                                     ctypes.POINTER(ctypes.c_double)]),
    "kgi_save_work_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32, _u64p, _u64p, _u64p, _u64p, ctypes.c_uint64,
                                        ctypes.c_double, ctypes.c_uint64]),
    "kgi_load_work_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint32), _u64p, _u64p, _u64p, _u64p,
                                        _u64p, ctypes.POINTER(ctypes.c_double), _u64p, _u64p]),
}
WALK_BYTES = 96          # one kangaroo of a work file: x[4], y[4], d[4] (Backup.cpp:536-539)
EXPORTED_SYMBOLS = sorted(_SIGS)
_lib = None


def load_library():
    global _lib
    if _lib is not None:
        return _lib
    path = os.path.abspath(LIB_PATH)
    why = "is missing" if not os.path.exists(path) else None
    if why is None:
        try:
            lib = ctypes.CDLL(path)
        except OSError as e:
            why = "cannot be loaded (%s)" % e
    if why is not None:
        raise RuntimeError("kangaroo_b200: %s %s: the host DP table (--dp-table host) is the reference's HashTable, which "
                           "kangaroo_b200/csrc/build_ingest.sh builds against the reference sources; --dp-table device and "
                           "--dp-table sharded keep the table and resolve collisions on the GPU without it" % (path, why))
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    _lib = lib
    return lib


def _limbs4(v):
    return (ctypes.c_uint64 * 4)(*[(int(v) >> (64 * k)) & _M64 for k in range(4)])


def _save_args(dp_bits, range_start, range_end, pubkey, total_count, total_time, total_walk):
    """the header arguments of kgi_save_work_ex / kgx_dptable_save_work"""
    return (int(dp_bits), _limbs4(range_start), _limbs4(range_end), _limbs4(pubkey[0]), _limbs4(pubkey[1]), int(total_count),
            float(total_time), int(total_walk))


def _load_work_ex(fn, handle, path, *extra):
    """kgi_load_work_ex / kgx_dptable_load_work (extra: their trailing arguments) -> (return code, WorkInfo)"""
    dp, cnt, tm = ctypes.c_uint32(0), ctypes.c_uint64(0), ctypes.c_double(0)
    rs, re_, kx, ky = (ctypes.c_uint64 * 4)(), (ctypes.c_uint64 * 4)(), (ctypes.c_uint64 * 4)(), (ctypes.c_uint64 * 4)()
    walk, off = ctypes.c_uint64(0), ctypes.c_uint64(0)
    rc = fn(handle, os.fsencode(path), ctypes.byref(dp), rs, re_, kx, ky, ctypes.byref(cnt), ctypes.byref(tm), ctypes.byref(walk),
            ctypes.byref(off), *extra)
    val = lambda a: sum(int(a[k]) << (64 * k) for k in range(4))
    return rc, WorkInfo(path, dp.value, val(rs), val(re_), (val(kx), val(ky)), cnt.value, tm.value, walk.value, off.value)


class DPTable:
    """Rank-0 DP table: reference HashTable + sharded batched insert (Kangaroo::AddToTable semantics per record)."""

    def __init__(self, threads=0, max_events=4096):
        self._lib = load_library()
        self._h = ctypes.c_void_p(self._lib.kgi_create(int(threads)))
        if not self._h:
            raise RuntimeError("kgi_create failed")
        self._ev = (Event * max_events)()
        self._cap = max_events
        self.threads = self._lib.kgi_threads(self._h)

    def close(self):
        if self._h:
            self._lib.kgi_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return int(self._lib.kgi_count(self._h))

    def reset(self):
        self._lib.kgi_reset(self._h)

    def _events(self, n):
        out = []
        for i in range(min(n, self._cap)):
            e = self._ev[i]
            out.append((int(e.kind), int(e.rank), int(e.kidx), (int(e.d_old[0]), int(e.d_old[1])), (int(e.d_new[0]), int(e.d_new[1]))))
        return out

    @staticmethod
    def _buf(buf, rec):
        a = np.ascontiguousarray(np.frombuffer(buf, dtype=np.uint8) if not isinstance(buf, np.ndarray) else buf.view(np.uint8).reshape(-1))
        assert a.size % rec == 0
        return a, a.size // rec

    def add_dp40(self, buf, rank=0):
        """buf: n x 40-byte DP records (bytes / uint8 ndarray) -> list of (kind, rank, kidx, d_old, d_new) events."""
        a, n = self._buf(buf, DP40_BYTES)
        ne = ctypes.c_uint32(0)
        rc = self._lib.kgi_add(self._h, a.ctypes.data_as(ctypes.c_void_p), n, int(rank), self._ev, self._cap, ctypes.byref(ne))
        if rc != 0:
            raise RuntimeError("kgi_add: malformed DP record (h >= 2^18)")
        return self._events(ne.value)

    def add_items(self, buf, wild_offset, rank=0):
        """buf: n x 56-byte engine ITEMs (biased distances) -> events; HashTable::Convert applied on the host."""
        a, n = self._buf(buf, ITEM_BYTES)
        wo = (ctypes.c_uint64 * 2)(int(wild_offset) & _M64, (int(wild_offset) >> 64) & _M64)
        ne = ctypes.c_uint32(0)
        rc = self._lib.kgi_add_items(self._h, a.ctypes.data_as(ctypes.c_void_p), n, int(rank), wo, self._ev, self._cap, ctypes.byref(ne))
        if rc != 0:
            raise RuntimeError("kgi_add_items failed")
        return self._events(ne.value)

    def resolve(self, d_old, d_new, key, range_start):
        """Kangaroo::CollisionCheck/CheckKey with the reference's Secp256K1 -> private key (int) or None."""
        a = (ctypes.c_uint64 * 2)(*d_old); b = (ctypes.c_uint64 * 2)(*d_new)
        out = (ctypes.c_uint64 * 4)()
        rc = self._lib.kgi_resolve(self._h, a, b, _limbs4(key[0]), _limbs4(key[1]), _limbs4(range_start), out)
        return sum(int(out[k]) << (64 * k) for k in range(4)) if rc == 1 else None

    @staticmethod
    def key_table(keys):
        """keys (list of (x, y); None = the point at infinity, stored as (0, 0)) -> the (K, 8) uint64 table resolve_multi takes"""
        out = np.zeros((len(keys), 8), dtype=np.uint64)
        for i, k in enumerate(keys):
            if k is not None:
                out[i] = [(int(k[c]) >> (64 * w)) & _M64 for c in (0, 1) for w in range(4)]
        return out

    def resolve_multi(self, d_old, d_new, keys, range_start):
        """resolve() against a key table (key_table(), or a list of points) -> (key index, private key) of the first key
        matched, or None"""
        kt = keys if isinstance(keys, np.ndarray) else self.key_table(keys)
        kt = np.ascontiguousarray(kt, dtype=np.uint64)
        a = (ctypes.c_uint64 * 2)(*d_old); b = (ctypes.c_uint64 * 2)(*d_new)
        idx, out = ctypes.c_uint32(0), (ctypes.c_uint64 * 4)()
        rc = self._lib.kgi_resolve_multi(self._h, a, b, kt.ctypes.data_as(_u64p), kt.shape[0], _limbs4(range_start), ctypes.byref(idx), out)
        return (int(idx.value), sum(int(out[k]) << (64 * k) for k in range(4))) if rc == 1 else None

    def save_work(self, path, dp_bits, range_start, range_end, pubkey, total_count=0, total_time=0.0, total_walk=0):
        """Header + table (+ the kangaroo count: the caller appends total_walk x 96-byte records right after)."""
        rc = self._lib.kgi_save_work_ex(self._h, os.fsencode(path),
                                        *_save_args(dp_bits, range_start, range_end, pubkey, total_count, total_time, total_walk))
        if rc != 0:
            raise RuntimeError("kgi_save_work: cannot write %s: %s" % (path, os.strerror(-rc)))

    def load_work(self, path):
        dp, cnt, tm = ctypes.c_uint32(0), ctypes.c_uint64(0), ctypes.c_double(0)
        rc = self._lib.kgi_load_work(self._h, os.fsencode(path), ctypes.byref(dp), ctypes.byref(cnt), ctypes.byref(tm))
        if rc != 0:
            raise RuntimeError("kgi_load_work: %s is not a HEADW work file" % path)
        return dp.value, cnt.value, tm.value

    def load_work_ex(self, path):
        """Kangaroo::LoadWork (Backup.cpp:149-207): the table into this DPTable -> WorkInfo (header, nbLoadedWalk and the
        offset of the kangaroo block)."""
        rc, info = _load_work_ex(self._lib.kgi_load_work_ex, self._h, path)
        if rc != 0:
            raise RuntimeError("kgi_load_work: %s is not a complete HEADW work file" % path)
        return info


class TableFull(RuntimeError):
    """An add that would take a DeviceDPTable past its capacity: nothing of it was inserted."""


def _limbs_u64(vals, k):
    """ints -> (n, k) uint64 little-endian limbs"""
    return np.array([[(int(v) >> (64 * w)) & _M64 for w in range(k)] for v in vals], dtype=np.uint64).reshape(-1, k)


class DeviceResolver:
    """kgx_resolver_*: tame/wild collisions resolved on one GPU against a key table -- kgi_resolve_multi's result (the first
    key in input order that +-Td +-Wd * G hits, and its private key) without the host.  keys: K = key - start*G per key, as
    DPTable.key_table gives them (or a list of points, None for the point at infinity); range_start below n.  The comb and
    the key index are built once here; run_raw is one stream-ordered kernel, and DeviceDPTable.add(resolver=) runs it inside
    the table's add.  A resolver of one key also checks received DP records (verify / verify_raw, kgx_resolver_verify), and
    groups the good ones by the shard of a sharded table that owns them in the same call (verify_partition /
    verify_partition_raw, kgx_resolver_verify_partition)."""

    def __init__(self, keys, range_start, device=0):
        from ._lib import load_library as load_engine
        self._lib = load_engine()
        kt = keys if isinstance(keys, np.ndarray) else DPTable.key_table(keys)
        kt = np.ascontiguousarray(kt, dtype=np.uint64)
        self.device, self.n_keys = int(device), int(kt.shape[0])
        self._h = ctypes.c_void_p(self._lib.kgx_resolver_create(self.device, kt.ctypes.data_as(_u64p), self.n_keys, _limbs4(range_start)))
        if not self._h:
            raise RuntimeError(self._lib.kgx_resolver_last_error(None).decode())

    def close(self):
        if self._h:
            self._lib.kgx_resolver_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def run_raw(self, pairs, n, key_out, priv_out, stream=0):
        """n collisions at device address pairs (n x 4 limbs {d_first, d_other}) -> key_out (n uint32) and priv_out (n x 4 limbs),
        device addresses, queued on `stream`"""
        rc = self._lib.kgx_resolver_run(self._h, ctypes.c_void_p(int(pairs)), int(n), ctypes.c_void_p(int(key_out)),
                                        ctypes.c_void_p(int(priv_out)), ctypes.c_void_p(int(stream)))
        if rc != 0:
            raise RuntimeError(self._lib.kgx_resolver_last_error(self._h).decode())

    def verify_scratch_bytes(self, n):
        """device scratch bytes verify_raw needs for n records"""
        return int(self._lib.kgx_resolver_verify_scratch_bytes(int(n)))

    def verify_raw(self, recs, n, good, counts, bad_idx, cap, scratch, scratch_bytes, stream=0):
        """kgx_resolver_verify: n 40-byte DP records at device address recs (8-byte aligned) checked against the one key ->
        good (device, the good records in input order), counts (device, 2 uint32: good, bad), bad_idx (device, the indices of
        the first cap bad records); queued on `stream`, not waited for"""
        rc = self._lib.kgx_resolver_verify(self._h, ctypes.c_void_p(int(recs)), int(n), ctypes.c_void_p(int(good)),
                                           ctypes.c_void_p(int(counts)), ctypes.c_void_p(int(bad_idx)), int(cap),
                                           ctypes.c_void_p(int(scratch)), int(scratch_bytes), ctypes.c_void_p(int(stream)))
        if rc != 0:
            raise RuntimeError(self._lib.kgx_resolver_last_error(self._h).decode())

    def verify(self, recs, cap=None, stream=None):
        """recs: a CUDA uint8 tensor of n x 40-byte records -> (good records as a CUDA uint8 tensor, number of bad records, the
        first cap (default: all) bad indices as a list); on `stream` or torch's current one, waited for"""
        import torch
        assert recs.is_cuda and recs.dtype == torch.uint8 and recs.numel() % DP40_BYTES == 0
        n = recs.numel() // DP40_BYTES
        cap = n if cap is None else int(cap)
        dev = recs.device
        st = stream or torch.cuda.current_stream(dev)
        with torch.cuda.stream(st):
            good = torch.empty(max(n, 1) * DP40_BYTES, dtype=torch.uint8, device=dev)
            counts = torch.empty(2, dtype=torch.int32, device=dev)
            bad = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
            nb = self.verify_scratch_bytes(n)
            scratch = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
            self.verify_raw(recs.data_ptr(), n, good.data_ptr(), counts.data_ptr(), bad.data_ptr(), cap, scratch.data_ptr(), nb,
                            st.cuda_stream)
            n_good, n_bad = (int(v) for v in counts.cpu().tolist())
            idx = bad[:min(n_bad, cap)].cpu().tolist()
        return good[:n_good * DP40_BYTES], n_bad, idx

    def verify_partition_scratch_bytes(self, n, world):
        """device scratch bytes verify_partition_raw needs for n records and `world` shards"""
        return int(self._lib.kgx_resolver_verify_partition_scratch_bytes(int(n), int(world)))

    def verify_partition_raw(self, recs, n, world, stride, out, counts, bad_idx, cap, scratch, scratch_bytes, stream=0):
        """kgx_resolver_verify_partition: verify_raw's check, then the good records grouped by the shard of `world` that owns
        their bucket, each group in input order, at out + shard * stride records (packed when stride = 0) -> counts (device,
        world + 1 uint32: each group's records, then the bad count) and bad_idx (device, the first cap bad indices); queued on
        `stream`, not waited for"""
        rc = self._lib.kgx_resolver_verify_partition(self._h, ctypes.c_void_p(int(recs)), int(n), int(world), int(stride),
                                                     ctypes.c_void_p(int(out)), ctypes.c_void_p(int(counts)),
                                                     ctypes.c_void_p(int(bad_idx)), int(cap), ctypes.c_void_p(int(scratch)),
                                                     int(scratch_bytes), ctypes.c_void_p(int(stream)))
        if rc != 0:
            raise RuntimeError(self._lib.kgx_resolver_last_error(self._h).decode())

    def verify_partition(self, recs, world, stride=0, cap=None, stream=None):
        """recs: a CUDA uint8 tensor of n x 40-byte records -> (out as a CUDA uint8 tensor of max(n, 1) records, or world x stride
        records with a stride, the good records per shard as a list, the number of bad records, the first cap (default: all)
        bad indices as a list); on `stream` or torch's current one, waited for"""
        import torch
        assert recs.is_cuda and recs.dtype == torch.uint8 and recs.numel() % DP40_BYTES == 0
        n = recs.numel() // DP40_BYTES
        cap = n if cap is None else int(cap)
        dev = recs.device
        st = stream or torch.cuda.current_stream(dev)
        with torch.cuda.stream(st):
            out = torch.empty((world * stride if stride else max(n, 1)) * DP40_BYTES, dtype=torch.uint8, device=dev)
            counts = torch.empty(world + 1, dtype=torch.int32, device=dev)
            bad = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
            nb = self.verify_partition_scratch_bytes(n, world)
            scratch = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
            self.verify_partition_raw(recs.data_ptr(), n, world, stride, out.data_ptr(), counts.data_ptr(), bad.data_ptr(), cap,
                                      scratch.data_ptr(), nb, st.cuda_stream)
            c = [int(v) for v in counts.cpu().tolist()]
            idx = bad[:min(c[world], cap)].cpu().tolist()
        return out, c[:world], c[world], idx

    def resolve(self, d_first, d_other, stream=None):
        """two lists of tagged distances (ints) -> [(key index, private key) or None]; on `stream` (a torch stream) or torch's
        current one, waited for"""
        import torch
        n = len(d_first)
        if n == 0:
            return []
        dev = torch.device("cuda", self.device)
        pairs = torch.from_numpy(np.ascontiguousarray(np.hstack([_limbs_u64(d_first, 2), _limbs_u64(d_other, 2)])).view(np.int64))
        st = stream or torch.cuda.current_stream(dev)
        with torch.cuda.stream(st):
            p = pairs.to(dev, non_blocking=False)
            key = torch.empty(n, dtype=torch.int32, device=dev)
            priv = torch.empty((n, 4), dtype=torch.int64, device=dev)
            self.run_raw(p.data_ptr(), n, key.data_ptr(), priv.data_ptr(), st.cuda_stream)
            key_h, priv_h = key.cpu().numpy().view(np.uint32), priv.cpu().numpy().view(np.uint64)
        return [None if k == NO_KEY else (int(k), sum(int(v) << (64 * w) for w, v in enumerate(pv))) for k, pv in zip(key_h.tolist(), priv_h)]


TABLE_ENTRIES = ("device", "host")   # DeviceDPTable(entries=): where the 32-byte entries live
HOST_ENTRIES = 1                     # KGX_DPT_HOST_ENTRIES (include/kgx.h)


def _entries_flags(entries):
    if entries not in TABLE_ENTRIES:
        raise ValueError("entries must be one of %s, not %r" % (", ".join(TABLE_ENTRIES), entries))
    return HOST_ENTRIES if entries == "host" else 0


class DeviceDPTable:
    """The rank-0 DP table in the memory of one GPU (libkgx.so, kgx_dptable_*): DPTable's add / __len__ / save_work /
    load_work_ex with exactly its results for the same records in the same order, inserted by CUDA kernels straight from device
    memory.  Its capacity (entries) is fixed at creation; an add that could pass it raises TableFull and changes nothing.
    add(resolver=) resolves the collisions of the add on the device (kgx_dptable_add_resolve).
    buckets=(lo, hi): a shard of the sharded table, holding the buckets [lo, hi) only (kgx_dptable_create_range).
    entries="host": the 32-byte entries in mapped, pinned host memory and only the index on the GPU (16 bytes of GPU memory
    per entry instead of 48), with exactly the same results (kgx_dptable_create_ex, KGX_DPT_HOST_ENTRIES)."""

    def __init__(self, capacity, device=None, max_events=4096, buckets=None, entries="device"):
        from ._lib import load_library as load_engine
        self._lib = load_engine()
        self.device = int(device if device is not None else 0)
        self.entries = entries
        lo, hi = (0, 1 << 18) if buckets is None else (int(buckets[0]), int(buckets[1]))
        self._h = ctypes.c_void_p(self._lib.kgx_dptable_create_ex(self.device, int(capacity), lo, hi, _entries_flags(entries)))
        if not self._h:
            raise RuntimeError(self._lib.kgx_dptable_last_error(None).decode())
        self.buckets = (lo, hi)
        self.capacity = int(capacity)
        self._ev = (Event * max_events)()
        self._evk = None                     # EventKey * max_events, made by the first add with a resolver
        self._cap = max_events
        self.threads = 0                     # no host workers

    @staticmethod
    def bytes_for(capacity, entries="device"):
        """GPU bytes of a table of that capacity and layout"""
        return DeviceDPTable.bytes_for_ex(capacity, entries)[0]

    @staticmethod
    def bytes_for_ex(capacity, entries="device"):
        """(GPU bytes, pinned host bytes) of a table of that capacity and layout"""
        from ._lib import load_library as load_engine
        host = ctypes.c_uint64(0)
        dev = int(load_engine().kgx_dptable_bytes_for_ex(int(capacity), _entries_flags(entries), ctypes.byref(host)))
        return dev, int(host.value)

    def close(self):
        if self._h:
            self._lib.kgx_dptable_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return int(self._lib.kgx_dptable_count(self._h))

    def memory_bytes(self):
        return int(self._lib.kgx_dptable_memory_bytes(self._h))

    def host_bytes(self):
        """pinned host bytes of the entries (0 with entries="device")"""
        return int(self._lib.kgx_dptable_host_bytes(self._h))

    def _err(self):
        return self._lib.kgx_dptable_last_error(self._h).decode()

    def reserve(self, n_records):
        """allocate now the scratch of adds of up to n_records records (adds otherwise grow it on demand)"""
        if self._lib.kgx_dptable_reserve(self._h, int(n_records), self._cap) != 0:
            raise RuntimeError("kgx_dptable_reserve: " + self._err())

    def add_raw(self, ptr, counts, stride, stream=0, resolver=None):
        """counts[r] records of rank r at device address ptr + r*stride*40 -> (return code, total events, Event array of the
        first min(total, max_events); with a resolver, EventKey records).  Raises TableFull (-2) and RuntimeError on a CUDA error
        (-3); -1 = malformed records skipped."""
        counts = [int(c) for c in counts]
        cnt = (ctypes.c_uint32 * len(counts))(*counts)
        ne = ctypes.c_uint32(0)
        args = (self._h, ctypes.c_void_p(int(ptr)), cnt, len(counts), int(stride))
        if resolver is None:
            out = self._ev
            rc = self._lib.kgx_dptable_add(*args, ctypes.cast(out, ctypes.c_void_p), self._cap, ctypes.byref(ne),
                                           ctypes.c_void_p(int(stream)))
        else:
            if self._evk is None:
                self._evk = (EventKey * self._cap)()
            out = self._evk
            rc = self._lib.kgx_dptable_add_resolve(*args, resolver._h, ctypes.cast(out, ctypes.c_void_p), self._cap, ctypes.byref(ne),
                                                   ctypes.c_void_p(int(stream)))
        if rc == -2:
            raise TableFull(self._err())
        if rc < -1:
            raise RuntimeError("kgx_dptable_add: " + self._err())
        return rc, ne.value, out

    def add(self, ptr, counts, stride, stream=0, resolver=None):
        """every rank's records of one step (device memory) -> list of (kind, rank, kidx, d_old, d_new) events; with a
        resolver (DeviceResolver on this table's GPU) (kind, rank, kidx, d_old, d_new, hit), hit = (key index, private key) of a
        collision event, or None: no key, or another kind of event"""
        rc, n, out = self.add_raw(ptr, counts, stride, stream, resolver)
        if rc != 0:
            raise RuntimeError("kgx_dptable_add: malformed DP record (h >= 2^18)")
        if resolver is None:
            return DPTable._events(self, n)
        evs = []
        for i in range(min(n, self._cap)):
            k = out[i]
            e = k.ev
            hit = None if k.key == NO_KEY else (int(k.key), sum(int(k.priv[w]) << (64 * w) for w in range(4)))
            evs.append((int(e.kind), int(e.rank), int(e.kidx), (int(e.d_old[0]), int(e.d_old[1])), (int(e.d_new[0]), int(e.d_new[1])), hit))
        return evs

    def add_dp40(self, buf, rank=0, stream=0):
        """DPTable.add_dp40 for records in device memory: buf = a CUDA uint8 tensor of n x 40 bytes"""
        assert buf.is_cuda and buf.numel() % DP40_BYTES == 0
        n = buf.numel() // DP40_BYTES
        counts = [0] * rank + [n]
        return self.add(buf.data_ptr() - rank * n * DP40_BYTES, counts, n, stream) if n else []

    def save_work(self, path, dp_bits, range_start, range_end, pubkey, total_count=0, total_time=0.0, total_walk=0, stream=0):
        rc = self._lib.kgx_dptable_save_work(self._h, os.fsencode(path),
                                             *_save_args(dp_bits, range_start, range_end, pubkey, total_count, total_time, total_walk),
                                             ctypes.c_void_p(int(stream)))
        if rc != 0:
            raise RuntimeError("kgx_dptable_save_work: cannot write %s: %s" % (path, self._err()))

    def load_work_ex(self, path, stream=0):
        """DPTable.load_work_ex into the device table; a file of more entries than the capacity raises TableFull"""
        rc, info = _load_work_ex(self._lib.kgx_dptable_load_work, self._h, path, ctypes.c_void_p(int(stream)))
        if rc == -28:                                            # -ENOSPC
            raise TableFull(self._err())
        if rc != 0:
            raise RuntimeError("kgx_dptable_load_work: %s" % self._err())
        return info

    def piece_bytes(self):
        """the size of this table's piece of a work file: its buckets' nbItem, maxItem and entries"""
        return int(self._lib.kgx_dptable_piece_bytes(self._h))

    def save_piece(self, path, offset, stream=0):
        """write this table's piece at byte `offset` of the existing file `path` (flushed and fsynced)"""
        rc = self._lib.kgx_dptable_save_range(self._h, os.fsencode(path), int(offset), ctypes.c_void_p(int(stream)))
        if rc != 0:
            raise RuntimeError("kgx_dptable_save_range: cannot write %s: %s" % (path, self._err()))

    def load_piece(self, path, max_entries, stream=0):
        """load_work_ex of this table's buckets only; more than max_entries entries in them raise TableFull"""
        rc, info = _load_work_ex(self._lib.kgx_dptable_load_range, self._h, path, ctypes.c_uint64(int(max_entries)),
                                 ctypes.c_void_p(int(stream)))
        if rc == -28:                                            # -ENOSPC
            raise TableFull(self._err())
        if rc != 0:
            raise RuntimeError("kgx_dptable_load_range: %s" % self._err())
        return info


class WorkHeader(collections.namedtuple("WorkHeader", "dp_bits range_start range_end key total_count total_time")):
    """The header's six fields as a tuple, and the file's version as the attribute `version` (outside the tuple, so the header
    still unpacks and compares as those six fields)"""

    def __new__(cls, dp_bits, range_start, range_end, key, total_count, total_time, version=0):
        self = super().__new__(cls, dp_bits, range_start, range_end, key, total_count, total_time)
        self.version = version
        return self


def read_work_header(path):
    """The fixed 156-byte HEADW header (Backup.cpp:368-394) without the table -> WorkHeader (dp_bits, range_start, range_end,
    (key x, key y), total_count, total_time; .version).  Needs no library."""
    with open(path, "rb") as f:
        raw = f.read(156)
    if len(raw) != 156 or struct.unpack_from("<I", raw)[0] != 0xFA6A8001:
        raise RuntimeError("%s is not a HEADW work file" % path)
    val = lambda o: int.from_bytes(raw[o:o + 32], "little")
    return WorkHeader(struct.unpack_from("<I", raw, 8)[0], val(12), val(44), (val(76), val(108)), struct.unpack_from("<Q", raw, 140)[0],
                      struct.unpack_from("<d", raw, 148)[0], struct.unpack_from("<I", raw, 4)[0])


class WorkInfo:
    """Header of a HEADW work file and where its kangaroos are."""

    def __init__(self, path, dp_bits, range_start, range_end, key, total_count, total_time, nb_walk, walk_offset):
        self.path, self.dp_bits, self.range_start, self.range_end, self.key = path, dp_bits, range_start, range_end, key
        self.total_count, self.total_time, self.nb_walk, self.walk_offset = total_count, total_time, nb_walk, walk_offset

    def walks(self, first=0, count=None):
        """kangaroos [first, first+count) of the file as a (count, 12) uint64 array of records (read from disk)."""
        count = self.nb_walk - first if count is None else count
        assert 0 <= first and first + count <= self.nb_walk
        return np.fromfile(self.path, dtype=np.uint64, count=count * 12, offset=self.walk_offset + first * WALK_BYTES).reshape(count, 12)
