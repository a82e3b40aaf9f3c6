"""Stand-alone multi-GPU driver of the jump engine: the role Kangaroo::Run / SolveKeyGPU (Kangaroo.cpp:913-1083,
510-644) plays in the reference, on the GPUs of one job: one process per GPU and an NCCL gather of the DP records to rank 0
(kangaroo_b200/dist.py).  Machines that join and leave use the reference's client/server mode instead, with
kangaroo_b200/server.py as the server.  Kept deliberately small: it exists to
exercise the engine end to end (BASELINE config 4) -- the full-featured caller remains the reference's own program
linked against the engine (INTEGRATION.md).

Per step (= one GPUEngine::Launch on every rank) nothing on the data path is Python:
  engine      kgx_collect(cap=0, relaunch=1): wait for launch i, start launch i+1, no host copy of records
  device      kgx_convert_dps: HashTable::Convert of launch i's DPs -> 40-byte `DP` records (Kangaroo.h:94-101)
  NCCL        all_gather(count) + gather(records) to rank 0          (dist.DPGather, wire "dp40")
  rank 0      one D2H copy -> (ingest thread, one step behind, overlapping the next launch) kgi_add: the reference's HashTable,
              bucket-sharded multi-threaded insert (ingest.DPTable)
              -> events: KGI_EV_COLLISION -> kgi_resolve (CollisionCheck/CheckKey with the reference's Secp256K1)
                         KGI_EV_RESET     -> (rank, kIdx) sent back to the owner, which re-creates that kangaroo
                                             (Kangaroo.cpp:601-609: CreateHerd(1) + SetKangaroo)
  all ranks   one small broadcast: [table stopped, n_resets, save next, chunks, n_solved, solved keys ..., (rank, kIdx) ...]

With --dp-table device, rank 0's table is ingest.DeviceDPTable in its GPU's memory (same events and work files): the step's
records are copied device to device into a staging buffer and inserted from there by the ingest thread on its own stream, no
host copy of them.  Its capacity is fixed; a full table stops the run (with --save-work, after writing the table it holds).
The insert resolves its tame/wild collisions on the same stream (ingest.DeviceResolver, kgi_resolve_multi's result against the
run's keys), so each collision event comes back with its key and private key; only --dp-table host loads
build/libkgx_ingest.so, the reference's HashTable and CheckKey.

With --dp-table sharded, every rank holds the device table of the buckets it owns and inserts them on an ingest thread of its
own: the records go to their owners (dist.DPExchange) in place of the gather, and a per-step block from every rank brings rank
0 the hits to claim (Solver._shard_round).  A full shard stops the run with the normal end-of-run save.

  single GPU :  python -m kangaroo_b200.solver in.txt --dp 12
  N GPUs     :  torchrun --nproc-per-node N -m kangaroo_b200.solver in.txt --dp 12

Work files (the reference's -w / -wi / -ws / -i, Backup.cpp): --save-work FILE writes the DP table, with --save-kangaroos also
every rank's herd (rank order, 96-byte records converted on the device, gathered to rank 0 in bounded chunks), at the end and
every --save-interval seconds; --resume FILE continues a run from such a file, or from one the reference wrote.  A file is a
consistent cut: its table holds the DPs of exactly the launches its herd has made, and its count is their jumps.  The save
decided at step k snapshots the herd on the device in stream order after launch i+1 (in flight at step k); step k+1
queues the table write on the ingest thread right behind launch i+1's DPs, so it writes the table of the cut; the herd chunks
follow over the next steps (Solver._save_start).  The end-of-run save does the same
with the launch in flight when the loop stops.  Kangaroos re-created at step k are re-created after the snapshot, so the
file holds them dead: a resumed run finds them again.  A save goes to FILE.tmp, is fsynced and renamed over FILE; a failed
save removes FILE.tmp and the run goes on.  On --resume only rank 0 reads the file.

--batch-keys saves and resumes through the same path with --batch-save FILE, --batch-save-interval SECS and --batch-resume
FILE: the work file of the cut followed by a batch block with every key, its solved flag and every kangaroo's target
(BatchSolver, kgx_workfile.h).
"""
import argparse
import collections
import contextlib
import ctypes
import functools
import os
import queue
import struct
import sys
import threading
import time

import numpy as np

from . import ecmath as ec
from .engine import GPUEngine, NB_JUMP, NB_RUN, WILD, random_herd_arrays
from .dist import DPExchange, DPGather, HerdGather, SlabView, DP40_BYTES, WALK_BYTES, owner_ranges
from .ingest import DPTable, DeviceDPTable, DeviceResolver, TableFull, EV_RESET, EV_COLLISION

ORDER = ec.N
MAX_RESETS = 255          # per step, carried in the control broadcast
MAX_KEYS = 65535          # --batch-keys: keys of one run (KGX_MAX_KEYS, the engine's uint16 targets)
MAX_SOLVED = 64           # --batch-keys: keys one step's control broadcast announces solved; more wait for the next step
SAVE_CHUNK = 1 << 18      # kangaroos per gather chunk of a save (24 MB buffer)
SAVE_CHUNKS_PER_STEP = 1  # chunks a step moves while a save is in progress (default herd: 17 steps)
SAVE_BUFFERS = 4          # rank 0's pinned chunk buffers queued to the writer
DP_TABLE_MARGIN = 4 << 30 # --dp-table device without a capacity: rank 0's free GPU memory after the engine, its staging
                          # buffers and the table's reserved per-add scratch, less this margin for NCCL, the gather buffer
                          # and torch's allocator.  Nothing else grows on the GPU: steps queued behind a save wait in host RAM
HOST_ENTRIES_MARGIN = 8 << 30   # --dp-table-entries host: host RAM (MemAvailable) left to the OS, torch, the pinned staging
                                # and save buffers and parked steps; the rest may hold pinned table entries


def init_dist():
    """torch.distributed for a multi-GPU run (WORLD_SIZE > 1), started once per process -> the module.  The backend comes from
    KGX_DIST_BACKEND: nccl (the default, one GPU per rank) or gloo, which lets several ranks share one GPU (the tests run a
    multi-rank solver on one GPU that way).  The collectives stay on CUDA tensors either way; HerdGather stages its
    point-to-point chunks through host memory under gloo."""
    import torch
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if not dist.is_initialized():
        backend = os.environ.get("KGX_DIST_BACKEND", "nccl")
        if backend == "nccl":
            dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    return dist


def scratch_bytes(n_records):
    """GPU memory of the device table's per-add scratch for adds of up to n_records records (kgx_dptable_reserve), rounded up"""
    m = 1024
    while m < n_records:
        m <<= 1
    return m * 80 + (16 << 20)


def default_table_capacity(free_bytes, margin=DP_TABLE_MARGIN, entries="device", host_limit=None):
    """the largest capacity whose device table of that layout (ingest.TABLE_ENTRIES) fits in free_bytes - margin, at most
    2^32-2 entries and, with entries="host", at most host_limit (host_entries_limit)"""
    room = free_bytes - margin
    cap = max(room // (16 if entries == "host" else 48), 0)
    while cap > 0 and DeviceDPTable.bytes_for(cap, entries) > room:
        cap = cap * 63 // 64
    cap = min(cap, (1 << 32) - 2)
    if entries == "host" and host_limit is not None:
        cap = min(cap, host_limit)
    return int(cap)


def mem_available():
    """the kernel's estimate of the host RAM available without swapping (/proc/meminfo MemAvailable), in bytes"""
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    raise RuntimeError("/proc/meminfo has no MemAvailable")


def host_entries_limit(available, tables, margin=HOST_ENTRIES_MARGIN):
    """--dp-table-entries host: the entries each of `tables` tables on this host may pin, at 32 bytes each, out of `available`
    bytes of host RAM less the margin"""
    return int(max(available - margin, 0) // max(int(tables), 1) // 32)


def tables_on_node(dp_table):
    """the device tables this host holds: one (rank 0's) for --dp-table device, one per local rank for sharded"""
    return int(os.environ.get("LOCAL_WORLD_SIZE", "1")) if dp_table == "sharded" else 1


def host_capacity_error(capacity, available, tables):
    """why an explicit --dp-table-capacity cannot hold host entries here, or None"""
    limit = host_entries_limit(available, tables)
    if capacity is not None and capacity > limit:
        return ("--dp-table-entries host: --dp-table-capacity %d entries would pin %.1f GB of host RAM, more than the host limit "
                "of %d entries (MemAvailable %.1f GB less %d GiB, shared by %d table(s) on this host, 32 bytes per entry)" %
                (capacity, 32 * capacity / 1e9, limit, available / 1e9, HOST_ENTRIES_MARGIN >> 30, tables))
    return None


def layout_note(entries):
    """the words the report lines add for a table's layout"""
    return " (host entries)" if entries == "host" else ""


def shard_headroom(world, max_found):
    """--dp-table sharded: the entries a shard keeps free.  A step brings a shard at most world * max_found records, and a run
    stopped at step k still inserts the launch in flight at its end, so a rank stops the run at the step where its bound plus
    two steps' records would pass its capacity."""
    return 2 * world * max_found


def sharded_capacity_error(capacity, world, max_found=1 << 17):
    """why --dp-table-capacity cannot be a shard's capacity on `world` ranks, or None"""
    if capacity is not None and capacity <= shard_headroom(world, max_found):
        return ("--dp-table sharded: a shard of capacity %d entries cannot hold the %d records two steps may bring on %d GPUs "
                "(2 x GPUs x %d); give more than %d" % (capacity, shard_headroom(world, max_found), world, max_found,
                                                        shard_headroom(world, max_found)))
    return None


# The per-step block of --dp-table sharded: every rank's report to rank 0, all gathered, a fixed number of int64 words.
#   0 hits, 1 resets, 2 shard entries, 3 stop (0 no, 1 shard full, 2 insert failed), 4 work-file piece size (-1 none),
#   5 piece written (0 no news, 1 ok, 2 failed), 6 busy (ingest work or reports outstanding), 7 herd chunks every rank moves
#   after this round (rank 0's block, in the end-of-run drain; the control broadcast carries them during the run),
#   then the stop message, the piece's error (BLOCK_MSG words of UTF-8 each), hits (key index, private key in 4 words, rank,
#   kIdx) and resets (rank, kIdx).  Hits and resets over the caps wait for the next step.
BLOCK_MSG = 32
BLOCK_HITS = MAX_SOLVED
BLOCK_WORDS = 8 + 2 * BLOCK_MSG + 7 * BLOCK_HITS + 2 * MAX_RESETS
_M64 = (1 << 64) - 1


def _msg_words(text):
    raw = text.encode("utf-8", "replace")[:8 * BLOCK_MSG - 1]
    return np.frombuffer(raw.ljust(8 * BLOCK_MSG, b"\0"), np.int64)


def encode_block(hits, resets, count, stop=0, msg="", size=-1, done=0, err="", busy=0, chunks=0):
    """-> (int64 array of BLOCK_WORDS, hits over the cap, resets over the cap)"""
    b = np.zeros(BLOCK_WORDS, np.int64)
    h, r = hits[:BLOCK_HITS], resets[:MAX_RESETS]
    b[:8] = [len(h), len(r), count, stop, size, done, busy, chunks]
    b[8:8 + BLOCK_MSG] = _msg_words(msg)
    b[8 + BLOCK_MSG:8 + 2 * BLOCK_MSG] = _msg_words(err)
    o = 8 + 2 * BLOCK_MSG
    for i, (idx, priv, rk, kidx) in enumerate(h):
        row = [idx] + [(priv >> (64 * k)) & _M64 for k in range(4)] + [rk, kidx]
        b[o + 7 * i:o + 7 * i + 7] = np.array(row, np.uint64).view(np.int64)
    o += 7 * BLOCK_HITS
    for i, (rk, kidx) in enumerate(r):
        b[o + 2 * i:o + 2 * i + 2] = [rk, kidx]
    return b, hits[len(h):], resets[len(r):]


def decode_block(b):
    """encode_block's array -> dict(hits, resets, count, stop, msg, size, done, err, busy, chunks)"""
    b = np.asarray(b, np.int64)
    nh, nr = int(b[0]), int(b[1])
    text = lambda w: w.tobytes().rstrip(b"\0").decode("utf-8", "replace")
    o = 8 + 2 * BLOCK_MSG
    hits = []
    for i in range(nh):
        w = [int(v) for v in b[o + 7 * i:o + 7 * i + 7].view(np.uint64)]
        hits.append((w[0], sum(w[1 + k] << (64 * k) for k in range(4)), w[5], w[6]))
    o += 7 * BLOCK_HITS
    resets = [(int(b[o + 2 * i]), int(b[o + 2 * i + 1])) for i in range(nr)]
    return dict(hits=hits, resets=resets, count=int(b[2]), stop=int(b[3]), msg=text(b[8:8 + BLOCK_MSG]), size=int(b[4]),
                done=int(b[5]), err=text(b[8 + BLOCK_MSG:8 + 2 * BLOCK_MSG]), busy=int(b[6]), chunks=int(b[7]))


def piece_offsets(sizes):
    """where each shard's piece of a work file starts (after the 156-byte header), then where the table ends"""
    return [156 + sum(sizes[:r]) for r in range(len(sizes) + 1)]


def work_header(dp_bits, range_start, range_end, pub, total_count, total_time):
    """the 156-byte HEADW header (Backup.cpp:368-394) the tables write"""
    v = lambda x: int(x).to_bytes(32, "little")
    return (struct.pack("<III", 0xFA6A8001, 0, int(dp_bits)) + v(range_start) + v(range_end) + v(pub[0]) + v(pub[1]) +
            struct.pack("<Qd", int(total_count), float(total_time)))


def create_jump_table(range_power):
    """Kangaroo::CreateJumpTable (Kangaroo.cpp:742-832, non-symmetry): 32 distances of rangePower/2+1 bits from MT19937
    seeded 0x600DCAFE (constant "for compatibility of workfiles"), redrawn until the mean is within 2^(jumpBit-1.05 ..
    -0.95); points = d*G.  numpy's RandomState is the same MT19937 with the same seeding, Int::Rand(nbit) consumes
    nbit/32 + 1 words (Int.cpp:988-1001)."""
    jump_bit = min(range_power // 2 + 1, 128)
    rs = np.random.RandomState(0x600DCAFE)
    lo, hi = 2.0 ** (jump_bit - 1.05), 2.0 ** (jump_bit - 0.95)
    nb, left = jump_bit // 32, jump_bit % 32
    for _ in range(100):
        dist = []
        for _i in range(NB_JUMP):
            words = [int(v) for v in rs.randint(0, 2**32, size=nb + 1, dtype=np.uint64)]
            words[nb] &= (1 << left) - 1
            v = sum(w << (32 * k) for k, w in enumerate(words))
            dist.append(v or 1)
        if lo < sum(dist) / NB_JUMP < hi:
            break
    pts = [ec.mul(d) for d in dist]
    return dist, [p[0] for p in pts], [p[1] for p in pts]


def dp_mask(bits):
    """Kangaroo::SetDP (Kangaroo.cpp:154-164)"""
    return 0 if bits == 0 else (~((1 << (64 - min(bits, 64))) - 1)) & 0xFFFFFFFFFFFFFFFF


# Rank 0's DP table, --dp-table host or device.  Each step's records land in one of two staging buffers: while the ingest
# thread inserts step k's records, step k+1's land in the other one.  The NCCL kernels of a step cannot start before the jump
# launch that occupies every SM has finished, so without this decoupling the insert would sit exposed between two launches.
# A step parked behind a save (Solver._submit) gets a buffer of its own in host RAM instead.  stage() runs on the main
# thread; insert() and save() (the header and the table of a work file) run on the ingest thread.
class HostTable:
    """the reference's HashTable in host RAM (ingest.DPTable), fed through pinned buffers"""
    label = "ingest"

    def __init__(self, torch, n_records, threads):
        self.torch = torch
        self.dps = DPTable(threads=threads)
        self._bufs = [torch.empty(n_records * DP40_BYTES, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self._i = 0
        self.save = self.dps.save_work
        self.info = "ingest threads: %d" % self.dps.threads

    def stage(self, counts, stride, src, park):
        nbytes = len(counts) * stride * DP40_BYTES
        if park:
            buf = self.torch.empty(nbytes, dtype=self.torch.uint8)
        else:
            buf, self._i = self._bufs[self._i], self._i ^ 1
        buf[:nbytes].copy_(src[:nbytes], non_blocking=True)
        self.torch.cuda.current_stream().synchronize()
        h = buf.numpy()
        return [(r, h[r * stride * DP40_BYTES: (r * stride + c) * DP40_BYTES]) for r, c in enumerate(counts)]

    def insert(self, segments):
        return [ev for r, buf in segments if buf.size != 0 for ev in self.dps.add_dp40(buf, r)]

    def close(self):
        self.dps.close()


class DeviceTable:
    """ingest.DeviceDPTable in rank 0's GPU memory, fed from device staging buffers on a stream of the ingest thread's own.
    The two staging buffers and a third one, which takes parked records back to the GPU, are all the GPU memory the records
    take; the table's per-add scratch is reserved up front, so the table needs no allocation while it runs.  Every insert
    resolves its collisions against the run's keys on the same stream (ingest.DeviceResolver): its events carry their hits."""
    label = "device table"

    def __init__(self, torch, n_records, device, capacity, wait_copy, keys, start, buckets=None, entries="device", tables=1):
        """wait_copy: the records' source is rewritten unordered with torch's stream (the engine's own buffer, on one GPU).
        keys: the key table the collisions are resolved against (DPTable.key_table: K = key - start*G per key).
        buckets: (lo, hi) of a shard (ShardedTable).  entries: the table's layout (ingest.TABLE_ENTRIES); with "host" the
        default capacity also keeps to this host's share of its RAM among `tables` tables (host_entries_limit)"""
        self.torch, self._wait_copy = torch, wait_copy
        self.resolver = DeviceResolver(keys, start, device=device)
        self._bufs = [torch.empty(n_records * DP40_BYTES, dtype=torch.uint8, device=torch.device("cuda", device)) for _ in range(3)]
        self._back = self._bufs.pop()
        if not capacity:
            capacity = default_table_capacity(torch.cuda.mem_get_info(device)[0] - scratch_bytes(n_records), entries=entries,
                                              host_limit=host_entries_limit(mem_available(), tables) if entries == "host" else None)
        self.dps = DeviceDPTable(capacity, device=device, buckets=buckets, entries=entries)
        self.dps.reserve(n_records)
        self._stream = torch.cuda.Stream(device=device)
        self._i = 0
        self.save = functools.partial(self.dps.save_work, stream=self._stream.cuda_stream)
        self.info = "dp table: device, capacity %d entries (%.2f GB)" % (self.dps.capacity, self.dps.memory_bytes() / 1e9)
        if entries == "host":
            self.info += ", entries in pinned host memory (%.2f GB)" % (self.dps.host_bytes() / 1e9)

    def stage(self, counts, stride, src, park):
        """the records are copied device to device (torch's stream), since the gather buffer and the engine's record buffer
        are rewritten by the next step; insert() runs behind that copy"""
        nbytes = len(counts) * stride * DP40_BYTES
        if park:
            buf = self.torch.empty(nbytes, dtype=self.torch.uint8)
            buf.copy_(src[:nbytes])                         # to pageable memory: complete when it returns
            return buf, list(counts), stride, None
        buf, self._i = self._bufs[self._i], self._i ^ 1
        buf[:nbytes].copy_(src[:nbytes], non_blocking=True)
        ev = self.torch.cuda.Event()
        ev.record()
        if self._wait_copy:
            ev.synchronize()
        return buf, list(counts), stride, ev

    def insert(self, batch):
        buf, counts, stride, ev = batch
        if ev is None:                                      # parked in host RAM: back to the GPU, on this stream
            with self.torch.cuda.stream(self._stream):
                self._back[:buf.numel()].copy_(buf)
            buf = self._back
        else:
            self._stream.wait_event(ev)                     # the records' copy into the staging buffer
        return self.dps.add(buf.data_ptr(), counts, stride, self._stream.cuda_stream, self.resolver)

    def close(self):
        self.dps.close()
        self.resolver.close()


class ShardedTable(DeviceTable):
    """--dp-table sharded: this rank's shard, a DeviceDPTable of the buckets the rank owns, fed what DPExchange brought it.
    Its capacity is the shard's; save_piece writes its piece of a work file at an offset."""
    label = "sharded table"

    def __init__(self, torch, n_records, device, capacity, keys, start, buckets, entries="device"):
        super().__init__(torch, n_records, device, capacity, False, keys, start, buckets, entries, tables_on_node("sharded"))
        self.save_piece = functools.partial(self.dps.save_piece, stream=self._stream.cuda_stream)


class WorkFile:
    """One work file as it is written: begin() puts the header and the table in FILE.tmp, append() adds herd records and
    finish() fsyncs it, renames it over FILE and fsyncs the directory, so the previous FILE stays whole until then.  After an
    error nothing more is written and finish() removes FILE.tmp."""

    def __init__(self, path, t0):
        self.path, self.tmp, self.t0, self.err, self.f = path, path + ".tmp", t0, None, None

    def begin(self, write_table):
        """write_table(path): the header and the table"""
        try:
            write_table(self.tmp)
            self.f = open(self.tmp, "ab")
        except (OSError, RuntimeError) as e:
            self.err = str(e)

    def append(self, data):
        try:
            if self.f is not None and self.err is None:
                self.f.write(data)
        except OSError as e:
            self.err = str(e)

    def finish(self):
        """-> (path, MB, seconds since t0, error or None)"""
        size = 0
        try:
            if self.err is None:
                self.f.flush()
                os.fsync(self.f.fileno())
                size = self.f.tell()
                self.f.close()
                os.replace(self.tmp, self.path)
                dfd = os.open(os.path.dirname(os.path.abspath(self.path)), os.O_RDONLY)
                try:
                    os.fsync(dfd)
                finally:
                    os.close(dfd)
        except OSError as e:
            self.err = str(e)
        if self.f is not None:
            self.f.close()                                  # a no-op when closed above
        if self.err is not None:
            with contextlib.suppress(OSError):
                os.remove(self.tmp)
        return self.path, size / 1048576.0, time.perf_counter() - self.t0, self.err


class Solver:
    def __init__(self, start, end, pub, dp_bits, grid=None, max_found=1 << 17, seed=None, ingest_threads=0,
                 save_work="", save_interval=0.0, save_kangaroos=False, resume=None, dp_table="host", dp_table_capacity=None,
                 dp_table_entries="device"):
        import torch
        self.torch = torch
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(self.local)
        self.dist = init_dist() if self.world > 1 else None
        self.start, self.end, self.pub, self.dp_bits = start, end, pub, dp_bits
        width = end - start
        self.range_power = width.bit_length()                         # Kangaroo::InitRange (:877-890)
        self.wdiv2 = width >> 1
        # Kangaroo::InitSearchKey (:892-909): keyToSearch = P - start*G
        self.key = ec.add(pub, ec.neg(ec.mul(start))) if start else pub
        self.key_table = self._key_table()
        gx, gy = grid or GPUEngine.GetGridSize(self.local, 0, 0)
        self.eng = GPUEngine(gx, gy, self.local, max_found)
        self.table = create_jump_table(self.range_power)
        self.eng.SetParams(dp_mask(dp_bits), *self.table)
        self.eng.SetWildOffset(self.wdiv2)
        # Kangaroo::CreateHerd (:670-738): tame d in [0, 2^rangePower), wild d - width/2; points on the device
        n = self.eng.nbKangaroo
        self.rng = np.random.Generator(np.random.PCG64((seed if seed is not None else int(time.time())) * 1000 + self.rank))
        sc, d128 = random_herd_arrays(n, self.range_power, self.wdiv2, self.rng)
        self._create_herd(sc, d128)
        self.sharded = dp_table == "sharded"
        self.gather = (DPGather(self.eng, self.dist, self.rank, self.world, torch, wire="dp40") if self.world > 1 and not self.sharded
                       else None)
        # rank 0's table stopped taking records: "full" (TableFull) or "error" (any other failure of an insert), with its message
        self.table_msg, self.table_kind, self.table_stopped = None, None, False
        self.shard_msg, self.shard_stop, self.exchange = None, False, None   # --dp-table sharded (_init_shard)
        self.last_saved = None              # rank 0: path of the last save that succeeded
        self.full_saved = None              # rank 0: (path, count, error or None) of the save a full table made
        self.parked = 0                     # rank 0: steps whose records waited in host RAM behind a save
        self.found = None                   # rank 0: the private key, once found
        self._announce = []                 # rank 0: keys solved, not yet in a control broadcast
        self.dpt = self.dps = None          # rank 0: HostTable / DeviceTable, and the table it holds
        self.entries = dp_table_entries     # the device table's layout: "device" or "host" (its entries in pinned host RAM)
        if self.sharded:
            self._init_shard(max_found, dp_table_capacity)
        elif self.rank == 0:
            self.dpt = (DeviceTable(torch, self.world * max_found, self.local, dp_table_capacity, self.gather is None, self.key_table,
                                    self.start, entries=dp_table_entries) if dp_table == "device"
                        else HostTable(torch, self.world * max_found, ingest_threads))
            self.dps = self.dpt.dps
        self._work = queue.Queue()
        self._done = queue.Queue()
        self._pending = 0
        self._acc_hits, self._acc_resets = [], []
        self._wf = None                     # ingest thread: the scheduled work file being written
        self._thread = None
        if self.rank == 0 or self.sharded:
            self._thread = threading.Thread(target=self._ingest_loop, daemon=True)
            self._thread.start()
        self._ctrl = torch.zeros(5 + MAX_SOLVED + 2 * MAX_RESETS, dtype=torch.int64, device="cuda")
        self.jumps = 0
        self.same_herd = 0                  # every rank: kangaroos listed to re-create by the control broadcasts
        self.resets_done = 0                # every rank: kangaroos of its herd re-created
        self.resets_reported = 0            # rank 0: dead kangaroos the table reported during the run, and the most in one step
        self.resets_most = 0
        self.recreated = 0                  # after run(): kangaroos re-created on every rank
        self._reset_backlog = []            # rank 0: resets past MAX_RESETS of a broadcast, sent first in the next one
        self.t_ingest = 0.0
        self.stop = False
        self.save_path, self.save_interval, self.save_kangaroos = save_work, float(save_interval), bool(save_kangaroos)
        self.time_offset = 0.0
        self.herd = (HerdGather(self.dist, self.rank, self.world, torch, n, torch.device("cuda", self.local), SAVE_CHUNK)
                     if save_kangaroos or resume else None)
        self._save_due = False              # decided at the end of step k, started in step k+1
        self._chunks_next = 0               # herd chunks step k+1 moves (decided at the end of step k)
        self._saving = False                # herd chunks of the current save still to move
        self._save_left, self._save_steps, self._save_stats, self._step_times = [], [], [], []
        self._saved = queue.Queue()         # ingest thread -> main: (path, MB, seconds, error) per finished save
        self._chunk_pool = queue.Queue()
        if self.rank == 0 and save_kangaroos:
            for _ in range(SAVE_BUFFERS):
                self._chunk_pool.put(torch.empty(SAVE_CHUNK * WALK_BYTES, dtype=torch.uint8).pin_memory())
        self.saves = []                     # (MB, seconds) per save, rank 0
        self.save_error = None
        if resume:
            self._resume(resume)
        self.jumps0 = self.jumps

    def _create_herd(self, sc, d128):
        self.eng.CreateHerdRaw(sc, d128, self.key)

    def _key_table(self):
        """the keys a collision is resolved against: the one key of the run"""
        return DPTable.key_table([self.key])

    def _hit(self, ev):
        """a collision event -> (key index, private key) or None.  The device tables resolved it with the insert; the host table
        runs the reference's CheckKey (Kangaroo.cpp:255-302) on the key."""
        if len(ev) > 5:
            return ev[5]
        priv = self.dps.resolve(ev[3], ev[4], self.key, self.start)
        return None if priv is None else (0, priv)

    # -- --dp-table sharded ---------------------------------------------------------------------------------------------
    # Every rank holds the shard of the buckets it owns (dist.owner_ranges) and runs an ingest thread of its own, one step
    # behind like rank 0's.  Per step: DPExchange brings each rank the records of its buckets; each rank's main thread then
    # sends every rank its block (encode_block: hits, resets, its shard's entries, a stop flag, its work-file piece's news), and
    # rank 0 claims the hits of all of them before the control broadcast.  A work file of the cut decided at step k: each rank's
    # ingest thread, right behind step k+1's records, reports its piece's size; once every size is in, every rank knows the
    # offsets and its ingest thread writes its piece there; rank 0 writes the header first and the kangaroos after the last
    # piece, and renames the file once every rank reported its piece written.
    def _init_shard(self, max_found, capacity):
        torch = self.torch
        err = sharded_capacity_error(capacity, self.world, max_found)
        if err:
            raise ValueError(err)
        self.buckets = owner_ranges(self.world)[self.rank]
        self.headroom = shard_headroom(self.world, max_found)
        self.dpt = ShardedTable(torch, self.world * max_found, self.local, capacity, self.key_table, self.start, self.buckets,
                                self.entries)
        self.dps = self.dpt.dps
        if self.dps.capacity <= self.headroom:
            raise RuntimeError(sharded_capacity_error(self.dps.capacity, self.world, max_found))
        self.exchange = DPExchange(self.eng, self.dist, self.rank, self.world, torch, max_found=max_found)
        caps = [self.dps.capacity]
        if self.dist is not None:
            t = torch.tensor([self.dps.capacity], dtype=torch.int64, device="cuda")
            g = torch.empty(self.world, dtype=torch.int64, device="cuda")
            self.dist.all_gather_into_tensor(g, t)
            caps = [int(v) for v in g.cpu().tolist()]
        self.shard_caps = caps
        self.dpt.info = ("dp table: sharded over %d GPUs, %d entries in all (rank 0: buckets [%d, %d), %d entries, %.2f GB)" %
                         (self.world, sum(caps), self.buckets[0], self.buckets[1], caps[0], self.dps.memory_bytes() / 1e9))
        if self.entries == "host":
            self.dpt.info += ", entries in pinned host memory (rank 0: %.2f GB)" % (self.dps.host_bytes() / 1e9)
        self.shard_total = 0                # entries of all shards, as the last blocks reported them
        self.shard_hits = [0] * self.world  # rank 0: collisions resolved to a key on each shard
        self.shard_msg = None               # rank 0: why a full shard stopped the run
        self.shard_stop = False             # every rank: a shard is full, the run ends with the normal end-of-run save
        self._handed = collections.deque()  # records of the steps handed to the ingest thread and not yet inserted
        self._handed_done = 0
        self._ingested = 0                  # ingest thread: steps inserted; _shard_count: the shard's entries after them
        self._shard_count = 0
        self._piece_q = queue.Queue()       # ingest thread -> main: ("size", bytes) / ("done", error or None) of a piece
        self._offsets_q = queue.Queue()     # main -> ingest thread: the offsets of every piece of the file being written
        self._pieces_result = queue.Queue() # rank 0, main -> ingest thread: every piece written (None) or the first error
        self._pieces_open = 0               # pieces queued on this rank whose "done" no block has carried yet
        self._sizes, self._pstat = {}, {}

    def _shard_round(self, drain=False):
        """every rank, once per step (and in the end-of-run drain): the blocks of all ranks.  -> (hits, resets) of every rank on
        rank 0, ([], []) elsewhere; and whether any rank still has work or news outstanding"""
        torch = self.torch
        hits, resets = self._harvest()
        done = self._ingested
        while self._handed_done < done:
            self._handed.popleft()
            self._handed_done += 1
        count = self._shard_count
        bound = count + sum(self._handed)
        stop, msg = 0, ""
        if self.table_msg is not None:
            stop, msg = 2, "shard %d: %s" % (self.rank, self.table_msg)
        elif not drain and bound + self.headroom > self.dps.capacity:
            stop, msg = 1, ("shard %d of %d (buckets [%d, %d)) holds up to %d entries of its capacity %d, and the next two steps "
                            "may bring %d" % (self.rank, self.world, self.buckets[0], self.buckets[1], bound, self.dps.capacity,
                                              self.headroom))
        size, pdone, perr = -1, 0, ""
        if not self._piece_q.empty():
            kind, v = self._piece_q.get()
            if kind == "size":
                size = v
            else:
                pdone, perr = (1, "") if v is None else (2, v)
                self._pieces_open -= 1
        busy = int(self._pending > 0 or self._pieces_open > 0 or self._saving)
        chunks = 0                                      # the drain moves herd chunks as rank 0's writer frees buffers
        if drain and self.rank == 0 and self._saving:
            chunks = min(len(self._save_left), self._chunk_pool.qsize())
        blk, self._acc_hits, self._acc_resets = encode_block(hits, resets, count, stop, msg, size, pdone, perr, busy, chunks)
        busy |= int(len(self._acc_hits) > 0 or len(self._acc_resets) > 0)
        blk[6] = busy
        if self.dist is not None:
            mine = torch.from_numpy(blk).to("cuda")
            allb = torch.empty(self.world * BLOCK_WORDS, dtype=torch.int64, device="cuda")
            self.dist.all_gather_into_tensor(allb, mine)
            blocks = [decode_block(b) for b in allb.cpu().numpy().reshape(self.world, BLOCK_WORDS)]
        else:
            blocks = [decode_block(blk)]
        for r, b in enumerate(blocks):
            if b["size"] >= 0:
                self._sizes[r] = b["size"]
            if b["done"]:
                self._pstat[r] = b["err"] if b["done"] == 2 else None
        if len(self._sizes) == self.world:              # every piece's size: the offsets (the same on every rank)
            self._offsets_q.put(piece_offsets([self._sizes[r] for r in range(self.world)]))
            self._sizes = {}
        if len(self._pstat) == self.world:              # every piece written or failed
            if self.rank == 0:
                errs = ["rank %d: %s" % (r, self._pstat[r]) for r in range(self.world) if self._pstat[r] is not None]
                self._pieces_result.put("; ".join(errs) if errs else None)
            self._pstat = {}
        self.shard_total = sum(b["count"] for b in blocks)
        self._shard_busy = any(b["busy"] for b in blocks)
        self._drain_chunks = blocks[0]["chunks"]
        if self.rank != 0:
            return [], []
        for r, b in enumerate(blocks):
            self.shard_hits[r] += len(b["hits"])
            if b["stop"] == 2 and self.table_msg is None:
                self.table_msg, self.table_kind = b["msg"], "error"
            elif b["stop"] == 1 and self.shard_msg is None:
                self.shard_msg = b["msg"]
        return [h for b in blocks for h in b["hits"]], [rk for b in blocks for rk in b["resets"]]

    def _shard_drain(self):
        """every rank, after the loop: blocks go round until every rank's records are inserted, its hits reported and the
        save in progress done: its herd chunks moved, as rank 0's writer frees buffers (that writer waits for the pieces'
        offsets, which only these rounds bring), and its pieces written"""
        while True:
            if (self._pending or self._pieces_open or self._saving) and self._done.empty() and self._piece_q.empty():
                time.sleep(0.002)
            hits, _ = self._shard_round(drain=True)
            if self.rank == 0:
                self._claim(hits, [])
            if self._drain_chunks:
                self._save_progress(self._drain_chunks)
            if not self._shard_busy:
                return

    def _write_piece(self, err):
        """ingest thread, behind the cut's records: this shard's piece of the file -> the offset where the table ends"""
        self._piece_q.put(("size", self.dps.piece_bytes()))
        offsets = self._offsets_q.get()
        if err is None and self.table_msg is not None:
            err = "the DP table lacks DPs of the launches this file would count (%s)" % self.table_msg
        if err is None:
            try:
                self.dpt.save_piece(self.save_path + ".tmp", offsets[self.rank])
            except RuntimeError as e:
                err = str(e)
        self._piece_q.put(("done", err))
        return offsets[-1]

    def table_entries(self):
        """entries of the DP table (every shard's, as last reported, with --dp-table sharded)"""
        return self.shard_total if self.sharded else len(self.dps)

    # -- work files ------------------------------------------------------------------------------------------------
    def _resume(self, path):
        """Kangaroo::LoadWork + FetchWalks (Backup.cpp:149-231): rank 0 loads the table; rank r takes the file's kangaroos
        [o_r, o_r + n_r) as its kIdx 0..n_r-1 (o_r = herd sizes of the lower ranks), verified on the device; the ones the
        file lacks keep the fresh random herd made above.  Only rank 0 reads the file; it sends every rank its records."""
        torch = self.torch
        info = torch.zeros(4, dtype=torch.int64, device="cuda")
        w = self._load_table(path)
        if self.rank == 0:
            info.copy_(torch.tensor([w.nb_walk, w.walk_offset, w.total_count, 0], dtype=torch.int64))
            self.time_offset = w.total_time
        if self.dist is not None:
            self.dist.broadcast(info, 0)
        nb_walk, offset, count, _ = (int(v) for v in info.cpu().tolist())
        self.jumps = count
        take = max(0, min(self.eng.nbKangaroo, nb_walk - self.herd.offsets[self.rank]))
        if self.rank == 0:
            print("Resume %s: %d DPs, count 2^%.2f, %d kangaroos in the file for %d in the herd" %
                  (path, self.table_entries(), np.log2(max(count, 1)), nb_walk, self.herd.total), flush=True)
            if nb_walk > self.herd.total:
                print("Warning: %d unhandled kangaroos" % (nb_walk - self.herd.total), flush=True)   # Kangaroo.cpp FectchKangaroos

        def read(first, cnt):                                   # rank 0 only
            return np.fromfile(path, dtype=np.uint8, count=cnt * WALK_BYTES, offset=offset + first * WALK_BYTES)

        t0 = time.perf_counter()
        recs = self.herd.scatter(nb_walk, read)                 # this rank's records, sent by rank 0 in bounded chunks
        bad = self.eng.ImportKangaroos(recs, self.key, verify=True) if take else 0
        if self.dist is not None:                               # every rank refuses together (none left waiting in a collective)
            t = torch.tensor([bad], dtype=torch.int64, device="cuda")
            self.dist.all_reduce(t)
            bad = int(t.item())
        if bad:
            raise RuntimeError("%s: %d kangaroos are not at d*G (tame) / key + d*G (wild): the file belongs to another key "
                               "or range" % (path, bad))
        if take:
            print("rank %d: %d kangaroos imported and verified in %.2f s" % (self.rank, take, time.perf_counter() - t0), flush=True)

    def _load_table(self, path):
        """the file's table into rank 0's table -> its WorkInfo on rank 0, None elsewhere.  --dp-table sharded: every rank
        loads its buckets; a shard the file's entries would leave less than the stop headroom refuses the run on every rank,
        before the first step."""
        if not self.sharded:
            return self.dps.load_work_ex(path) if self.rank == 0 else None
        torch = self.torch
        limit = self.dps.capacity - self.headroom
        w, err = None, None
        try:
            w = self.dps.load_piece(path, limit)
        except TableFull as e:
            err = e
        flags = [1 if err is not None else 0, len(self.dps)]
        if self.dist is not None:
            t = torch.tensor(flags, dtype=torch.int64, device="cuda")
            g = torch.empty(2 * self.world, dtype=torch.int64, device="cuda")
            self.dist.all_gather_into_tensor(g, t)
            flags = [int(v) for v in g.cpu().tolist()]
        refused = [r for r in range(self.world) if flags[2 * r]]
        if refused:
            r = refused[0]
            lo, hi = owner_ranges(self.world)[r]
            raise RuntimeError("--dp-table sharded: %s: buckets [%d, %d) of shard %d hold more than its capacity %d less the stop "
                               "headroom %d (%d entries); resume it on more GPUs, with a larger --dp-table-capacity or "
                               "--dp-table host" % (path, lo, hi, r, self.shard_caps[r], self.headroom,
                                                    self.shard_caps[r] - self.headroom))
        self.shard_total = sum(flags[1::2])
        self._shard_count = len(self.dps)
        return w

    def _export(self, first, count, dst):
        self.eng.SnapshotExport(first, count, dst.data_ptr())

    # A save runs alongside the launches.  Its first step queues the table write on the ingest thread right behind the DPs of
    # the cut (that thread alone touches the table, so it writes the table of the cut); then every step moves up to
    # SAVE_CHUNKS_PER_STEP herd chunks (device conversion + gather to rank 0 + copy into a free pinned buffer) and queues their
    # writes behind it.  The ingest thread writes, fsyncs and renames.  A step moves a chunk only when rank 0 has a pinned
    # buffer the writer has freed, so the step loop never waits for the disk: a slow disk only makes the save take more steps.
    def _save_start(self, kangaroos, chunks):
        """first step of a save of the current cut: with kangaroos, the snapshot was taken one step earlier"""
        self._saving = True
        self._save_left = list(range(len(self.herd.plan))) if kangaroos else []
        self._save_steps = []                                  # times of the steps that moved this save
        self._save_stats.append(self._save_steps)
        if self.sharded:
            self._pieces_open += 1                             # every rank writes its piece of the table
        if self.rank == 0:
            nwalk = self.herd.total if kangaroos else 0
            self._work.put(("begin", self.jumps, self.time_offset + time.time() - self.t_start, nwalk, time.perf_counter(),
                            self._cut(kangaroos)))
        else:
            self._cut(kangaroos)                               # every rank takes part (--batch-keys: the targets' gather)
            if self.sharded:
                self._work.put(("piece",))
        self._save_progress(chunks)

    def _save_progress(self, chunks):
        if not self._saving:
            return
        while self._save_left and chunks > 0:
            j = self._save_left.pop(0)
            chunks -= 1
            v = self.herd.chunk(j, self._export)
            if self.rank == 0:
                buf = self._chunk_pool.get()                     # back-pressure: the writer frees buffers as it goes
                buf[:v.numel()].copy_(v)
                self._work.put(("chunk", buf, v.numel()))
        if not self._save_left:
            if self.rank == 0:
                self._work.put(("end",))
            self._saving = False

    def _write(self, job):
        """ingest thread: one piece of a scheduled work file (jobs arrive in file order)"""
        kind = job[0]
        if kind == "begin":
            count, total_time, nwalk, t0, self._wf_cut = job[1:]
            self._wf = WorkFile(self.save_path, t0)
            if self.sharded:
                self._begin_sharded(self._wf, count, total_time, nwalk)
            elif self.table_msg is not None:
                self._wf.err = "the DP table lacks DPs of the launches this file would count (%s)" % self.table_msg
            else:
                self._write_table(self._wf, count, total_time, nwalk)
        elif kind == "piece":
            self._write_piece(None)
        elif kind == "chunk":
            buf, nbytes = job[1], job[2]
            try:
                self._wf.append(memoryview(buf.numpy()[:nbytes]))
            finally:
                self._chunk_pool.put(buf)
        else:
            self._end_file(self._wf, self._wf_cut)
            if self.sharded:                                   # the other ranks' pieces: written, or the first error
                err = self._pieces_result.get()
                if err is not None and self._wf.err is None:
                    self._wf.err = err
            self._finish(self._wf, scheduled=True)
            self._wf = None

    def _begin_sharded(self, wf, count, total_time, nwalk):
        """rank 0's ingest thread: FILE.tmp with the header (a new file: no other rank writes before every size is in, which
        needs this rank's), this shard's piece, then the kangaroo count after the last piece"""
        try:
            with open(wf.tmp, "wb") as f:
                f.write(work_header(self.dp_bits, self.start, self.end, self.pub, count, total_time))
        except OSError as e:
            wf.err = str(e)
        end = self._write_piece(wf.err)
        if wf.err is None:
            try:
                wf.f = open(wf.tmp, "r+b")
                wf.f.seek(end)
                wf.f.write(struct.pack("<Q", int(nwalk)))
            except OSError as e:
                wf.err = str(e)

    def _write_table(self, wf, count, total_time, nwalk):
        wf.begin(lambda tmp: self.dpt.save(tmp, self.dp_bits, self.start, self.end, self.pub, total_count=count,
                                           total_time=total_time, total_walk=nwalk))

    def _cut(self, kangaroos):
        """every rank, first step of a save: what a file of this cut holds beyond the table and the records (rank 0: passed to
        _end_file with the file's last job)"""
        return None

    def _end_file(self, wf, cut):
        """ingest thread: the file's table and records are written; append what follows them"""

    def _finish(self, wf, scheduled):
        """ingest thread: close a work file -> its error or None.  scheduled: begun by _save_start (not the full table's save)"""
        res = wf.finish()
        self._on_saved(*res)
        self._saved.put(res + (scheduled,))
        return res[3]

    def _on_saved(self, path, mb, seconds, err):
        """ingest thread, right after a save finished (or failed)"""

    def _report_saves(self, block_for=0):
        """rank 0: log the saves finished so far; block_for = saves still to wait for"""
        while block_for > 0 or not self._saved.empty():
            path, mb, secs, err, scheduled = self._saved.get()
            st = []
            if scheduled:                                  # a save _save_start began: its step times
                block_for -= 1
                st = self._save_stats.pop(0) if self._save_stats else []
            if err is not None:
                self.save_error = err
                print("SaveWork %s failed: %s (the previous file is kept)" % (path, err), flush=True)
                continue
            self.saves.append((mb, secs))
            self.last_saved = path
            print("SaveWork %s: %.1f MB in %.2f s, written beside %d steps; longest of them %.1f ms (median step %.1f ms)" %
                  (path, mb, secs, len(st), 1e3 * max(st or [0]), 1e3 * float(np.median(self._step_times[-64:] or [0]))), flush=True)

    # -- rank 0: ingest -------------------------------------------------------------------------------------------
    def _events(self, batch, jumps_before, malformed=0):
        """the table's events for one step's records"""
        if self.table_msg is not None:                  # the run is stopping: later steps' DPs are not inserted
            return []
        try:
            ev = self.dpt.insert(batch)
        except TableFull as e:
            if self.sharded:                            # the stop rule keeps a shard from filling: an error if it does
                self.table_msg, self.table_kind = str(e), "full"
            else:
                self._on_full(str(e), jumps_before)
            return []
        if malformed:
            raise RuntimeError("kgx_dp_partition: %d malformed DP records (h >= 2^18)" % malformed)
        return ev

    def _on_full(self, msg, jumps_before):
        """ingest thread: the table cannot take this step's records.  With --save-work, and no save open, the table is written
        at once as the cut it is: the launches before this one, without kangaroos (their state of that cut is gone)."""
        self.table_msg, self.table_kind = msg, "full"
        if self.save_path and self._wf is None:
            wf = WorkFile(self.save_path, time.perf_counter())
            self._write_table(wf, jumps_before, self.time_offset + time.time() - self.t_start, 0)
            self._end_file(wf, self._cut(kangaroos=False))
            self.full_saved = (self.save_path, jumps_before, self._finish(wf, scheduled=False))

    def _ingest(self, events):
        """rank 0, ingest thread: one step's events -> (hits [(key index, private key, rank, kIdx)], resets).  Resolving stops
        at the first key found."""
        hits, resets = [], []
        for ev in events:
            kind, rk, kidx = ev[:3]
            if kind == EV_COLLISION and not hits:
                m = self._hit(ev)
                if m is None:
                    resets.append((rk, kidx))                                    # "unexpected wrong collision, reset kangaroo"
                else:
                    hits.append(m + (rk, kidx))
            elif kind == EV_RESET:
                resets.append((rk, kidx))
        return hits, resets

    def _claim(self, hits, resets):
        """rank 0: the first hit solves the key; the run stops, so later hits are ignored"""
        if hits and self.found is None:
            self.found = hits[0][1]
            self._announce.append(0)

    def _ingest_loop(self):
        while True:
            job = self._work.get()
            if job is None:
                return
            if job[0] == "dps":
                try:
                    t0 = time.perf_counter()
                    res = self._ingest(self._events(*job[1:]))
                    self.t_ingest += time.perf_counter() - t0
                except Exception as e:                  # the table failed: stop the run (every rank, next step) instead of
                    if self.table_msg is None:          # leaving the main thread waiting for this step's result
                        self.table_msg, self.table_kind = "%s: %s" % (type(e).__name__, e), "error"
                    res = [], []
                if self.sharded:                        # the count first: the main thread's bound may only overestimate
                    self._shard_count = len(self.dps)
                    self._ingested += 1
                self._done.put(res)
            else:
                self._write(job)

    def _submit(self, counts, stride, src, jumps_before, malformed=0):
        """hand one step's records (counts[r] of rank r at src[r*stride*40:], device memory) to the ingest thread.  At most
        one older step may still be in that thread, reading the other staging buffer.  While a save keeps it busy, further
        steps are parked in host RAM instead of waiting: the step loop never waits for the disk, and the backlog takes no GPU
        memory however long the save lasts."""
        park = self._pending >= 2 and self._writes_pending()
        if park:
            self.parked += 1
        while not park and self._pending >= 2:
            self._take()
        if self.sharded:
            self._handed.append(sum(counts))
        self._work.put(("dps", self.dpt.stage(counts, stride, src, park), jumps_before, malformed))
        self._pending += 1

    def _writes_pending(self):
        if self.sharded:                                # an ingest thread waits for the offsets of its piece meanwhile
            return self._saving or self._pieces_open > 0 or (self.rank == 0 and len(self._save_stats) > 0)
        return self._saving or len(self._save_stats) > 0

    def _take(self):
        hits, resets = self._done.get()
        self._pending -= 1
        self._acc_hits += hits
        self._acc_resets += resets

    def _harvest(self, wait_all=False):
        """results of the inserts finished so far -> (hits, resets)"""
        while self._pending and (wait_all or not self._done.empty()):
            self._take()
        res = self._acc_hits, self._acc_resets
        self._acc_hits, self._acc_resets = [], []
        return res

    def _wild_key(self, kidx):
        return self.key

    def _reset_kangaroo(self, kidx):
        """Kangaroo.cpp:601-609: CreateHerd(1, type) + SetKangaroo(kIdx) on the owning engine."""
        v = int(self.rng.integers(0, 1 << 62)) | (int(self.rng.integers(0, 1 << 62)) << 62) | (int(self.rng.integers(0, 1 << 62)) << 124)
        v &= (1 << self.range_power) - 1
        if kidx % 2 == WILD:
            d = (v - self.wdiv2) % ORDER
            pos = ec.add(self._wild_key(kidx), ec.mul(d))
        else:
            d = v
            pos = ec.mul(d)
        if pos is None:
            return
        self.eng.SetKangaroo(kidx, pos[0], pos[1], d)
        self.resets_done += 1

    def _solved(self, solved):
        """every rank: the keys solved this step (every rank follows rank 0's broadcast) -> True when the run is done"""
        return bool(solved)

    def step(self, may_save=True):
        """one Launch on every rank"""
        torch = self.torch
        n_found = self.eng.collect_count(relaunch=True)                  # launch i done, launch i+1 running
        self._gather(n_found)
        solved, resets = [], []
        self._save_work_done = self._save_due or self._saving
        if self._save_due:                                               # decided at the end of the previous step
            self._save_due = False
            self._last_save = time.time()
            self._save_start(self.save_kangaroos, self._chunks_next)     # behind launch i+1's DPs: the cut
        elif self._saving:
            self._save_progress(self._chunks_next)
        if self.sharded:
            hits, resets = self._shard_round()
        if self.rank == 0:
            if not self.sharded:
                hits, resets = self._harvest()
            self._claim(hits, resets)
            self.resets_reported += len(resets)
            self.resets_most = max(self.resets_most, len(resets))
            solved, self._announce = self._announce[:MAX_SOLVED], self._announce[MAX_SOLVED:]
            self.table_stopped = self.table_msg is not None
            self.shard_stop = self.sharded and self.shard_msg is not None
        save_next = (may_save and self.save_interval > 0 and self.rank == 0 and not self._saving and
                     time.time() - self._last_save >= self.save_interval)
        if self.sharded:                                                 # one file at a time: its pieces share FILE.tmp
            save_next = save_next and not self._save_stats
        # herd chunks the next step may move: only into pinned buffers the writer has already freed, so a step never waits for
        # the disk (rank 0 decides, every rank follows)
        chunks = min(SAVE_CHUNKS_PER_STEP, self._chunk_pool.qsize()) if self.rank == 0 else 0
        # control word: table stopped + save flag + chunks + keys solved + kangaroos to re-create, back to their owners.  Resets
        # past MAX_RESETS wait for the next step's broadcast, ahead of that step's own (a kangaroo listed twice meanwhile is
        # re-created twice: harmless)
        if self.dist is not None:
            if self.rank == 0:
                resets = self._reset_backlog + resets
                resets, self._reset_backlog = resets[:MAX_RESETS], resets[MAX_RESETS:]
                c = [2 if self.shard_stop and not self.table_stopped else int(self.table_stopped), len(resets), int(save_next), chunks,
                     len(solved)] + solved + \
                    [v for rk in resets for v in rk]
                self._ctrl[:len(c)].copy_(torch.tensor(c, dtype=torch.int64))
            self.dist.broadcast(self._ctrl, 0)
            c = self._ctrl.cpu().tolist()
            self.table_stopped, save_next, chunks, ns = c[0] == 1, bool(c[2]), c[3], c[4]
            self.shard_stop = c[0] == 2
            solved = c[5:5 + ns]
            resets = [(c[5 + ns + 2 * i], c[6 + ns + 2 * i]) for i in range(c[1])]
        self.stop = self._solved(solved) or self.table_stopped or self.shard_stop   # (--batch-keys: retargets, before the resets)
        self._chunks_next = chunks
        if save_next and not self.stop:
            if self.save_kangaroos:
                self.eng.SnapshotBegin()                                 # stream order: after launch i+1, before the resets below
            self._save_due = True
        for rk, kidx in resets:
            self.same_herd += 1
            if rk == self.rank and not self.stop:
                self._reset_kangaroo(kidx)

    def _gather(self, n_found):
        """this launch's DP records of every rank -> rank 0's ingest thread"""
        cnt = min(n_found, self.eng.maxFound)
        jumps_before = self.jumps
        self.jumps += self.eng.nbKangaroo * NB_RUN * self.world
        res = None
        if self.sharded:
            counts, cap, recv, bad = self.exchange.step(cnt)                # every rank: the records of its buckets
            self._submit(counts, cap, recv, jumps_before, bad)
        elif self.gather is not None:
            res = self.gather.step_flat(cnt)                             # rank 0: (counts, cap, device tensor [world*cap*40])
        elif cnt:
            ptr = self.eng.convert_dps_device_ptr()
            res = [cnt], cnt, self.torch.as_tensor(SlabView(ptr + 4, cnt * DP40_BYTES), device="cuda")
        if res is not None:
            self._submit(*res, jumps_before)

    def run(self, max_steps=1 << 30, verbose=True):
        self.eng.callKernel()
        t0 = time.time()
        self.t_start = self._last_save = t0
        steps = 0
        self.steady = None                      # (time, jumps) after the first 32 steps: NCCL communicator set-up, first table growth
        self._step_times = step_times = []
        for s in range(max_steps):
            ts = time.perf_counter()
            self.step(may_save=s + 1 < max_steps)
            step_times.append(time.perf_counter() - ts)
            if self._save_work_done:
                self._save_steps.append(step_times[-1])
            steps += 1
            if self.rank == 0:
                self._report_saves()
            if steps == 32:
                self.steady = (time.time(), self.jumps)
            if verbose and self.rank == 0 and (s % 64 == 63 or self.stop):
                dt = time.time() - t0
                print("[%6.1fs] 2^%.2f jumps  %.0f MJump/s  %d DPs  dead %d  %s %.1f ms/step" %
                      (dt, np.log2(max(self.jumps, 1)), (self.jumps - self.jumps0) / dt / 1e6, self.table_entries(), self.same_herd,
                       self.dpt.label, 1e3 * self.t_ingest / steps), flush=True)
            if self.stop:
                break
        if self.sharded:                                        # a save in progress: finish it first
            self._shard_drain()
        elif self._saving:                                      # a save still moving its herd: finish it first
            self._save_progress(len(self._save_left))
        if self.save_path and not self.table_stopped:
            # end-of-run cut: the launch still in flight is collected, its DPs go into the table before it is written
            if self.save_kangaroos:
                self.eng.SnapshotBegin()
            self._gather(self.eng.collect_count(relaunch=False))
        else:
            self.eng.sync()
        t1 = time.time()
        if self.save_path and not self.table_stopped:           # (sharded: the drain below moves the herd chunks)
            self._save_start(self.save_kangaroos, len(self.herd.plan) if self.save_kangaroos and not self.sharded else 0)
        if self.sharded:
            self._shard_drain()
        if self.rank == 0:                                      # drain: the last steps' records may still be in the ingest thread
            self._claim(*self._harvest(wait_all=True))
            self._report_saves(block_for=len(self._save_stats))
        self.recreated = self.resets_done
        if self.dist is not None:                               # the kangaroos every rank re-created, for rank 0's report
            t = self.torch.tensor([self.resets_done], dtype=self.torch.int64, device="cuda")
            self.dist.all_reduce(t)
            self.recreated = int(t.item())
        self.elapsed = t1 - t0
        self.steps = steps
        self.steady_rate = ((self.jumps - self.steady[1]) / (t1 - self.steady[0]) if self.steady and steps > 64
                            else (self.jumps - self.jumps0) / self.elapsed)
        return self.found

    def close(self):
        if self._thread is not None:
            self._harvest(wait_all=True)
            self._work.put(None)
            self._thread.join(timeout=10)
            self._thread = None
        self.eng.close()
        if self.dpt is not None:
            self.dpt.close()


# -- --batch-keys: every key of the input in one run, one tame herd shared by all of them -------------------------------------
# The reference solves the keys of an input one after another, each with a new herd and an empty table (Kangaroo::Run,
# Kangaroo.cpp:1021-1066).  Tame trails (d*G) and their DPs do not depend on the key, so here one engine, one herd and one
# table serve them all: the wild half of the herd is spread over the unsolved keys, and when a key is solved its wilds move
# on to the others (kgx_retarget), keeping their distance.  Rank 0 finds the key of a tame/wild collision with
# kgi_resolve_multi, since the stored entry carries no kIdx.
def spread(kidx, live):
    """The key of wild kangaroo kIdx among the live keys (in input order): live[(kIdx >> 1) % len(live)].  The herd's first
    assignment and kgx_retarget both follow it, so the wilds of every rank are spread evenly over the live keys."""
    kidx = np.asarray(kidx, dtype=np.int64)
    return np.asarray(live, dtype=np.uint16)[(kidx >> 1) % len(live)]


def assign_targets(n, live):
    """targets of a new multi-key herd of n kangaroos: the wild ones (odd kIdx) spread over the live keys, the tame ones 0"""
    t = np.zeros(n, dtype=np.uint16)
    wild = np.arange(WILD, n, 2)
    t[wild] = spread(wild, live)
    return t


def retarget_targets(targets, frm, live):
    """the host mirror of kgx_retarget(frm, live): the wilds of key frm move to spread(kIdx, live)"""
    kidx = np.arange(targets.size)
    moved = (kidx % 2 == WILD) & (targets == frm)
    out = targets.copy()
    out[moved] = spread(kidx[moved], live)
    return out


def key_classes(keys):
    """Keys that are the same point, or each other's negative, share one search: -> (rep, neg) with rep[i] the first key of
    i's class in input order and neg[i] true when keys[i] == -keys[rep[i]].  None (the point at infinity) is its own class."""
    rep, neg, first = list(range(len(keys))), [False] * len(keys), {}
    for i, k in enumerate(keys):
        if k is None:
            continue
        j = first.setdefault(k[0], i)                   # same x: the same point or its negative
        if j != i:
            rep[i], neg[i] = j, k[1] != keys[j][1]
    return rep, neg


def class_members(rep):
    """the keys of every class, from key_classes' rep -> {first key of the class: [its keys in input order]}; built once, so
    that claiming a class visits its own keys and not every key of the input"""
    members = {}
    for i, r in enumerate(rep):
        members.setdefault(r, []).append(i)
    return members


def class_privs(start, priv_rep, neg):
    """the private key of a key of the class solved with priv_rep: keyToSearch = priv - start*G, so the negative of a key
    has priv 2*start - priv_rep"""
    return (2 * start - priv_rep) % ORDER if neg else priv_rep


# Batch work files (--batch-save / --batch-resume): the single-key file of the cut (table, kangaroo records; header key = input
# key 0, wild distances relative to each wild's own target) followed by the batch block (kgx_workfile.h: the keys, their solved
# flags and private keys, every kangaroo's target).  The order that keeps a cut consistent: the keys rank 0 announces solved
# at step k are retargeted on every rank at step k, before the snapshot a save decided at step k takes, and a save's solved
# flags are the keys announced up to the step that took its snapshot.  So a file shows a key solved exactly when the wilds of
# it were moved on before the snapshot; a key found but not yet announced is written unsolved, with its wilds still on it.
class BatchSolver(Solver):
    """--batch-keys.  pubs: every public key of the input.  After run(), rank 0 holds priv[i] (None: not found).
    save_work / save_interval: --batch-save / --batch-save-interval; resume: --batch-resume FILE with resume_block its batch
    block (worktool.BatchBlock, from batch_resume_file: the targets on rank 0 only)."""

    def __init__(self, start, end, pubs, dp_bits, grid=None, max_found=1 << 17, seed=None, ingest_threads=0, dp_table="host",
                 dp_table_capacity=None, save_work="", save_interval=0.0, resume=None, resume_block=None, dp_table_entries="device"):
        self.pubs = list(pubs)
        if not 1 <= len(self.pubs) <= MAX_KEYS:
            raise ValueError("--batch-keys takes 1 to %d keys, not %d" % (MAX_KEYS, len(self.pubs)))
        # Kangaroo::InitSearchKey per key; pub == start*G leaves the point at infinity: solved at start, priv = start
        self.keys = [ec.add(p, ec.neg(ec.mul(start))) if start else p for p in self.pubs]
        self.priv = [start if k is None else None for k in self.keys]
        # a key listed twice, or the negative of another, is searched once, as the first of its class: kgi_resolve_multi
        # reports the first matching key, so the later ones would never be hit
        self.rep, self.neg = key_classes(self.keys)
        self.members = class_members(self.rep)
        self.announced = set()              # every rank: classes (their first key) announced solved, those of the file included
        self._resume_block = resume_block
        if resume_block is not None:
            for i, done in enumerate(resume_block.solved):
                if done:
                    self.priv[i] = resume_block.privs[i]
                    self.announced.add(self.rep[i])
        self.live = [i for i, k in enumerate(self.keys) if k is not None and self.rep[i] == i and i not in self.announced]
        super().__init__(start, end, self.pubs[0], dp_bits, grid, max_found, seed, ingest_threads, dp_table=dp_table,
                         dp_table_capacity=dp_table_capacity, dp_table_entries=dp_table_entries, save_work=save_work,
                         save_interval=save_interval, save_kangaroos=bool(save_work), resume=resume)

    def _resume(self, path):
        """Solver._resume with the targets: rank 0 loads the table and sends every rank its records and their targets; each
        rank imports its slice verified against each record's own target key.  The wilds of keys the file shows solved then
        move on to the live keys (the spread rule, as a retarget would have moved them); kangaroos the file lacks keep the
        fresh herd spread over the live keys."""
        torch = self.torch
        info = torch.zeros(4, dtype=torch.int64, device="cuda")
        w = self._load_table(path)
        if self.rank == 0:
            info.copy_(torch.tensor([w.nb_walk, w.walk_offset, w.total_count, 0], dtype=torch.int64))
            self.time_offset = w.total_time
        if self.dist is not None:
            self.dist.broadcast(info, 0)
        nb_walk, offset, count, _ = (int(v) for v in info.cpu().tolist())
        self.jumps = count
        off = self.herd.offsets[self.rank]
        take = max(0, min(self.eng.nbKangaroo, nb_walk - off))
        if self.rank == 0:
            tg = self._resume_block.targets
            print("Resume %s: %d DPs, count 2^%.2f, %d kangaroos in the file for %d in the herd, %d of %d keys solved in the file, "
                  "%d keys left to search" % (path, self.table_entries(), np.log2(max(count, 1)), nb_walk, self.herd.total,
                                              sum(self._resume_block.solved), len(self.keys), len(self.live)), flush=True)
            if nb_walk > self.herd.total:
                print("Warning: %d unhandled kangaroos" % (nb_walk - self.herd.total), flush=True)
        if self.dist is not None:                               # the targets, as bytes (NCCL has no 16-bit integers)
            t = torch.zeros(2 * max(nb_walk, 1), dtype=torch.uint8, device="cuda")
            if self.rank == 0 and nb_walk:
                t[:2 * nb_walk].copy_(torch.from_numpy(tg.view(np.uint8)))
            self.dist.broadcast(t, 0)
            tg = t.cpu().numpy().view(np.uint16)
        mine = np.ascontiguousarray(tg[off:off + take])

        def read(first, cnt):                                   # rank 0 only
            return np.fromfile(path, dtype=np.uint8, count=cnt * WALK_BYTES, offset=offset + first * WALK_BYTES)

        t0 = time.perf_counter()
        recs = self.herd.scatter(nb_walk, read)
        bad = self.eng.ImportKangaroosMulti(recs, [k or (0, 0) for k in self.keys], mine, verify=True) if take else 0
        if self.dist is not None:
            t = torch.tensor([bad], dtype=torch.int64, device="cuda")
            self.dist.all_reduce(t)
            bad = int(t.item())
        if bad:
            raise RuntimeError("%s: %d kangaroos are not at d*G (tame) / key[target] + d*G (wild): the file belongs to other keys "
                               "or another range" % (path, bad))
        self.targets[:take] = mine
        if self.live:
            wild = self.targets[WILD::2]
            for idx in sorted(set(np.unique(wild).tolist()) - set(self.live)):
                self.eng.Retarget(idx, self.live)
                self.targets = retarget_targets(self.targets, idx, self.live)
        if take:
            print("rank %d: %d kangaroos imported and verified in %.2f s" % (self.rank, take, time.perf_counter() - t0), flush=True)

    def _cut(self, kangaroos):
        """every rank: the snapshot's targets, gathered to rank 0 in rank order -> rank 0: the batch block of the cut"""
        targets = np.zeros(0, dtype=np.uint16)
        if kangaroos:
            targets = self.eng.SnapshotExportTargets(0, self.eng.nbKangaroo)
            if self.dist is not None:                            # as bytes, padded to the largest herd
                torch, width = self.torch, 2 * max(self.herd.sizes)
                t = torch.zeros(width, dtype=torch.uint8, device="cuda")
                t[:2 * targets.size].copy_(torch.from_numpy(targets.view(np.uint8)))
                bufs = [torch.empty(width, dtype=torch.uint8, device="cuda") for _ in range(self.world)] if self.rank == 0 else None
                self.dist.gather(t, bufs, dst=0)
                if self.rank == 0:
                    targets = np.concatenate([b.cpu().numpy().view(np.uint16)[:n] for b, n in zip(bufs, self.herd.sizes)])
        if self.rank != 0:
            return None
        from .worktool import BatchBlock
        solved = [p is not None and (k is None or self.rep[i] in self.announced) for i, (k, p) in enumerate(zip(self.keys, self.priv))]
        return BatchBlock(self.pubs, solved, [p if done else None for p, done in zip(self.priv, solved)], targets)

    def _end_file(self, wf, cut):
        if cut is None or wf.f is None or wf.err is not None:
            return
        from .worktool import batch_block
        try:
            wf.append(memoryview(batch_block(cut, wf.f.tell())))
        except (OSError, ValueError) as e:
            wf.err = str(e)

    def _create_herd(self, sc, d128):
        self.targets = assign_targets(self.eng.nbKangaroo, self.live or [0])         # host mirror of the engine's targets
        self.eng.CreateHerdMulti(sc, d128, [k or (0, 0) for k in self.keys], self.targets)

    def _wild_key(self, kidx):
        return self.keys[int(self.targets[kidx])]

    def _key_table(self):
        return DPTable.key_table(self.keys)

    def _hit(self, ev):
        return ev[5] if len(ev) > 5 else self.dps.resolve_multi(ev[3], ev[4], self.key_table, self.start)

    def _ingest(self, events):
        """rank 0, ingest thread -> (hits [(key index, private key, rank, kIdx)], resets): every collision is resolved"""
        hits, resets = [], []
        for ev in events:
            kind, rk, kidx = ev[:3]
            if kind == EV_COLLISION:
                m = self._hit(ev)
                if m is None:
                    resets.append((rk, kidx))                    # matches no key: "unexpected wrong collision, reset kangaroo"
                else:
                    hits.append(m + (rk, kidx))
            elif kind == EV_RESET:
                resets.append((rk, kidx))                        # same herd, wild/wild across keys included
        return hits, resets

    def _claim(self, hits, resets):
        """rank 0: a hit on an unsolved key solves it.  A hit on a solved key resets the kangaroo that made it: a tame one that
        ran onto the abandoned trail of a moved wild would re-walk it, or a wild DP from before its move."""
        for idx, priv, rk, kidx in hits:
            r = self.rep[idx]
            if self.priv[r] is None:
                self.priv[r] = class_privs(self.start, priv, self.neg[idx])
                for i in self.members[r]:                       # the other keys of its class
                    self.priv[i] = class_privs(self.start, self.priv[r], self.neg[i])
                self._announce.append(r)
            else:
                resets.append((rk, kidx))

    def _solved(self, solved):
        """every rank moves the wilds of each solved key to the live ones (a reset kangaroo starts at its current key)"""
        for idx in solved:
            self.announced.add(idx)
            self.live.remove(idx)
            if self.live:
                self.eng.Retarget(idx, self.live)                        # stream order: after launch i+1, before the resets
                self.targets = retarget_targets(self.targets, idx, self.live)
        return not self.live

    def run(self, max_steps=1 << 30, verbose=True):
        if not self.live:                                                # every key solved at start
            self.elapsed, self.steps, self.steady_rate = 1e-9, 0, 0.0
            return None
        return super().run(max_steps, verbose)


def _run_batch(start, end, pubs, dp, grid, a, block=None):
    t0 = time.perf_counter()
    s = BatchSolver(start, end, pubs, dp, grid, seed=a.seed, ingest_threads=a.ingest_threads, dp_table=a.dp_table,
                    dp_table_capacity=a.dp_table_capacity, save_work=a.batch_save, save_interval=a.batch_save_interval,
                    resume=a.batch_resume or None, resume_block=block, dp_table_entries=a.dp_table_entries)
    t_setup = time.perf_counter() - t0
    if s.rank == 0:
        print("Range width: 2^%d  kangaroos/GPU: %d  GPUs: %d  dp: %d  %s  keys: %d in one run" %
              (s.range_power, s.eng.nbKangaroo, s.world, dp, s.dpt.info, len(pubs)), flush=True)
    t0 = time.perf_counter()
    s.run(a.max_steps)
    t_run = time.perf_counter() - t0
    t0 = time.perf_counter()
    rc = 0
    if s.rank == 0:
        rc = report(s, a)
        solved = sum([print_key(i, pub, s.priv[i]) for i, pub in enumerate(pubs)])
        rc |= solved < len(pubs)
        print("Batch: %d/%d keys solved, %d jumps (2^%.2f) in total, %.3f sqrt(N) jumps per key (N = 2^%d), %d DPs" %
              (solved, len(pubs), s.jumps, np.log2(max(s.jumps, 1)), s.jumps / len(pubs) / 2.0 ** (s.range_power / 2),
               s.range_power, s.table_entries()), flush=True)
    t_results = time.perf_counter() - t0
    t0 = time.perf_counter()
    s.close()
    if s.rank == 0:
        # where the time outside the jump loop goes: the loop ends when the last key is found, the DP records still queued
        # are then inserted, and closing frees the engine and every entry of the table
        print("Batch time: set-up %.2f s (engine, herd, table), jump loop %.2f s, after the loop %.2f s (last DPs into the table), "
              "results %.2f s, close %.2f s (engine and table freed)" %
              (t_setup, s.elapsed, t_run - s.elapsed, t_results, time.perf_counter() - t0), flush=True)
    return rc


def report(s, a):
    """rank 0, after the run: the rate line, then why the table stopped the run or where the work file went -> 1 when the
    table stopped the run or the work file was not written, else 0"""
    print("Solver rate: %.0f MJump/s steady state (after the first 32 steps), %.0f MJump/s over all %d steps (%.2f s); "
          "rank-0 %s %.2f ms/step; %d DPs; %d dead kangaroos re-created (%d reported by the table, at most %d in one step)" %
          (s.steady_rate / 1e6, (s.jumps - s.jumps0) / s.elapsed / 1e6, s.steps, s.elapsed, s.dpt.label,
           1e3 * s.t_ingest / max(s.steps, 1), s.table_entries(), s.recreated, s.resets_reported, s.resets_most))
    if s.sharded:
        print("Hits resolved per shard: %s" % " ".join(str(v) for v in s.shard_hits))
    if s.shard_stop and not s.table_stopped:
        print("DP table shard full%s, run stopped: %s.  Resume the work file with a larger --dp-table-capacity, on more GPUs or "
              "with --dp-table host" % (layout_note(s.entries), s.shard_msg))
    if s.table_stopped:
        print(table_message(s, a))
        return 1
    if s.save_path and s.save_error is None:
        mb, dt_save = s.saves[-1]
        print("work file written: %s (%.1f MB in %.2f s, count 2^%.2f)" % (s.save_path, mb, dt_save, np.log2(max(s.jumps, 1))))
    elif s.save_path:
        print("work file NOT written: %s: %s" % (s.save_path, s.save_error))
        return 1
    return 0


def print_key(i, pub, priv):
    """rank 0: key i's result line -> whether priv is pub's private key"""
    if priv is not None and ec.mul(priv) == pub:
        print("Key#%2d Pub:  0x%064X\n       Priv: 0x%X" % (i, pub[0], priv))
        return True
    print("Key#%2d not found" % i)
    return False


def table_message(s, a):
    """rank 0, after the run: why the table stopped it, and which work file, if any, to resume"""
    what = "full" if s.table_kind == "full" else "failed"
    msg = "DP table %s%s, run stopped: %s." % (what, layout_note(s.entries), s.table_msg)
    saved = s.full_saved
    if saved and saved[2] is None:
        msg += (" %s holds the table as it was before this step's launch (count 2^%.2f, no kangaroos); resume it with "
                "--dp-table host or a larger --dp-table-capacity" % (saved[0], np.log2(max(saved[1], 1))))
    elif s.last_saved:
        msg += (" The last work file written, %s, is a consistent cut from before the table stopped; resume it with "
                "--dp-table host or a larger --dp-table-capacity" % s.last_saved)
    elif s.save_path:
        msg += " No work file was written."
    elif what == "full":
        msg += " Use --dp-table host or a larger --dp-table-capacity (with --save-work, the run writes a resumable file first)."
    return msg


def _resume_header(path):
    """the work file's header, read on rank 0 only and broadcast: the other ranks need not see the file"""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    hdr = None
    if int(os.environ.get("RANK", "0")) == 0:
        from .ingest import read_work_header
        h = read_work_header(path)
        hdr = (h.dp_bits, h.range_start, h.range_end, h.key)
    if world > 1:
        dist = init_dist()
        box = [hdr]
        dist.broadcast_object_list(box, 0)
        hdr = box[0]
    return hdr


def batch_resume_file(path):
    """--batch-resume: rank 0 reads the file's header and batch block and sends every rank (dp, start, end, block) with the
    block's targets left on rank 0, or the reason the file cannot be resumed (a string)"""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    res = None
    if int(os.environ.get("RANK", "0")) == 0:
        from .ingest import read_work_header
        from .worktool import read_batch
        try:
            h = read_work_header(path)
            block = read_batch(path)
            if block is None:
                res = ("%s is a plain HEADW work file (no batch block): resume it with --resume, without --batch-keys" % path)
            else:
                res = (h.dp_bits, h.range_start, h.range_end, block)
        except (OSError, RuntimeError, ValueError) as e:
            res = "cannot resume %s: %s" % (path, e)
    if world > 1:
        from .worktool import BatchBlock
        dist = init_dist()
        box = [res if isinstance(res, str) or res is None else
               res[:3] + (BatchBlock(res[3].pubs, res[3].solved, res[3].privs, np.zeros(0, np.uint16), res[3].offset),)]
        dist.broadcast_object_list(box, 0)
        if int(os.environ.get("RANK", "0")) != 0:
            res = box[0]
    return res


def config_difference(start, end, pubs, f_start, f_end, f_pubs):
    """the first difference between a config (range, keys in order) and a batch work file's, or None"""
    if start != f_start:
        return "the config's range start 0x%X is not the file's 0x%X" % (start, f_start)
    if end != f_end:
        return "the config's range end 0x%X is not the file's 0x%X" % (end, f_end)
    for i, (p, q) in enumerate(zip(pubs, f_pubs)):
        if p != q:
            return "key #%d differs: the config has 04%064X%064X, the file 04%064X%064X" % (i, p[0], p[1], q[0], q[1])
    if len(pubs) != len(f_pubs):
        return "the config lists %d keys, the file %d" % (len(pubs), len(f_pubs))
    return None


def parse_args(argv=None):
    """the command line -> (arguments, range start, range end, public keys, dp bits, grid, batch block or None); argparse
    exits on a usage error.  Loads build/libkgx_ingest.so only for --dp-table host, to refuse the run when it is missing."""
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", help="range start, end and public keys (optional with --resume)")
    ap.add_argument("--dp", type=int, default=None, help="distinguished-point bits (default 12, or the file's with --resume)")
    ap.add_argument("--grid", default="")
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("--max-steps", type=int, default=1 << 30)
    ap.add_argument("--ingest-threads", type=int, default=0, help="workers of the rank-0 DP table (0 = min(8, cores))")
    ap.add_argument("--save-work", default="", help="write the DP table as a reference work file (HEADW) at the end (-w)")
    ap.add_argument("--save-interval", type=float, default=0.0,
                    help="also save every SECONDS while running (-wi); 0 = at the end only")
    ap.add_argument("--save-kangaroos", action="store_true", help="save every rank's herd with the table (-ws)")
    ap.add_argument("--resume", default="", metavar="FILE",
                    help="continue from a work file (-i): range, key and dp come from the file unless given")
    ap.add_argument("--dp-table", choices=("host", "device", "sharded"), default="host",
                    help="where the DP table is kept: host = the reference's HashTable in rank 0's host RAM, inserted by "
                         "--ingest-threads workers (build/libkgx_ingest.so, built only with the reference sources); device = a hash table with the same results in rank 0's GPU memory, inserted "
                         "by CUDA kernels straight from the gathered records (fixed capacity: a full table stops the run); "
                         "sharded = the device table split by bucket over every rank's GPU, each rank inserting the records of its "
                         "buckets (a full shard stops the run with the normal end-of-run work file; every rank writes its piece of "
                         "a work file into FILE.tmp itself, so FILE's directory must be one file system for all ranks)")
    ap.add_argument("--dp-table-capacity", type=int, default=None, metavar="ENTRIES",
                    help="--dp-table device: entries the table holds, 48 bytes of GPU memory each (default: what fits in rank "
                         "0's free GPU memory after the engine, less %d GiB); --dp-table sharded: entries of each GPU's shard "
                         "(default: the same rule on each GPU)" % (DP_TABLE_MARGIN >> 30))
    ap.add_argument("--dp-table-entries", choices=("device", "host"), default=None,
                    help="--dp-table device or sharded: where the table's 32-byte entries live.  device (default) = GPU "
                         "memory, 48 bytes per entry in all; host = pinned host RAM mapped into the GPU, which then holds 16 bytes "
                         "per entry (the index), for about 2.6x the entries per GPU.  The default capacity with host is also at "
                         "most 2^32-2 and the host RAM available (MemAvailable) less %d GiB, at 32 bytes per entry, shared by "
                         "the tables of this host; a larger --dp-table-capacity is refused" % (HOST_ENTRIES_MARGIN >> 30))
    ap.add_argument("--batch-keys", action="store_true",
                    help="solve every key of the config in one run: one tame herd and one DP table shared by all keys, the "
                         "wild kangaroos spread over the unsolved ones")
    ap.add_argument("--batch-save", default="", metavar="FILE",
                    help="--batch-keys only: write a batch work file (a HEADW work file with every rank's herd, then every key, "
                         "its solved flag and every kangaroo's target key) at the end, and with --batch-save-interval while running")
    ap.add_argument("--batch-save-interval", type=float, default=0.0, metavar="SECS",
                    help="also save every SECS seconds (0 = at the end only)")
    ap.add_argument("--batch-resume", default="", metavar="FILE",
                    help="--batch-keys only: continue a batch run from FILE; the keys, range and dp come from the file (a config, "
                         "if given, must list the same range and keys in the same order)")
    a = ap.parse_args(argv)
    if a.batch_keys and (a.resume or a.save_work or a.save_interval or a.save_kangaroos):
        ap.error("--batch-keys cannot be combined with --save-work, --save-interval, --save-kangaroos or --resume "
                 "(a work file carries one key)")
    if (a.batch_save or a.batch_save_interval or a.batch_resume) and not a.batch_keys:
        ap.error("--batch-save, --batch-save-interval and --batch-resume need --batch-keys")
    if a.batch_save_interval and not a.batch_save:
        ap.error("--batch-save-interval needs --batch-save FILE")
    if a.batch_keys and not a.config and not a.batch_resume:
        ap.error("--batch-keys needs a config file")
    if a.dp_table_capacity is not None and a.dp_table not in ("device", "sharded"):
        ap.error("--dp-table-capacity needs --dp-table device or sharded")
    if a.dp_table_capacity is not None and not 0 < a.dp_table_capacity < (1 << 32) - 1:
        ap.error("--dp-table-capacity must be 1 .. 2^32-2 entries, not %d" % a.dp_table_capacity)
    if a.dp_table == "sharded" and sharded_capacity_error(a.dp_table_capacity, int(os.environ.get("WORLD_SIZE", "1"))):
        ap.error(sharded_capacity_error(a.dp_table_capacity, int(os.environ.get("WORLD_SIZE", "1"))))
    if a.dp_table_entries is not None and a.dp_table not in ("device", "sharded"):
        ap.error("--dp-table-entries needs --dp-table device or sharded (--dp-table host keeps the reference's table in host RAM)")
    a.dp_table_entries = a.dp_table_entries or "device"
    if a.dp_table_entries == "host" and host_capacity_error(a.dp_table_capacity, mem_available(), tables_on_node(a.dp_table)):
        ap.error(host_capacity_error(a.dp_table_capacity, mem_available(), tables_on_node(a.dp_table)))
    block = None
    if a.batch_resume:
        res = batch_resume_file(a.batch_resume)
        if isinstance(res, str):
            ap.error("--batch-resume: " + res)
        file_dp, start, end, block = res
        pubs = block.pubs
        if a.config:
            diff = config_difference(*ec.parse_config(a.config), start, end, pubs)
            if diff:
                ap.error("--batch-resume: the config does not match %s: %s" % (a.batch_resume, diff))
        dp = a.dp if a.dp is not None else file_dp
    elif a.resume:
        file_dp, start, end, pub = _resume_header(a.resume)
        pubs = [pub]
        if a.config:
            start, end, pubs = ec.parse_config(a.config)
        dp = a.dp if a.dp is not None else file_dp
    elif a.config:
        start, end, pubs = ec.parse_config(a.config)
        dp = a.dp if a.dp is not None else 12
    else:
        ap.error("a config file or --resume FILE is required")
    if (a.save_interval > 0 or a.save_kangaroos) and not a.save_work:
        ap.error("--save-interval and --save-kangaroos need --save-work FILE")
    if a.batch_keys and not pubs:
        ap.error("--batch-keys needs a config with at least one public key")
    if a.batch_keys and len(pubs) > MAX_KEYS:
        ap.error("--batch-keys takes at most %d keys, the config has %d" % (MAX_KEYS, len(pubs)))
    if a.dp_table == "host":
        from . import ingest
        try:
            ingest.load_library()
        except RuntimeError as e:
            ap.error(str(e))
    grid = tuple(int(v) for v in a.grid.split(",")) if a.grid else None
    return a, start, end, pubs, dp, grid, block


def main(argv=None):
    a, start, end, pubs, dp, grid, block = parse_args(argv)
    rc = _run_batch(start, end, pubs, dp, grid, a, block) if a.batch_keys else 0
    for i, pub in enumerate([] if a.batch_keys else pubs):
        s = Solver(start, end, pub, dp, grid, seed=a.seed, ingest_threads=a.ingest_threads, save_work=a.save_work,
                   save_interval=a.save_interval, save_kangaroos=a.save_kangaroos, resume=a.resume or None, dp_table=a.dp_table,
                   dp_table_capacity=a.dp_table_capacity, dp_table_entries=a.dp_table_entries)
        if s.rank == 0:
            print("Range width: 2^%d  kangaroos/GPU: %d  GPUs: %d  dp: %d  %s" %
                  (s.range_power, s.eng.nbKangaroo, s.world, dp, s.dpt.info), flush=True)
        key = s.run(a.max_steps)
        if s.rank == 0:
            rc |= report(s, a)
            rc |= not print_key(i, pub, key)
        s.close()
    try:
        import torch.distributed as dist
        if dist.is_initialized():
            dist.destroy_process_group()
    except Exception:
        pass
    return rc


if __name__ == "__main__":
    sys.exit(main())
