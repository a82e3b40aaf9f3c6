"""python -m kangaroo_b200.server: the DP server of the reference's client/server mode (Network.cpp, protocol version 3), with
every received DP checked on the GPU before it is kept.

Unmodified reference clients (`kangaroo -c SERVER`) and the drop-in build/kangaroo_b200 connect to it as to `kangaroo -s`.
The server holds the one DP table of the search in GPU memory (ingest.DeviceDPTable), resolves its collisions there
(ingest.DeviceResolver) and writes the work files the solver, worktool and the reference read.

Threads:
  acceptor     accepts connections and starts a handler for each
  handlers     one per connection: the protocol.  A SENDDP message is read whole, in host chunks of at most 2^20 records,
               answered with the status, then queued with its connection; the queue has a byte budget and a handler blocks
               while it is full.  Records are never touched one by one in Python.
  ingest       owns the GPUs (GpuSink): per batch of up to 2^20 queued records, one copy to a GPU,
               kgx_resolver_verify_partition (the check of every record against the key, and the good ones grouped by the
               shard that owns their bucket, in input order), the counts back, then DeviceDPTable.add of each group with the
               resolver, on the shard's stream.  Saves are queued like records, so a work file holds the table after every
               record queued before it.
  main         the status line, periodic saves, signals and the end of the run.

The table is one shard per --devices entry (--device D, the default, is the one entry D), in the buckets the solver's
--dp-table sharded gives its ranks; one shard holds every bucket.  The work files are byte for byte those of one table
whatever the shards.

The protocol layer (Server) talks to its sink through three calls -- put(message, chunks), status(), reset_dead() -- so that
a test can run it with a fake sink in place of the GPU path.
"""
import argparse
import collections
import errno
import os
import signal
import socket
import struct
import sys
import threading
import time

import numpy as np

from . import ecmath as ec

PROTOCOL_VERSION = 3
DP_MAGIC = 0x67DEDDC1           # SERVER_HEADER: the first word of a SENDDP header
HEADKS = 0xFA6A8003             # a kangaroo file of the reference's -wss
KANG_PER_BLOCK = 2048           # kangaroos per block of SAVEKANG / LOADKANG
CMD_GETCONFIG, CMD_STATUS, CMD_SENDDP, CMD_SETKNB, CMD_SAVEKANG, CMD_LOADKANG, CMD_RESETDEAD = 0, 1, 2, 3, 4, 5, ord("R")
STATUS_OK, STATUS_END, STATUS_BACKUP = 0, 1, 2
DEFAULT_PORT = 17403
CMD_TIMEOUT = 3.0               # seconds a command's body has to arrive (the reference's -nt default)
CLIENT_TIMEOUT = 3600.0         # a connection that sends no command for this long is closed
CHUNK_RECORDS = 1 << 20         # records per host chunk of a message, and per ingest batch
QUEUE_BYTES = 512 << 20         # the record queue's budget
END_GRACE = 10.0                # seconds the server waits for clients to leave once the key is found
STATUS_PERIOD = 5.0             # seconds between status lines
DP40 = 40
EVENT_BYTES = 136               # device scratch per event slot of an add (kgx_dptable_reserve)
MAX_SHARDS = 256                # KGX_DPT_MAX_RANKS: the shards of one table


class ClientGone(Exception):
    """the connection ended, timed out or broke the protocol"""


def recv_into(sock, view):
    """fill the memoryview from the socket (its timeout applies to each receive) or raise ClientGone"""
    got = 0
    while got < len(view):
        try:
            k = sock.recv_into(view[got:])
        except (socket.timeout, OSError) as e:
            raise ClientGone(str(e) or "timeout")
        if k == 0:
            raise ClientGone("connection closed")
        got += k


def recv_exact(sock, n):
    buf = bytearray(n)
    recv_into(sock, memoryview(buf))
    return bytes(buf)


def file_name_error(name):
    """why a kangaroo file name sent by a client is refused, or None: only one path component of the working directory"""
    if not name:
        return "empty name"
    if len(name) >= 256:
        return "name of %d bytes (at most 255)" % len(name)
    for c in (b"/", b"\\", b"\0"):
        if c in name:
            return "name holds %r" % c.decode()
    if name in (b".", b".."):
        return "name %r" % name.decode()
    return None


def kang_checksum(raw):
    """the sum of 16-byte little-endian values (a multiple of 16 bytes) as an int"""
    w = np.frombuffer(raw, dtype=np.uint32).reshape(-1, 4).sum(axis=0, dtype=np.uint64)   # < 2^32 values: no overflow
    return sum(int(v) << (32 * k) for k, v in enumerate(w))


class Client:
    """one connection: its address, the kangaroo count it announced (SETKNB) and the wrong records it sent"""

    def __init__(self, sock, addr):
        self.sock, self.addr = sock, addr
        self.name = "%s:%d" % (addr[0], addr[1])
        self.knb = 0
        self.wrong = 0


class Message:
    """one SENDDP message: where it came from and, once checked, how many of its records were wrong"""

    def __init__(self, client, n, thread_id, process_id, gpu_id):
        self.client, self.n = client, n
        self.thread_id, self.process_id, self.gpu_id = thread_id, process_id, gpu_id
        self.bad = 0

    def wrong_line(self):
        return ("%d wrong DPs of %d from %s (processId %d, threadId %d, gpuId %d): dropped" %
                (self.bad, self.n, self.client.name, self.process_id, self.thread_id, self.gpu_id))


class Server:
    """The protocol: listens on (bind, port) and serves every connection on a thread of its own.  start, end, key (x, y) and
    dp are what GETCONFIG sends; sink takes the records (put), gives the status (status) and zeroes the dead count
    (reset_dead).  Kangaroo files of SAVEKANG / LOADKANG live in workdir; a name that is a symbolic link, or that names one of
    the `protected` files (the server's work file, config, resume file) or their .tmp, is refused."""

    def __init__(self, start, end, key, dp, sink, bind="0.0.0.0", port=DEFAULT_PORT, workdir=".", out=print,
                 cmd_timeout=CMD_TIMEOUT, idle_timeout=CLIENT_TIMEOUT, protected=()):
        self.config = (struct.pack("<I", PROTOCOL_VERSION) + b"".join(int(v).to_bytes(32, "little") for v in (start, end, key[0], key[1]))
                       + struct.pack("<i", int(dp)))
        self.sink, self.bind, self.port, self.workdir, self.out = sink, bind, int(port), workdir, out
        self.cmd_timeout, self.idle_timeout = cmd_timeout, idle_timeout
        self.protected = {os.path.realpath(os.fsencode(p) + t) for p in protected if p for t in (b"", b".tmp")}
        self.clients = set()
        self._lock = threading.Lock()
        self._handlers = []                                  # handler threads still running (pruned at each accept)
        self._acceptor = None
        self._closing = False
        self._lsock = None

    def listen(self):
        s = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
        s.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        s.bind((self.bind, self.port))
        s.listen(64)
        s.settimeout(0.25)                                  # the acceptor polls _closing
        self._lsock, self.port = s, s.getsockname()[1]
        self._acceptor = threading.Thread(target=self._accept_loop, name="acceptor", daemon=True)
        self._acceptor.start()
        self.out("Kangaroo server is ready and listening to TCP port %d ..." % self.port)

    def n_clients(self):
        with self._lock:
            return len(self.clients)

    def kangaroos(self):
        with self._lock:
            return sum(c.knb for c in self.clients)

    def close(self):
        """stop accepting, close every connection and wait for the handlers"""
        self._closing = True
        if self._acceptor is not None:
            self._acceptor.join()                            # no handler starts after this
        with self._lock:
            for c in self.clients:
                try:
                    c.sock.shutdown(socket.SHUT_RDWR)
                except OSError:
                    pass
            handlers = list(self._handlers)
        for t in handlers:
            t.join()
        if self._lsock is not None:
            self._lsock.close()

    def _accept_loop(self):
        while not self._closing:
            try:
                sock, addr = self._lsock.accept()
            except socket.timeout:
                continue
            except OSError:
                break
            c = Client(sock, addr)
            with self._lock:
                if self._closing:
                    sock.close()
                    break
                self.clients.add(c)
                t = threading.Thread(target=self._handle, args=(c,), name="client %s" % c.name, daemon=True)
                self._handlers = [h for h in self._handlers if h.is_alive()] + [t]
            t.start()

    def _handle(self, c):
        try:
            self._serve(c)
        except ClientGone as e:
            if not self._closing:
                self.out("Closing connection with %s (%s)" % (c.name, e))
        finally:
            with self._lock:
                self.clients.discard(c)
            c.sock.close()

    def _send(self, c, data):
        try:
            c.sock.sendall(data)
        except OSError as e:
            raise ClientGone(str(e))

    def _file_name(self, c):
        """a kangaroo file's name from the client -> its path in workdir; ClientGone when refused"""
        size = struct.unpack("<I", recv_exact(c.sock, 4))[0]
        if size >= 256:
            raise ClientGone("file name too long (%d bytes, at most 255)" % size)
        name = recv_exact(c.sock, size)
        why = file_name_error(name)
        if why:
            raise ClientGone("kangaroo file name refused: %s" % why)
        path = os.path.join(os.fsencode(self.workdir), name)
        if os.path.realpath(path) in self.protected or os.path.realpath(path + b".tmp") in self.protected:
            raise ClientGone("kangaroo file name refused: %r is one of the server's own files" % name.decode(errors="replace"))
        if os.path.islink(path) or os.path.islink(path + b".tmp"):
            raise ClientGone("kangaroo file name refused: %s is a symbolic link" % os.fsdecode(path))
        return path

    def _serve(self, c):
        sock = c.sock
        while not self._closing:
            sock.settimeout(self.idle_timeout)
            try:
                cmd = sock.recv(1)
            except (socket.timeout, OSError) as e:
                raise ClientGone(str(e) or "idle timeout")
            if not cmd:
                return
            sock.settimeout(self.cmd_timeout)
            cmd = cmd[0]
            if cmd == CMD_GETCONFIG:
                self.out("New connection from %s" % c.name)
                self._send(c, self.config)
            elif cmd == CMD_STATUS:
                self._send(c, struct.pack("<i", self.sink.status()))
            elif cmd == CMD_SETKNB:
                knb = struct.unpack("<Q", recv_exact(sock, 8))[0]
                with self._lock:
                    c.knb = knb
            elif cmd == CMD_RESETDEAD:
                recv_exact(sock, 2)
                self.sink.reset_dead()
                self._send(c, b"OK\n")
            elif cmd == CMD_SENDDP:
                self._senddp(c)
            elif cmd == CMD_SAVEKANG:
                self._savekang(c)
            elif cmd == CMD_LOADKANG:
                self._loadkang(c)
            else:
                raise ClientGone("unexpected command [%d]" % cmd)

    def _senddp(self, c):
        magic, nb, tid, pid, gid = struct.unpack("<5I", recv_exact(c.sock, 20))
        if magic != DP_MAGIC:
            raise ClientGone("unexpected DP header 0x%08X" % magic)
        if nb == 0:
            raise ClientGone("unexpected number of DP [0]")
        chunks, left = [], nb
        while left:
            k = min(left, CHUNK_RECORDS)
            buf = np.empty(k * DP40, dtype=np.uint8)
            recv_into(c.sock, memoryview(buf))
            chunks.append(buf)
            left -= k
        self._send(c, struct.pack("<i", self.sink.status()))
        self.sink.put(Message(c, nb, tid, pid, gid), chunks)

    def _savekang(self, c):
        path = self._file_name(c)
        nb = struct.unpack("<Q", recv_exact(c.sock, 8))[0]
        tmp = path + b".tmp"
        total = 0
        try:
            fd = os.open(tmp, os.O_WRONLY | os.O_CREAT | os.O_TRUNC | os.O_NOFOLLOW, 0o644)   # never through a link
            with os.fdopen(fd, "wb") as f:
                f.write(struct.pack("<IIQ", HEADKS, 0, nb))
                left = nb
                while left:
                    k = min(left, KANG_PER_BLOCK)
                    raw = recv_exact(c.sock, 16 * k)
                    f.write(raw)
                    total += kang_checksum(raw)
                    left -= k
                got = int.from_bytes(recv_exact(c.sock, 32), "little")
        except OSError as e:
            if e.errno != errno.ELOOP:                       # a link at NAME.tmp is not ours to remove
                self._remove(tmp)
            raise ClientGone("cannot write %s: %s" % (os.fsdecode(tmp), e))
        except ClientGone:
            self._remove(tmp)
            raise
        if got != total % (1 << 256):
            self._remove(tmp)
            self.out("Warning, kangaroo backup wrong checksum %s from %s: not written" % (os.fsdecode(path), c.name))
        else:
            os.replace(tmp, path)                            # replaces a link at NAME itself, never its target

    @staticmethod
    def _remove(path):
        try:
            os.remove(path)
        except OSError:
            pass

    def _loadkang(self, c):
        path = self._file_name(c)
        try:
            f = os.fdopen(os.open(path, os.O_RDONLY | os.O_NOFOLLOW), "rb")
        except OSError as e:
            if e.errno == errno.ELOOP:
                raise ClientGone("kangaroo file name refused: %s is a symbolic link" % os.fsdecode(path))
            self.out("LoadKang: cannot open %s for reading: %s" % (os.fsdecode(path), e.strerror))
            self._send(c, struct.pack("<Q", 0))
            return
        with f:
            head = f.read(16)
            if len(head) != 16 or struct.unpack_from("<I", head)[0] != HEADKS:
                raise ClientGone("LoadKang: %s is not a kangaroo file" % os.fsdecode(path))
            nb = struct.unpack_from("<Q", head, 8)[0]
            self._send(c, struct.pack("<Q", nb))
            total, left = 0, nb
            while left:
                k = min(left, KANG_PER_BLOCK)
                raw = f.read(16 * k).ljust(16 * k, b"\0")
                total += kang_checksum(raw)
                self._send(c, raw)
                left -= k
            self._send(c, (total % (1 << 256)).to_bytes(32, "little"))


class RecordQueue:
    """the handlers' messages and the main thread's save and stop requests, in order, under a byte budget for records"""

    def __init__(self, budget=QUEUE_BYTES):
        self.budget, self.bytes = budget, 0
        self.items = collections.deque()
        self.cv = threading.Condition()
        self.blocked_s = 0.0                                 # handler time spent waiting for room

    def put_records(self, msg, chunks):
        for i, buf in enumerate(chunks):
            with self.cv:
                t0 = None
                while self.bytes > 0 and self.bytes + buf.nbytes > self.budget:
                    t0 = t0 or time.perf_counter()
                    self.cv.wait()
                if t0 is not None:
                    self.blocked_s += time.perf_counter() - t0
                self.bytes += buf.nbytes
                self.items.append(("recs", (msg, buf, i == len(chunks) - 1)))
                self.cv.notify_all()

    def put(self, kind, arg=None):
        with self.cv:
            self.items.append((kind, arg))
            self.cv.notify_all()

    def take(self, max_records):
        """-> ("recs", [(msg, buf, last), ...]): the first queued chunk and those after it that keep the batch within max_records
        records, or (kind, arg) of a request"""
        with self.cv:
            while not self.items:
                self.cv.wait()
            kind, arg = self.items[0]
            if kind != "recs":
                self.items.popleft()
                return kind, arg
            batch, n = [], 0
            while self.items and self.items[0][0] == "recs" and (not batch or n + self.items[0][1][1].nbytes // DP40 <= max_records):
                arg = self.items.popleft()[1]
                batch.append(arg)
                n += arg[1].nbytes // DP40
                self.bytes -= arg[1].nbytes
            self.cv.notify_all()
            return "recs", batch


class GpuSink:
    """The ingest thread and what it owns.  The table is split into one shard per `devices` entry (shard_plan), a DeviceDPTable
    of its buckets on that entry's GPU: one entry is the one table over every bucket, and a GPU listed k times holds k shards.
    Each distinct GPU has one resolver of the one key, shared by its shards, and one set of batch buffers; each shard has its
    own stream and, when there are several GPUs, a staging buffer on its GPU.  Everything is allocated here.  capacity is per
    shard; by default each GPU's free memory, less its buffers, is split evenly among its shards.  put / status / reset_dead
    are the Server's sink calls.

    The ingest thread, per batch: one copy to the next GPU in turn (spreading the verify), kgx_resolver_verify_partition there
    (the check, the good records grouped by shard in input order, the per-shard and bad counts), the counts back; then, unless
    some shard would overflow (nothing of the batch is added then), each shard's group -- read in place on the batch's GPU, or
    copied to the shard's staging buffer on another one -- added with its GPU's resolver on the shard's stream.  Each add
    waits for its own work, and a batch is done before the next starts, so every bucket sees its records in queue order, as
    the one table does.  A save writes the header, then each shard's piece at its offset: the one table's file, byte for byte."""

    def __init__(self, start, end, pub, dp, devices=(0,), capacity=None, resume=None, save_path="", out=print, entries="device"):
        import torch
        from .ingest import DeviceDPTable, DeviceResolver, DPTable, TableFull
        from .solver import DP_TABLE_MARGIN, default_table_capacity, host_entries_limit, mem_available, scratch_bytes
        self.torch = torch
        self.start, self.end, self.pub, self.dp = start, end, pub, dp
        self.save_path, self.out = save_path, out
        devices = list(devices)
        torch.cuda.set_device(devices[0])
        self.plan = shard_plan(devices)
        W = len(self.plan)
        gpus = sorted(set(devices))
        K = ec.add(pub, ec.neg(ec.mul(start))) if start else pub
        self.gpus = {}                                        # device -> its resolver, batch buffers and stream
        for d in gpus:
            dev = torch.device("cuda", d)
            r = DeviceResolver(DPTable.key_table([K]), start, device=d)
            nb = r.verify_partition_scratch_bytes(CHUNK_RECORDS, W)
            self.gpus[d] = dict(resolver=r, nb=nb,
                                recs=torch.empty(CHUNK_RECORDS * DP40, dtype=torch.uint8, device=dev),
                                out=torch.empty(CHUNK_RECORDS * DP40, dtype=torch.uint8, device=dev),
                                bad=torch.empty(CHUNK_RECORDS, dtype=torch.int32, device=dev),
                                counts=torch.empty(W + 1, dtype=torch.int32, device=dev),
                                scratch=torch.empty(nb, dtype=torch.uint8, device=dev))
        self._host = torch.empty(CHUNK_RECORDS * DP40, dtype=torch.uint8).pin_memory()
        self._host_np = self._host.numpy()
        self._counts_h = torch.empty(W + 1, dtype=torch.int32).pin_memory()
        staged = len(gpus) > 1
        per_shard = scratch_bytes(CHUNK_RECORDS) + EVENT_BYTES * CHUNK_RECORDS + (CHUNK_RECORDS * DP40 if staged else 0)
        self.entries = entries
        host_limit = host_entries_limit(mem_available(), W) if entries == "host" else None   # the host's RAM shared by all shards
        caps = {}
        for d in gpus:                                        # before any table takes memory
            k = devices.count(d)
            caps[d] = capacity or default_table_capacity((torch.cuda.mem_get_info(d)[0] - DP_TABLE_MARGIN) // k - per_shard,
                                                         margin=0, entries=entries, host_limit=host_limit)
        # a record makes at most one event, so room for a whole batch's events means no event of an add is ever cut off: a
        # hit cannot be pushed out by the RESETs of clients that keep resending, and the dead count is exact
        self.shards = []
        for s, (d, lo, hi) in enumerate(self.plan):
            dev = torch.device("cuda", d)
            t = DeviceDPTable(caps[d], device=d, max_events=CHUNK_RECORDS, buckets=(lo, hi), entries=entries)
            t.reserve(CHUNK_RECORDS)
            self.shards.append(dict(table=t, device=d, lo=lo, hi=hi, stream=torch.cuda.Stream(device=dev),
                                    staging=torch.empty(CHUNK_RECORDS * DP40, dtype=torch.uint8, device=dev) if staged else None))
            # a GPU checks its batches on its first shard's stream; torch makes its pool of streams at the first one, so
            # no stream is made before the capacity is read from the free memory
            self.gpus[d].setdefault("stream", self.shards[-1]["stream"])
        self.table = ShardTables([sh["table"] for sh in self.shards])
        self.shard_capacity = max(caps.values())
        self.time0 = 0.0
        if resume:
            info = None
            for s, sh in enumerate(self.shards):
                try:
                    info = sh["table"].load_piece(resume, sh["table"].capacity, stream=sh["stream"].cuda_stream)
                except TableFull as e:                       # refused before listening
                    where = " (shard %d of %d, buckets [%d, %d) on cuda:%d)" % (s, W, sh["lo"], sh["hi"], sh["device"]) if W > 1 else ""
                    raise TableFull("%s%s" % (e, where))
            self.time0 = info.total_time
            self.resumed = (len(self.table), info.nb_walk)
        self.t_start = time.perf_counter()
        self.queue = RecordQueue()
        self.dead = self.wrong = self.wrong_collisions = self.received = 0
        self.saving = 0
        self.solved = None                                   # the private key once found
        self.full = None                                     # why the table stopped the run
        self.failed = None                                   # an ingest error
        self.last_save = None                                # (path, error or None)
        self.batches, self.t_copy, self.t_verify, self.t_add, self.t_peer = 0, 0.0, 0.0, 0.0, 0.0
        self._turn = 0                                        # batches taken: the next one goes to gpus[_turn % len(gpus)]
        self._thread = threading.Thread(target=self._loop, name="ingest", daemon=True)
        self._thread.start()

    def describe(self):
        """the start line's words for the table"""
        if len(self.shards) == 1:
            return "capacity %d entries (%.2f GB) on cuda:%d%s" % (self.table.capacity, self.table.memory_bytes() / 1e9, self.plan[0][0],
                                                                  host_note(self.table))
        return "in %d shards on cuda:%s, capacity %d entries each (%.2f GB in all)%s" % (
            len(self.shards), ",".join(str(d) for d, _, _ in self.plan), self.shard_capacity, self.table.memory_bytes() / 1e9,
            host_note(self.table))

    # -- the Server's sink -----------------------------------------------------------------------------------------------
    def put(self, msg, chunks):
        self.queue.put_records(msg, chunks)

    def status(self):
        if self.solved is not None:
            return STATUS_END
        return STATUS_BACKUP if self.saving else STATUS_OK

    def reset_dead(self):
        self.dead = 0

    # -- the main thread ---------------------------------------------------------------------------------------------------
    def elapsed(self):
        return self.time0 + time.perf_counter() - self.t_start

    def request_save(self):
        """queue a save of --save-work behind every record queued so far (status BACKUP until it is written)"""
        if self.save_path:
            self.saving += 1
            self.queue.put("save")

    def finish(self):
        """write the work file of everything queued, then stop the ingest thread"""
        self.request_save()
        self.queue.put("stop")
        self._thread.join()

    def close(self):
        for sh in self.shards:
            sh["table"].close()
        for g in self.gpus.values():
            g["resolver"].close()

    # -- the ingest thread -------------------------------------------------------------------------------------------------
    def _loop(self):
        while True:
            kind, arg = self.queue.take(CHUNK_RECORDS)
            if kind == "stop":
                return
            try:
                if kind == "save":
                    self._save()
                elif self.full is None and self.failed is None:
                    self._ingest(arg)
            except Exception as e:                           # a CUDA error: the run stops with what the table holds
                self.failed = "%s: %s" % (type(e).__name__, e)

    def _save(self):
        from .solver import WorkFile
        wf = WorkFile(self.save_path, time.perf_counter())
        wf.begin(self._write_table)
        path, mb, secs, err = wf.finish()
        self.last_save = (path, err)
        if err is None:
            self.out("Work file %s written: %d DPs, %.1f MB in %.2f s" % (path, len(self.table), mb, secs))
        else:
            self.out("Work file %s NOT written: %s (the previous file is kept)" % (path, err))
        self.saving -= 1

    def _write_table(self, path):
        from .solver import piece_offsets, work_header
        with open(path, "wb") as f:
            f.write(work_header(self.dp, self.start, self.end, self.pub, 0, self.elapsed()))
        offsets = piece_offsets([sh["table"].piece_bytes() for sh in self.shards])
        for sh, o in zip(self.shards, offsets):
            sh["table"].save_piece(path, o, stream=sh["stream"].cuda_stream)
        with open(path, "r+b") as f:
            f.seek(offsets[-1])
            f.write(struct.pack("<Q", 0))                    # no kangaroos

    def _stage(self, batch):
        """the batch's records into the pinned host buffer -> (bytes, records, end of each chunk in records)"""
        sizes = [buf.nbytes for _, buf, _ in batch]
        ends = np.cumsum(sizes) // DP40
        off = 0
        for (_, buf, _), sz in zip(batch, sizes):
            self._host_np[off:off + sz] = buf
            off += sz
        return off, int(ends[-1]), ends

    def _charge(self, batch, ends, n_bad, bad):
        """n_bad wrong records, the device tensor bad holding their indices, charged to their messages and clients"""
        if n_bad:
            bad = bad[:n_bad].cpu().numpy()
            per_chunk = np.bincount(np.searchsorted(ends, bad, side="right"), minlength=len(batch))
            for (msg, _, _), k in zip(batch, per_chunk.tolist()):
                msg.bad += k
                msg.client.wrong += k
            self.wrong += n_bad
        for msg, _, last in batch:
            if last and msg.bad:
                self.out(msg.wrong_line())

    def _ingest(self, batch):
        torch = self.torch
        W = len(self.shards)
        off, n, ends = self._stage(batch)
        d = sorted(self.gpus)[self._turn % len(self.gpus)]
        self._turn += 1
        g = self.gpus[d]
        st = g["stream"]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        with torch.cuda.stream(st):
            ev[0].record(st)
            g["recs"][:off].copy_(self._host[:off], non_blocking=True)
            ev[1].record(st)
            g["resolver"].verify_partition_raw(g["recs"].data_ptr(), n, W, 0, g["out"].data_ptr(), g["counts"].data_ptr(),
                                               g["bad"].data_ptr(), CHUNK_RECORDS, g["scratch"].data_ptr(), g["nb"], st.cuda_stream)
            ev[2].record(st)
            self._counts_h.copy_(g["counts"], non_blocking=True)
        st.synchronize()
        self.t_copy += ev[0].elapsed_time(ev[1]) / 1e3
        self.t_verify += ev[1].elapsed_time(ev[2]) / 1e3
        c = [int(v) for v in self._counts_h.tolist()]
        self.received += n
        with torch.cuda.stream(st):
            self._charge(batch, ends, c[W], g["bad"])
        for s, sh in enumerate(self.shards):                 # a saved file is always a cut between whole batches
            t = sh["table"]
            if len(t) + c[s] > t.capacity:
                if W > 1:
                    self.full = ("shard %d of %d (buckets [%d, %d) on cuda:%d) holds %d entries, capacity %d; this batch brought it "
                                 "%d more" % (s, W, sh["lo"], sh["hi"], sh["device"], len(t), t.capacity, c[s]))
                else:                                        # the words of the add's refusal (TableFull), then the table's state
                    self.full = ("DP table full: %d entries + %d records of this call > capacity %d (%d entries, capacity %d; this batch "
                                 "brought %d more)" % (len(t), c[s], t.capacity, len(t), t.capacity, c[s]))
                return
        t0 = time.perf_counter()
        first = 0
        for s, sh in enumerate(self.shards):
            k, src = c[s], g["out"][first * DP40:(first + c[s]) * DP40]
            first += k
            if not k:
                continue
            if sh["device"] != d:                           # another GPU: into the shard's staging buffer, on its stream
                p0 = time.perf_counter()
                with torch.cuda.stream(sh["stream"]):
                    sh["staging"][:k * DP40].copy_(src, non_blocking=True)
                sh["stream"].synchronize()
                self.t_peer += time.perf_counter() - p0
                src = sh["staging"]
            evs = sh["table"].add(src.data_ptr(), [k], k, sh["stream"].cuda_stream, self.gpus[sh["device"]]["resolver"])
            self._events(evs)
        self.t_add += time.perf_counter() - t0
        self.batches += 1

    def _events(self, evs):
        from .ingest import EV_RESET, EV_COLLISION
        from .solver import print_key
        for e in evs:
            if e[0] == EV_RESET:
                self.dead += 1                               # the reference's collisionInSameHerd
            elif e[0] == EV_COLLISION:
                if e[5] is not None:
                    if self.solved is None and ec.mul(e[5][1]) == self.pub:
                        self.solved = e[5][1]
                        print_key(0, self.pub, self.solved)
                        sys.stdout.flush()
                else:
                    self.wrong_collisions += 1
                    self.out("Unexpected wrong collision (kIdx %d, bucket h of d %016X%016X / %016X%016X)" %
                             (e[2], e[3][1], e[3][0], e[4][1], e[4][0]))


def shard_plan(devices):
    """--devices -> [(device, lo, hi)] per shard: shard s of W holds the buckets [floor(s*2^18/W), floor((s+1)*2^18/W)), the
    range rank s of the solver's --dp-table sharded holds, so the pieces of a work file sit where the solver puts them"""
    from .dist import owner_ranges
    return [(d, lo, hi) for d, (lo, hi) in zip(devices, owner_ranges(len(devices)))]


def host_note(table):
    """the words the start line adds for a table with its entries in pinned host memory"""
    hb = table.host_bytes()
    return ", entries in pinned host memory (%.2f GB)" % (hb / 1e9) if hb else ""


class ShardTables:
    """the shards of a GpuSink as one table for the status line and the messages: entries, capacity and memory summed"""

    def __init__(self, tables):
        self.shards = tables
        self.capacity = sum(t.capacity for t in tables)

    def __len__(self):
        return sum(len(t) for t in self.shards)

    def memory_bytes(self):
        return sum(t.memory_bytes() for t in self.shards)

    def host_bytes(self):
        return sum(t.host_bytes() for t in self.shards)

    def fullest(self):
        """-> (shard, entries, capacity) of the shard with the largest fill"""
        s = max(range(len(self.shards)), key=lambda i: len(self.shards[i]) / self.shards[i].capacity)
        return s, len(self.shards[s]), self.shards[s].capacity


def expected_dps(start, end, kangaroos, dp):
    """log2 of the DPs the reference expects a search to need (Kangaroo::ComputeExpected, no symmetry)"""
    n = 2.0 ** max((end - start).bit_length(), 1)
    theta = 2.0 ** dp
    z0 = 2.0 * (2.0 - 2.0 ** 0.5) * np.pi ** 0.5
    return float(np.log2(z0 * (n * (kangaroos * theta + n ** 0.5)) ** (1.0 / 3.0) / theta))


def time_str(t):
    t = int(t)
    if t >= 86400:
        return "%.1fd" % (t / 86400.0)
    h, m, s = t // 3600, (t % 3600) // 60, t % 60
    return "%02d:%02d:%02d" % (h, m, s) if h else "%02d:%02d" % (m, s)


def status_line(server, sink):
    k = server.kangaroos()
    line = ("[Client %d][Kang 2^%.2f][DP Count 2^%.2f/2^%.2f][Dead %d][Wrong %d][%s][%d / %d entries]" %
            (server.n_clients(), np.log2(max(k, 1)), np.log2(max(len(sink.table), 1)),
             expected_dps(sink.start, sink.end, k, sink.dp), sink.dead, sink.wrong, time_str(sink.elapsed()), len(sink.table),
             sink.table.capacity))
    if len(sink.table.shards) > 1:
        s, n, cap = sink.table.fullest()
        line += "[fullest shard %d: %d / %d, %.1f%%]" % (s, n, cap, 100.0 * n / cap)
    return line


def parse_args(argv=None):
    """-> (arguments, range start, range end, public key, dp); argparse exits on a usage error or a refused config"""
    ap = argparse.ArgumentParser(prog="python -m kangaroo_b200.server",
                                 description="DP server for the reference's clients (kangaroo -c), with the DP table, a check "
                                             "of every received DP and the collision resolver on the GPU")
    ap.add_argument("config", nargs="?", help="range start, end and the one public key (optional with --resume)")
    ap.add_argument("--dp", type=int, default=None, help="distinguished-point bits the clients use (required without --resume)")
    ap.add_argument("--bind", default="0.0.0.0", help="address to listen on (default 0.0.0.0)")
    ap.add_argument("--port", type=int, default=DEFAULT_PORT, help="TCP port (default %d; 0 = an ephemeral port)" % DEFAULT_PORT)
    ap.add_argument("--device", type=int, default=None, help="the GPU that holds the table (default 0)")
    ap.add_argument("--devices", default=None, metavar="D0,D1,...",
                    help="split the table into one shard per entry, on that GPU (a GPU may be listed more than once), in the "
                         "solver's --dp-table sharded bucket ranges; two or more entries (at most %d)" % MAX_SHARDS)
    ap.add_argument("--dp-table-capacity", type=int, default=None, metavar="E",
                    help="entries the table holds, 48 bytes of GPU memory each (default: what fits in the free GPU memory); "
                         "with --devices, the entries of each shard (default: each GPU's free memory split among its shards)")
    ap.add_argument("--dp-table-entries", choices=("device", "host"), default="device",
                    help="where the table's 32-byte entries live: device (default) = GPU memory, 48 bytes per entry in all; "
                         "host = pinned host RAM mapped into the GPU, which then holds 16 bytes per entry, for about 2.6x the "
                         "entries per GPU.  The default capacity with host is also at most the host RAM available (MemAvailable) "
                         "less a margin, at 32 bytes per entry, shared by all shards; a larger --dp-table-capacity is refused")
    ap.add_argument("--save-work", default="", metavar="FILE", help="write the table as a HEADW work file at exit")
    ap.add_argument("--save-interval", type=float, default=0.0, metavar="SECS", help="also save every SECS seconds")
    ap.add_argument("--resume", default="", metavar="FILE", help="start from a work file: range, key and dp come from it")
    a = ap.parse_args(argv)
    if a.dp_table_capacity is not None and not 0 < a.dp_table_capacity < (1 << 32) - 1:
        ap.error("--dp-table-capacity must be 1 .. 2^32-2 entries, not %d" % a.dp_table_capacity)
    if a.save_interval and not a.save_work:
        ap.error("--save-interval needs --save-work FILE")
    if a.dp is not None and not 0 <= a.dp <= 64:
        ap.error("--dp must be 0 .. 64")
    if a.devices is not None:
        if a.device is not None:
            ap.error("give --device or --devices, not both")
        try:
            a.devices = [int(v) for v in a.devices.split(",")] if a.devices.strip() else []
        except ValueError:
            ap.error("--devices must be GPU indices separated by commas, not %r" % a.devices)
        if not a.devices:
            ap.error("--devices: the list is empty")
        if len(a.devices) > MAX_SHARDS:
            ap.error("--devices: %d entries, at most %d shards" % (len(a.devices), MAX_SHARDS))
        if min(a.devices) < 0:
            ap.error("--devices: GPU indices are not negative")
        a.device = a.devices[0]
    elif a.device is None:
        a.device = 0
    if a.dp_table_entries == "host":
        from .solver import host_capacity_error, mem_available
        err = host_capacity_error(a.dp_table_capacity, mem_available(), len(a.devices or [a.device]))
        if err:
            ap.error(err.replace("table(s)", "shard(s)"))
    pubs = None
    if a.config:
        start, end, pubs = ec.parse_config(a.config)
        if len(pubs) != 1:
            ap.error("%s holds %d keys: a server serves exactly one key (GETCONFIG carries one key)" % (a.config, len(pubs)))
    if a.resume:
        from .ingest import read_work_header
        try:
            h = read_work_header(a.resume)
        except (OSError, RuntimeError) as e:
            ap.error("--resume: %s" % e)
        if pubs is not None and (start, end, pubs[0]) != (h.range_start, h.range_end, h.key):
            ap.error("--resume: %s is not the config's search: the file has range 0x%X .. 0x%X and key 04%064X%064X" %
                     (a.resume, h.range_start, h.range_end, h.key[0], h.key[1]))
        start, end, pubs = h.range_start, h.range_end, [h.key]
        dp = a.dp if a.dp is not None else h.dp_bits
    elif pubs is None:
        ap.error("a config file or --resume FILE is required")
    elif a.dp is None:
        ap.error("--dp is required: the server gives the clients their dp")
    else:
        dp = a.dp
    return a, start, end, pubs[0], dp


def main(argv=None):
    a, start, end, pub, dp = parse_args(argv)
    out = lambda s: print(s, flush=True)
    from .ingest import TableFull
    try:
        sink = GpuSink(start, end, pub, dp, a.devices or [a.device], capacity=a.dp_table_capacity, resume=a.resume or None,
                       save_path=a.save_work, out=out, entries=a.dp_table_entries)
    except TableFull as e:
        out("--resume %s refused: %s; give a larger --dp-table-capacity" % (a.resume, e))
        return 1
    if a.resume:
        out("Resume %s: %d DPs" % (a.resume, sink.resumed[0]))
        if sink.resumed[1]:
            out("%d kangaroos in %s skipped: the server keeps no herd" % (sink.resumed[1], a.resume))
    out("Range 0x%X .. 0x%X  dp %d  key 04%064X%064X  table %s" % (start, end, dp, pub[0], pub[1], sink.describe()))
    stop = threading.Event()
    signals = []

    def on_signal(signum, frame):
        signals.append(signum)
        stop.set()

    old = {s: signal.signal(s, on_signal) for s in (signal.SIGINT, signal.SIGTERM)}
    server = Server(start, end, pub, dp, sink, bind=a.bind, port=a.port, out=out,
                    protected=[a.save_work, a.config, a.resume])
    try:
        server.listen()
    except OSError as e:
        out("Cannot listen on %s:%d: %s" % (a.bind, a.port, e))
        sink.finish()
        sink.close()
        return 1
    rc, solved_at = 1, None
    next_status = time.monotonic() + STATUS_PERIOD
    next_save = time.monotonic() + a.save_interval if a.save_interval > 0 else None
    try:
        while not stop.wait(0.1):
            now = time.monotonic()
            if sink.full is not None or sink.failed is not None:
                break
            if sink.solved is not None:
                solved_at = solved_at or now
                if server.n_clients() == 0 or now - solved_at >= END_GRACE:
                    rc = 0
                    break
            if now >= next_status:
                out(status_line(server, sink))
                next_status = now + STATUS_PERIOD
            if next_save is not None and now >= next_save and not sink.saving:
                sink.request_save()
                next_save = now + a.save_interval
    finally:
        server.close()
        sink.finish()
        for s, h in old.items():
            signal.signal(s, h)
    out(status_line(server, sink))
    if signals:
        out("Stopped by signal %d" % signals[0])
        rc = 1
    if sink.full is not None:
        out("DP table full%s, server stopped: %s.  Resume with --resume %s --dp-table-capacity %d or more; the clients reconnect "
            "and resend the DPs they hold." % (" (host entries)" if a.dp_table_entries == "host" else "", sink.full, a.save_work or "FILE (give --save-work to write one)",
                                               2 * sink.shard_capacity))
        rc = 1
    if sink.failed is not None:
        out("Ingest failed, server stopped: %s" % sink.failed)
        rc = 1
    if a.save_work and (sink.last_save is None or sink.last_save[1] is not None):
        rc = 1
    out("Server: %d DPs received, %d wrong, %d dead, %d wrong collisions; %d batches: copy %.3f ms, verify %.3f ms, add %.3f ms "
        "per batch; handlers blocked %.2f s on a full queue" %
        (sink.received, sink.wrong, sink.dead, sink.wrong_collisions, sink.batches, 1e3 * sink.t_copy / max(sink.batches, 1),
         1e3 * sink.t_verify / max(sink.batches, 1), 1e3 * sink.t_add / max(sink.batches, 1), sink.queue.blocked_s))
    if len(sink.shards) > 1:
        out("Shards: verify is verify+partition; add includes %.3f ms per batch of copies to other GPUs" %
            (1e3 * sink.t_peer / max(sink.batches, 1)))
    sink.close()
    return rc


if __name__ == "__main__":
    sys.exit(main())
