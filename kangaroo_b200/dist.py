"""Multi-GPU distinguished-point gather: independent herds one per GPU, DP records gathered to rank 0.

The reference has no collective: multi-GPU is threads sharing one host hash table under a mutex (Kangaroo.cpp:
594-612) and multi-host is a hand-rolled TCP client/server (Network.cpp).  In-box replacement (SURVEY.md 2b, 8e):
one process per GPU (torch.distributed), no exchange inside the jump loop, and per Launch a variable-length
gather of the 56-byte DP records (GPUMath.h:173-188 layout) to rank 0, which alone owns the hash table:

    counts  : all_gather of one int32 per rank                     (every rank learns max count)
    payload : gather of the first `cap` records of each rank's DP slab, cap = max count rounded up to 256
              records -- equal-sized buffers, so it is a plain NCCL gather over NVLink/NVSwitch (gloo on CPU)

The payload is read straight from the engine's device DP slab (no host bounce); the jump kernel of the NEXT
launch is already running on the engine's own stream while the gather proceeds on torch's stream.
"""
ITEM_BYTES = 56
DP40_BYTES = 40
ROUND = 256


class SlabView:
    """Wraps a raw device pointer as a torch uint8 tensor through __cuda_array_interface__."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


class DPGather:
    def __init__(self, engine, dist, rank, world, torch, device=None, slab_fn=None, max_found=None, wire="item56"):
        """engine: kangaroo_b200.GPUEngine (or None with slab_fn for the CPU/gloo tests).
        slab_fn() -> uint8 tensor [4 + max_found*56] of the most recently completed launch."""
        self.eng, self.dist, self.rank, self.world, self.torch = engine, dist, rank, world, torch
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.max_found = max_found if max_found is not None else engine.maxFound
        self._views = {}
        # wire = "item56": raw engine records; "dp40": the reference's 40-byte DP records, converted on the device
        # (HashTable::Convert, SURVEY 8f/f1) -- 29 % less gather traffic and ready for HashTable::Add(h, x, d)
        self.rec = ITEM_BYTES if wire == "item56" else DP40_BYTES
        self.wire = wire
        self._slab_fn = slab_fn if slab_fn is not None else (self._engine_slab if wire == "item56" else self._engine_dp40)
        self.total_gathered = 0
        self.last = None
        self._flat = None                # rank 0: step_flat's receive buffer, allocated by its first call

    def _engine_slab(self):
        ptr = self.eng.dp_slab_device_ptr()
        v = self._views.get(ptr)
        if v is None:
            nbytes = 4 + self.max_found * ITEM_BYTES
            v = self.torch.as_tensor(SlabView(ptr, nbytes), device=self.device)
            self._views[ptr] = v
        return v

    def _engine_dp40(self):
        ptr = self.eng.convert_dps_device_ptr()
        v = self._views.get(("dp40", ptr))
        if v is None:
            v = self.torch.as_tensor(SlabView(ptr, 4 + self.max_found * DP40_BYTES), device=self.device)
            self._views[("dp40", ptr)] = v
        return v

    def _gather(self, n_found, recv):
        """The count exchange and the gather: recv(cap) -> rank 0's receive buffers, one per rank of cap records each.
        n_found = records this rank produced (capped to max_found here).  Returns (counts list, cap, buffers or None)."""
        torch = self.torch
        cnt = min(int(n_found), self.max_found)
        mine = torch.tensor([cnt], dtype=torch.int32, device=self.device)
        counts = torch.empty(self.world, dtype=torch.int32, device=self.device)
        self.dist.all_gather_into_tensor(counts, mine)
        counts_h = counts.cpu().tolist()
        cap = min(max(ROUND, (max(counts_h) + ROUND - 1) // ROUND * ROUND), self.max_found)
        local = self._slab_fn()[4:4 + cap * self.rec]
        bufs = recv(cap) if self.rank == 0 else None
        self.dist.gather(local, bufs, dst=0)
        if self.device.type == "cuda":
            torch.cuda.current_stream().synchronize()   # the slab is recycled by the launch after next
        self.total_gathered += sum(counts_h)
        return counts_h, cap, bufs

    def step(self, n_found):
        """Gather this launch's DP records to rank 0.  Returns on rank 0 a list of (rank, uint8 tensor [cnt*56]);
        None elsewhere."""
        counts, cap, bufs = self._gather(n_found, lambda cap: [self.torch.empty(cap * self.rec, dtype=self.torch.uint8,
                                                                                  device=self.device) for _ in range(self.world)])
        self.last = [(r, bufs[r][:counts[r] * self.rec]) for r in range(self.world)] if self.rank == 0 else None
        return self.last

    def step_flat(self, n_found):
        """Like step(), but rank 0 receives every rank's records in ONE contiguous device tensor (rank r at offset r*cap*rec),
        so that the whole step's DPs reach rank 0's table with a single copy.  Returns (counts list, cap, tensor) on rank 0,
        None elsewhere."""
        if self.rank == 0 and self._flat is None:
            self._flat = self.torch.empty(self.world * self.max_found * self.rec, dtype=self.torch.uint8, device=self.device)
        counts, cap, _ = self._gather(n_found, lambda cap: [self._flat[r * cap * self.rec:(r + 1) * cap * self.rec]
                                                            for r in range(self.world)])
        return (counts, cap, self._flat) if self.rank == 0 else None


WALK_BYTES = 96          # one kangaroo of a work file (Backup.cpp:536-539)


class HerdGather:
    """The herds of all ranks to rank 0 as one work-file kangaroo block, in rank order (rank 0's kIdx 0..n0-1, then rank
    1's, ...), so that the reference reads it as one herd.  Herd sizes may differ per rank (GetGridSize runs per GPU): they
    are exchanged once here.  The block moves in chunks of at most `chunk` records that never span two ranks; every chunk
    goes through one fixed buffer of chunk*96 bytes on `device` (a point-to-point send from its owner to rank 0).

    Every rank calls chunk(j) for j in range(len(plan)) in the same order."""

    def __init__(self, dist, rank, world, torch, n_local, device, chunk):
        self.dist, self.rank, self.world, self.torch, self.device = dist, rank, world, torch, device
        if dist is not None and world > 1:
            mine = torch.tensor([int(n_local)], dtype=torch.int64, device=device)
            sizes = torch.empty(world, dtype=torch.int64, device=device)
            dist.all_gather_into_tensor(sizes, mine)
            self.sizes = [int(v) for v in sizes.cpu().tolist()]
        else:
            self.sizes = [int(n_local)]
        self.offsets = [sum(self.sizes[:r]) for r in range(len(self.sizes))]
        self.total = sum(self.sizes)
        self.chunk_records = int(chunk)
        self.plan = [(r, first, min(self.chunk_records, n - first)) for r, n in enumerate(self.sizes) for first in range(0, n, self.chunk_records)]
        self._buf = None
        # gloo's send / recv take host tensors only: under gloo every chunk crosses through a host buffer of the same size
        self._staged = dist is not None and world > 1 and dist.get_backend() == "gloo"
        self._host = None

    def _host_view(self, nbytes):
        if self._host is None:
            self._host = self.torch.empty(self.chunk_records * WALK_BYTES, dtype=self.torch.uint8,
                                          pin_memory=self.device.type == "cuda")
        return self._host[:nbytes]

    def _send(self, view, dst):
        if self._staged:
            h = self._host_view(view.numel())
            h.copy_(view)
            view = h
        self.dist.send(view, dst=dst)

    def _recv(self, view, src):
        if self._staged:
            h = self._host_view(view.numel())
            self.dist.recv(h, src=src)
            view.copy_(h)
        else:
            self.dist.recv(view, src=src)

    def chunk(self, j, export):
        """Move chunk j of the plan to rank 0.  export(first, count, dst) writes this rank's records [first, first+count)
        into dst (a uint8 tensor of count*96 bytes on `device`); it is called on the owning rank only.  Returns the records
        (a view of the gather buffer, valid until the next call) on rank 0, None elsewhere."""
        r, first, count = self.plan[j]
        if self.rank != r and self.rank != 0:
            return None
        if self._buf is None:
            self._buf = self.torch.empty(self.chunk_records * WALK_BYTES, dtype=self.torch.uint8, device=self.device)
        view = self._buf[:count * WALK_BYTES]
        if self.rank == r:
            export(first, count, view)
        if r != 0:
            if self.rank == r:
                self._send(view, 0)
            else:
                self._recv(view, r)
            if self.device.type == "cuda":
                self.torch.cuda.current_stream().synchronize()   # the next export rewrites the buffer from another stream
        return view if self.rank == 0 else None

    def scatter(self, nb_walk, read):
        """The reverse, for a resume (FetchWalks): the first nb_walk kangaroos of a file, read on rank 0 only, to their
        ranks through the same chunk plan and buffer.  read(first, count) -> uint8 numpy array of count*96 bytes (called on
        rank 0).  Returns this rank's records [0, min(n_r, nb_walk - o_r)) as a uint8 numpy array."""
        import numpy as np
        off = self.offsets[self.rank]
        out = np.empty(max(0, min(self.sizes[self.rank], nb_walk - off)) * WALK_BYTES, dtype=np.uint8)
        for r, first, count in self.plan:
            count = max(0, min(count, nb_walk - self.offsets[r] - first))
            if count == 0 or (self.rank != r and self.rank != 0):
                continue
            if self._buf is None:
                self._buf = self.torch.empty(self.chunk_records * WALK_BYTES, dtype=self.torch.uint8, device=self.device)
            view = self._buf[:count * WALK_BYTES]
            if self.rank == 0:
                view.copy_(self.torch.from_numpy(read(self.offsets[r] + first, count)))
            if r != 0:
                if self.rank == 0:
                    self._send(view, r)
                else:
                    self._recv(view, 0)
                if self.device.type == "cuda":
                    self.torch.cuda.current_stream().synchronize()
            if self.rank == r:
                out[first * WALK_BYTES:(first + count) * WALK_BYTES] = view.cpu().numpy()
        return out


def decode_records(buf):
    """uint8 tensor/bytes of 56-byte records -> list of (x, d_biased, kidx) Python ints (GPUEngine.cu:653-671)."""
    b = bytes(buf.cpu().numpy().tobytes()) if hasattr(buf, "cpu") else bytes(buf)
    out = []
    for o in range(0, len(b), ITEM_BYTES):
        x = int.from_bytes(b[o:o + 32], "little")
        d = int.from_bytes(b[o + 32:o + 48], "little")
        k = int.from_bytes(b[o + 48:o + 56], "little")
        out.append((x, d, k))
    return out


def decode_dp40(buf):
    """40-byte DP records -> list of (kIdx32, h, x128, dist (signed int), type): HashTable::CalcDistAndType (HashTable.cpp:249-260)."""
    b = bytes(buf.cpu().numpy().tobytes()) if hasattr(buf, "cpu") else bytes(buf)
    out = []
    for o in range(0, len(b), DP40_BYTES):
        kidx = int.from_bytes(b[o:o + 4], "little")
        h = int.from_bytes(b[o + 4:o + 8], "little")
        x = int.from_bytes(b[o + 8:o + 24], "little")
        d = int.from_bytes(b[o + 24:o + 40], "little")
        ktype = (d >> 126) & 1
        mag = d & ((1 << 126) - 1)
        out.append((kidx, h, x, -mag if d >> 127 else mag, ktype))
    return out


# ---- the sharded DP table (--dp-table sharded): every rank's records to the ranks that own their buckets ----------------------
NBUCKET = 1 << 18        # HASH_SIZE: the buckets of a DP table, h = x.bits64[2] & 0x3FFFF


def owner_ranges(world):
    """[(lo, hi)] per rank: rank r of W owns the buckets [floor(r*2^18/W), floor((r+1)*2^18/W))"""
    return [(r * NBUCKET // world, (r + 1) * NBUCKET // world) for r in range(world)]


def owner_of(h, world):
    """the rank that owns bucket h (h < 2^18), as kgx_partition.cuh computes it: the last r with floor(r*2^18/W) <= h"""
    return ((h + 1) * world - 1) // NBUCKET


class DPExchange:
    """The sharded table's exchange, beside DPGather: each rank's 40-byte DP records go to the ranks that own their buckets.

        partition : kgx_dp_partition groups this rank's records by owner (stable), group r at record r*max_found
        counts    : all_gather of every rank's W + 1 counts (its groups, then its malformed records): every rank learns what it
                    receives, and cap = the largest count rounded up to 256 records
        payload   : one equal-split all_to_all_single of cap records per (source, destination) pair into a [W][cap] buffer

    A shard receives source rank 0's records first, then rank 1's, ..., each in the order its source produced them: restricted to
    one bucket, the order the single table sees.  step() returns (records from each source, cap, receive buffer, malformed
    records of this rank); the buffer is rewritten by the next step.

    engine: kangaroo_b200.GPUEngine, or None with partition_fn for the CPU (gloo) tests: partition_fn(n) -> (uint8 tensor of W
    groups of max_found records, W + 1 counts as an int32 tensor)."""

    def __init__(self, engine, dist, rank, world, torch, device=None, max_found=None, partition_fn=None):
        self.eng, self.dist, self.rank, self.world, self.torch = engine, dist, rank, world, torch
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.max_found = max_found if max_found is not None else engine.maxFound
        self._partition = partition_fn if partition_fn is not None else self._engine_partition
        self._send = self._recv = self._scratch = self._counts = None
        self.total_exchanged = 0

    def _engine_partition(self, n):
        """this launch's converted records grouped by owner on the device (torch's stream)"""
        import ctypes
        torch, W = self.torch, self.world
        lib = self.eng._lib
        if self._send is None:
            self._send = torch.empty(W * self.max_found * DP40_BYTES, dtype=torch.uint8, device=self.device)
            self._counts = torch.empty(W + 1, dtype=torch.int32, device=self.device)
            nb = int(lib.kgx_dp_partition_scratch_bytes(self.max_found, W))
            self._scratch = torch.empty(nb, dtype=torch.uint8, device=self.device)
        src = self.eng.convert_dps_device_ptr() + 4
        rc = lib.kgx_dp_partition(ctypes.c_void_p(src), int(n), W, self.max_found, ctypes.c_void_p(self._send.data_ptr()),
                                  ctypes.c_void_p(self._counts.data_ptr()), ctypes.c_void_p(self._scratch.data_ptr()),
                                  self._scratch.numel(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError("kgx_dp_partition failed (%d)" % rc)
        return self._send, self._counts

    def step(self, n_found):
        torch, W, R = self.torch, self.world, DP40_BYTES
        n = min(int(n_found), self.max_found)
        send, counts = self._partition(n)
        if W == 1:
            c = [int(v) for v in counts.cpu().tolist()]
            res = [c[0]], c[0], send, c[1]
        else:
            allc = torch.empty(W * (W + 1), dtype=torch.int32, device=self.device)
            self.dist.all_gather_into_tensor(allc, counts)
            m = allc.cpu().view(W, W + 1).tolist()                          # m[source][destination], then malformed
            cap = min(max(ROUND, (max(max(row[:W]) for row in m) + ROUND - 1) // ROUND * ROUND), self.max_found)
            if self._recv is None:
                self._recv = torch.empty(W * self.max_found * R, dtype=torch.uint8, device=self.device)
            payload = send.view(W, self.max_found * R)[:, :cap * R].reshape(-1)   # [W][cap]: a copy unless cap = max_found
            recv = self._recv[:W * cap * R]
            self.dist.all_to_all_single(recv, payload)
            res = [m[s][self.rank] for s in range(W)], cap, recv, m[self.rank][W]
        if self.device.type == "cuda":
            torch.cuda.current_stream().synchronize()   # the engine's record buffer is recycled by the launch after next
        self.total_exchanged += sum(res[0])
        return res
