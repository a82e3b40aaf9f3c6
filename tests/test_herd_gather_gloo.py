"""world_size-2 gloo test (CPU) of the chunked herd gather a work-file save uses (kangaroo_b200/dist.py HerdGather): herds
of unequal size, a chunk size that divides neither, rank 0 receives every kangaroo record in rank order; and the reverse
used by a resume, where rank 0 alone reads the file and sends every rank its records."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

SIZES = (1000, 1538)
CHUNK = 300
NB_WALK = 2300            # fewer than the two herds hold: rank 1 keeps 238 fresh kangaroos


def _herd(rank):
    n = SIZES[rank]
    return (np.arange(n * 12, dtype=np.uint64).reshape(n, 12) + np.uint64(rank << 40)) * np.uint64(0x9E3779B97F4A7C15)


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from kangaroo_b200.dist import HerdGather, WALK_BYTES
    herd = _herd(rank)
    g = HerdGather(dist, rank, world, torch, len(herd), torch.device("cpu"), CHUNK)
    calls = []

    def export(first, count, dst):
        calls.append((first, count))
        assert dst.numel() == count * WALK_BYTES
        dst.copy_(torch.from_numpy(herd[first:first + count].copy().view(np.uint8).reshape(-1)))

    got = []
    for j in range(len(g.plan)):
        v = g.chunk(j, export)
        if rank == 0:
            got.append(v.numpy().copy())
        else:
            assert v is None
    assert sum(c for _, c in calls) == len(herd) and max(c for _, c in calls) <= CHUNK
    # the reverse (resume): a file of NB_WALK kangaroos, read on rank 0 only, scattered in rank order
    block = np.concatenate([_herd(0), _herd(1)])[:NB_WALK]
    reads = []

    def read(first, count):
        assert rank == 0 and count <= CHUNK
        reads.append(count)
        return block[first:first + count].copy().view(np.uint8).reshape(-1)

    mine = g.scatter(NB_WALK, read)
    take = max(0, min(len(herd), NB_WALK - g.offsets[rank]))
    assert mine.tobytes() == herd[:take].tobytes()
    if rank == 0:
        assert sum(reads) == NB_WALK
        q.put((g.sizes, g.offsets, g.total, np.concatenate(got).tobytes()))
    dist.destroy_process_group()


def test_chunked_herd_gather_world2_gloo():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    sizes, offsets, total, block = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert sizes == list(SIZES) and offsets == [0, SIZES[0]] and total == sum(SIZES)
    assert block == np.concatenate([_herd(0), _herd(1)]).tobytes()
