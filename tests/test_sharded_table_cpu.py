"""CPU tests of --dp-table sharded: the owner ranges and the partition model, the per-step block's encoding, the capacity
refusals, and dist.DPExchange over gloo at world sizes 2 to 4 (the record exchange every step makes)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from kangaroo_b200 import solver as S
from kangaroo_b200.dist import DPExchange, NBUCKET, owner_of, owner_ranges
from tests import shard_model as sm


def recs_of(rng, n, kidx0=0, buckets=None, bad=0):
    """n records (kIdx = kidx0 + position), h random or drawn from `buckets`; the last `bad` of them malformed"""
    h = rng.integers(0, NBUCKET, size=n, dtype=np.uint64) if buckets is None else rng.choice(np.asarray(buckets, np.uint64), size=n)
    if bad:
        h[n - bad:] = np.uint64(NBUCKET) + rng.integers(0, 1 << 20, size=bad, dtype=np.uint64)
    out = rng.integers(0, 1 << 63, size=(n, 5), dtype=np.uint64)
    out[:, 0] = (h << np.uint64(32)) | np.arange(kidx0, kidx0 + n, dtype=np.uint64)
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 7, 8, 256])
def test_owner_ranges_cut_at_floor_r_2p18_over_w(world):
    rng = owner_ranges(world)
    assert [lo for lo, _ in rng] == [r * NBUCKET // world for r in range(world)]
    assert rng[0][0] == 0 and rng[-1][1] == NBUCKET and all(rng[r][1] == rng[r + 1][0] for r in range(world - 1))
    h = np.arange(NBUCKET, dtype=np.int64)
    own = ((h + 1) * world - 1) // NBUCKET                      # the kernel's formula
    assert (own == sm.owners(h, world)).all()
    for r, (lo, hi) in enumerate(rng):
        for b in {lo - 1, lo, hi - 1, hi} & set(range(NBUCKET)):
            assert owner_of(b, world) == (r if lo <= b < hi else r - 1 if b < lo else r + 1)


@pytest.mark.parametrize("world", [1, 2, 3, 7, 8, 256])
def test_partition_model_is_stable_and_complete(world):
    rng = np.random.default_rng(world)
    bounds = sm.owner_bounds(world)
    edges = sorted({b + d for b in bounds for d in (-1, 0) if 0 <= b + d < NBUCKET})
    recs = np.concatenate([recs_of(rng, 3000), recs_of(rng, 500, 3000, edges), recs_of(rng, 20, 3500, bad=7)])
    groups, bad = sm.partition(recs, world)
    assert bad == 7 and sum(len(g) for g in groups) == len(recs) - 7
    for r, g in enumerate(groups):
        h = g[:, 0] >> np.uint64(32)
        assert ((h >= np.uint64(bounds[r])) & (h < np.uint64(bounds[r + 1]))).all()
        k = (g[:, 0] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        assert (np.diff(k) > 0).all()                            # input order kept
    one, _ = sm.partition(recs[:0], world)
    assert all(len(g) == 0 for g in one)


def test_block_round_trip_and_carry_over():
    hits = [(i % 7, (1 << 255) - 1 - i, i % 3, 1000 + i) for i in range(S.BLOCK_HITS + 5)]
    resets = [(i % 4, (1 << 32) - 1 - i) for i in range(S.MAX_RESETS + 9)]
    b, lh, lr = S.encode_block(hits, resets, 123456789012, stop=1, msg="shard 2 of 8 é", size=1 << 40, done=2, err="disk full",
                               busy=1, chunks=3)
    assert b.dtype == np.int64 and b.size == S.BLOCK_WORDS
    d = S.decode_block(b)
    assert d["hits"] == hits[:S.BLOCK_HITS] and d["resets"] == resets[:S.MAX_RESETS]
    assert lh == hits[S.BLOCK_HITS:] and lr == resets[S.MAX_RESETS:]
    assert (d["count"], d["stop"], d["size"], d["done"], d["busy"], d["chunks"]) == (123456789012, 1, 1 << 40, 2, 1, 3)
    assert d["msg"] == "shard 2 of 8 é" and d["err"] == "disk full"
    b2, lh2, lr2 = S.encode_block(lh, lr, 0)                    # the next step carries the rest
    d2 = S.decode_block(b2)
    assert d2["hits"] == lh and d2["resets"] == lr and lh2 == [] and lr2 == []
    assert (d2["stop"], d2["size"], d2["done"], d2["msg"], d2["err"]) == (0, -1, 0, "", "")
    long = S.decode_block(S.encode_block([], [], 0, msg="x" * 1000)[0])["msg"]
    assert long == "x" * (8 * S.BLOCK_MSG - 1)


def test_piece_offsets_and_header():
    assert S.piece_offsets([8 * 5, 8 * 7 + 32, 8]) == [156, 196, 284, 292]
    h = S.work_header(12, 5, 9, (3, 4), 77, 1.5)
    assert len(h) == 156 and h[:4] == bytes.fromhex("01806afa")


def test_capacity_refusals(capsys):
    assert S.shard_headroom(8, 1 << 17) == 2 * 8 * (1 << 17)
    assert S.sharded_capacity_error(None, 8) is None
    assert S.sharded_capacity_error(2 * (1 << 17) + 1, 1) is None
    assert "cannot hold" in S.sharded_capacity_error(2 * (1 << 17), 1)
    assert "cannot hold" in S.sharded_capacity_error(4 * (1 << 17), 2)
    cfg = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "in56.txt")
    for argv, want in [([cfg, "--dp-table", "sharded", "--dp-table-capacity", "1000"], "cannot hold"),
                       ([cfg, "--dp-table", "host", "--dp-table-capacity", "1000000"], "needs --dp-table device or sharded"),
                       ([cfg, "--dp-table", "sharded", "--dp-table-capacity", str(1 << 32)], "must be 1 .. 2^32-2")]:
        with pytest.raises(SystemExit):
            S.main(argv)
        assert want in capsys.readouterr().err


# ---- DPExchange over gloo ---------------------------------------------------------------------------------------------------
MAX_FOUND = 1536


def step_records(step, rank, world):
    """rank's records of a step: some ranks send nothing at some steps, some only to one owner, some malformed"""
    rng = np.random.default_rng(1000 * step + rank)
    n = [0, 700, MAX_FOUND, 37][(step + rank) % 4]
    if step == 1 and rank == world - 1:
        return recs_of(rng, 300, rank << 20, buckets=[NBUCKET - 1]), 0              # all to the last rank
    bad = 3 if n and step == 2 else 0
    bounds = sm.owner_bounds(world)
    edges = [b + d for b in bounds for d in (-1, 0) if 0 <= b + d < NBUCKET]
    r = recs_of(rng, n, rank << 20, edges if step == 3 else None, bad)
    return r, bad


def _exchange_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    out = []
    for step in range(5):
        recs, bad = step_records(step, rank, world)

        def part(n, recs=recs):
            assert n == len(recs)
            groups, nbad = sm.partition(recs, world)
            send = np.zeros((world, MAX_FOUND, 5), np.uint64)
            for d, g in enumerate(groups):
                send[d, :len(g)] = g
            counts = torch.tensor([len(g) for g in groups] + [nbad], dtype=torch.int32)
            return torch.from_numpy(send.view(np.uint8).reshape(-1)), counts

        ex = DPExchange(None, dist, rank, world, torch, device=torch.device("cpu"), max_found=MAX_FOUND, partition_fn=part)
        counts, cap, recv, nbad = ex.step(len(recs))
        buf = recv.numpy().view(np.uint64).reshape(world, cap, 5)
        got = [buf[s, :counts[s]].copy() for s in range(world)]
        out.append((step, counts, cap, nbad, [g.tobytes() for g in got]))
    q.put((rank, out))
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_exchange_delivers_each_shard_its_records_in_source_order_gloo(world):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_exchange_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for step in range(5):
        per_source = [step_records(step, r, world) for r in range(world)]
        want = sm.arrivals([p[0] for p in per_source], world)
        for d in range(world):
            st, counts, cap, nbad, got = res[d][step]
            assert counts == [len(seg) for seg in want[d]]
            assert got == [seg.tobytes() for seg in want[d]]
            assert nbad == per_source[d][1]
            assert cap % 256 == 0 or cap == MAX_FOUND
            assert cap >= max(len(sm.partition(p[0], world)[0][dd]) for p in per_source for dd in range(world))
