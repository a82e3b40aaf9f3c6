"""A plain model of the sharded DP table's data plane (--dp-table sharded): which rank owns a bucket, the stable partition of
one rank's 40-byte DP records by owner (kgx_dp_partition), and the order in which a shard receives every rank's records
(dist.DPExchange: source rank, then record order)."""
import numpy as np

NB = 1 << 18


def owner_bounds(world):
    """the first bucket of every rank, then 2^18: rank r owns [floor(r*2^18/W), floor((r+1)*2^18/W))"""
    return [r * NB // world for r in range(world + 1)]


def owners(h, world):
    """the owner of every bucket h (uint64 array, all below 2^18), found by search in the bounds"""
    return np.searchsorted(np.asarray(owner_bounds(world)[1:], np.uint64), np.asarray(h, np.uint64), side="right")


def partition(recs, world):
    """(n, 5) uint64 records -> ([records of owner r, in input order] for every r, malformed records (h >= 2^18))"""
    recs = np.asarray(recs, np.uint64).reshape(-1, 5)
    h = recs[:, 0] >> np.uint64(32)
    good = h < np.uint64(NB)
    own = np.full(len(recs), world, np.int64)
    own[good] = owners(h[good], world)
    return [recs[own == r] for r in range(world)], int((~good).sum())


def arrivals(per_source, world):
    """per_source[s] = rank s's records of one step -> the segments every shard receives: shard d gets, for each source s in
    order, the records of s it owns, in s's order"""
    parts = [partition(p, world)[0] for p in per_source]
    return [[parts[s][d] for s in range(len(per_source))] for d in range(world)]
