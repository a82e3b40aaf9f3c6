"""Shared helpers of the batch merge tests: small batch work files on the 64-key 2^56 fixture, written in Python (a HEADW
table from tests.worktool_util.Work, no kangaroo, then the batch block of kgx_batch_block)."""
import os

from kangaroo_b200 import ecmath as ec
from kangaroo_b200.worktool import BatchBlock, batch_block
from tests.worktool_util import Work, tagged

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CFG64 = os.path.join(GOLD, "in56_64keys.txt")
START, END, PUBS = ec.parse_config(CFG64)
ANSWERS = [int(v, 16) for v in open(os.path.join(GOLD, "in56_64keys.answers.txt")).read().split()]


def collision_pair(a, b, j, d_t=0x1234567):
    """a tame entry in Work a and a wild entry of key j in Work b at the same point d_t*G, with d_t counted from k_j"""
    k = ANSWERS[j] - START
    t = k + d_t
    a.add(ec.mul(t)[0], tagged(t, False))
    b.add(ec.mul(t)[0], tagged(d_t, True))


def work(dp=8, start=START, end=END, count=100, time=1.0, tame=(), pub0=None):
    w = Work(dp, start, end, pub0 or PUBS[0], count, time)
    for d in tame:
        w.add(ec.mul(d)[0], tagged(d, False))
    return w


def write_batch(path, w, pubs=None, solved=(), privs=None):
    """w's bytes with a kangaroo count of 0, then a batch block of pubs (default: the fixture's 64 keys) with the keys of
    `solved` solved at privs (default: the fixture's answers)"""
    pubs = PUBS if pubs is None else pubs
    privs = ANSWERS if privs is None else privs
    raw = w.to_bytes(walk_count=True)
    flags = [i in solved for i in range(len(pubs))]
    blk = BatchBlock(pubs, flags, [privs[i] if f else None for i, f in enumerate(flags)], [], len(raw))
    with open(path, "wb") as f:
        f.write(raw)
        f.write(batch_block(blk, len(raw)).tobytes())
    return str(path)


def refusal_inputs(tmp_path, what):
    """two inputs that kgx_work_merge_batch refuses, and the message it gives"""
    a = write_batch(tmp_path / "a.work", work(tame=(11, 22)), solved=(1,))
    if what == "order":
        pubs = list(PUBS)
        pubs[3], pubs[4] = pubs[4], pubs[3]
        privs = list(ANSWERS)
        privs[3], privs[4] = privs[4], privs[3]
        return [a, write_batch(tmp_path / "b.work", work(tame=(33,)), pubs=pubs, privs=privs)], "key lists differ"
    if what == "fewer":
        return [a, write_batch(tmp_path / "b.work", work(tame=(33,)), pubs=PUBS[:63])], "key lists differ"
    if what == "plain":
        return [a, work(tame=(33,)).write(str(tmp_path / "b.work"))], "plain HEADW"
    if what == "range":
        return [a, write_batch(tmp_path / "b.work", work(end=END + 1, tame=(33,)))], "range differs"
    if what == "range+fewer":                             # two faults in one input: the range is refused first
        return [a, write_batch(tmp_path / "b.work", work(end=END + 1, tame=(33,)), pubs=PUBS[:63])], "range differs"
    if what == "conflict":
        privs = list(ANSWERS)
        privs[1] = (2 * START - ANSWERS[1]) % ec.N
        return [a, write_batch(tmp_path / "b.work", work(tame=(33,)), solved=(1,), privs=privs)], "different private keys"
    if what == "tampered":
        privs = list(ANSWERS)
        privs[7] += 1
        return [a, write_batch(tmp_path / "b.work", work(tame=(33,)), solved=(7,), privs=privs)], "does not give its public key"
    raise ValueError(what)


CPU_REFUSALS = ["order", "fewer", "plain", "range", "range+fewer", "conflict"]
