"""-m gpu: merging batch work files (kgx_work_merge_batch, `worktool merge` on --batch-save files): the device resolver
against the host's kgi_resolve_multi at 1, 64 and 65535 keys, the merged table against kgx_work_merge, the solved keys of
the inputs and of the merge, the refusals, --batch-resume of the merged file and merge --dir."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200 import worktool as wt
from tests.batch_merge_util import ANSWERS, CFG64, PUBS, START, collision_pair, refusal_inputs, work, write_batch
from tests.worktool_util import TYPE_BIT

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")
GRID = ["--dp", "8", "--grid", "32,128"]
M126 = (1 << 126) - 1
SIGN = 1 << 127


def solver(args, timeout=900):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    return p.returncode, p.stdout + p.stderr


def tool(args, timeout=900):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.worktool"] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    return p.returncode, p.stdout + p.stderr


def privs(out):
    return {int(i): int(v, 16) for i, v in re.findall(r"Key#\s*(\d+) Pub:\s+0x[0-9A-F]+\s+Priv: 0x([0-9A-F]+)", out)}


# ---- the resolver --------------------------------------------------------------------------------------------------------
def key_table(n, rng):
    """n keys K = k*G with known scalars: 64 random ones below 2^124, then consecutive ones (one point addition each); among
    them key 3 listed again at 9, the negative of key 4 at 10, one at infinity (None) at 11, one with k = 2^126 + 5 (above any
    single |d|) at 12 and, past 64 keys, key 5 again as the last key"""
    ks = [int(rng.integers(1, 1 << 62)) << 62 | int(rng.integers(0, 1 << 62)) for _ in range(min(n, 64))]
    pts = [ec.mul(k) for k in ks]
    if n > 64:
        k, p = int(rng.integers(1, 1 << 62)) << 60, None
        p = ec.mul(k)
        for i in range(64, n):
            ks.append(k + i - 64)
            pts.append(p)
            p = ec.add(p, ec.G)
        ks[n - 1], pts[n - 1] = ks[5], pts[5]
    if n >= 64:
        ks[9], pts[9] = ks[3], pts[3]
        ks[10], pts[10] = ec.N - ks[4], ec.neg(pts[4])
        ks[11], pts[11] = 0, None
        ks[12], pts[12] = (1 << 126) + 5, ec.mul((1 << 126) + 5)
    return ks, pts


def collisions(ks, rng):
    """(d_first, d_other) pairs: for keys at the start, the end and the special indices, tame = k + w with the wild |w| random,
    at 0 and at 2^126 - 1 - k, in all four sign combinations and both orders; then m2 = 0, m1 carrying into bit 126, same-herd
    pairs and pairs of random magnitudes"""
    n = len(ks)
    idx = sorted({0, n - 1} | ({3, 4, 5, 9, 10, 11, 12, 63} if n >= 64 else set()) | set(rng.integers(0, n, 8).tolist()))
    out = []

    def pair(t, w):
        for st in (0, SIGN):
            for sw in (0, SIGN):
                a, b = t | st, w | TYPE_BIT | sw
                out.extend([(a, b), (b, a)])

    for j in idx:
        k = ks[j]
        if k >= 1 << 125:                                  # keys 10 and 12
            continue
        for w in (int(rng.integers(0, 1 << 62)) << 60, 0, M126 - k):
            pair(k + w, w)
    t = int(rng.integers(1, 1 << 62)) << 62
    pair(t, t)                                             # m2 = 0: the key at infinity, if any
    pair(0, 0)                                             # m1 = m2 = 0
    pair(M126, M126)
    pair(M126, M126 - 1)                                   # m1 = 2^127 - 3
    pair((1 << 125) + 3, (1 << 125) + 2)                   # m1 = 2^126 + 5: key 12
    for _ in range(16):
        pair(int(rng.integers(0, 1 << 62)) << 64 | int(rng.integers(0, 1 << 62)), int(rng.integers(0, 1 << 62)) << 64)
    for a, b in ((5, 7), (5 | SIGN, 7 | SIGN)):
        out.extend([(a, b), (a | TYPE_BIT, b | TYPE_BIT)])
    return out


@needs_ingest
@pytest.mark.parametrize("n", [1, 64, 65535])
def test_resolver_equals_the_host_resolver(n):
    from kangaroo_b200.ingest import DPTable
    rng = np.random.default_rng(n)
    ks, pts = key_table(n, rng)
    coll = collisions(ks, rng)
    t = DPTable(threads=1)
    kt = DPTable.key_table(pts)
    limbs = lambda v: (v & 0xFFFFFFFFFFFFFFFF, v >> 64)
    try:
        for start in (START, ec.N - 3, 0):
            got = wt.resolve([c[0] for c in coll], [c[1] for c in coll], pts, start)
            want = [t.resolve_multi(limbs(a), limbs(b), kt, start) for a, b in coll]
            assert got == want
            hits = [g for g in got if g is not None]
            assert len(hits) >= 24
            for i, priv in hits:
                assert (priv - start) % ec.N == ks[i] % ec.N
            if n >= 64:
                found = {i for i, _ in hits}
                assert found >= {0, 3, 4, 5, 11, 12, 63}
                assert not found & {9, 10, n - 1 if n > 64 else 9}                 # listed after the same point or its negative
    finally:
        t.close()
    with pytest.raises(ValueError, match="not below n"):
        wt.resolve([0], [TYPE_BIT], pts, ec.N)


# ---- merges of solver-written files --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """two short --batch-keys --batch-save runs of the 64-key 2^56 fixture with different seeds"""
    d = tmp_path_factory.mktemp("runs")
    paths = []
    for seed in (3, 4):
        p = str(d / ("run%d.work" % seed))
        rc, out = solver([CFG64, "--batch-keys", "--seed", str(seed), "--max-steps", "40", "--batch-save", p] + GRID)
        assert os.path.exists(p), out[-3000:]
        paths.append(p)
    return paths


def headw_part(path, dest):
    b = wt.read_batch(path)
    with open(path, "rb") as f, open(dest, "wb") as g:
        g.write(f.read(b.offset))
    return dest


@needs_ingest
def test_merged_table_is_the_single_key_merge_of_the_headw_parts(runs, tmp_path):
    dest = str(tmp_path / "m.work")
    rc, out = tool(["merge"] + runs + ["-o", dest])
    assert rc == 0, out[-3000:]
    plain = [headw_part(p, str(tmp_path / ("p%d.work" % i))) for i, p in enumerate(runs)]
    ref = str(tmp_path / "ref.work")
    r = wt.merge_files(plain, ref)
    want = open(ref, "rb").read()
    got = open(dest, "rb").read()
    assert got[:len(want)] == want
    b = wt.read_batch(dest)
    assert b.offset == len(want) and b.nb_walk == 0 and b.pubs == PUBS
    blocks = [wt.read_batch(p) for p in runs]
    for i in range(64):
        if any(x.solved[i] for x in blocks):
            assert b.solved[i] and b.privs[i] == ANSWERS[i]
        if b.solved[i]:
            assert b.privs[i] == ANSWERS[i]
    c = wt.check(dest)
    assert c.ok and c.n_keys == 64 and c.walks == 0 and c.entries == r.entries
    rc, out = tool(["check", dest])
    assert rc == 0 and "[100.000% OK]" in out and "64 keys" in out, out
    res = wt.merge_batch_files(runs, str(tmp_path / "again.work"))
    assert res.collisions == r.collisions == res.same_herd + res.no_key + res.already_solved + res.solving
    assert res.n_listed == 0 and res.solved_in_inputs + res.solved_by_merge + res.left == 64
    assert open(str(tmp_path / "again.work"), "rb").read() == got


def test_solved_keys_of_both_inputs_are_kept(tmp_path):
    """a holds keys {1, 3} solved, b {3, 5}; a collision on key 3 changes nothing, one on key 9 solves it"""
    a, b = work(tame=(11, 22, 33)), work(tame=(44, 55))
    collision_pair(a, b, 3, d_t=0x555)
    collision_pair(b, a, 9)
    pa = write_batch(tmp_path / "a.work", a, solved=(1, 3))
    pb = write_batch(tmp_path / "b.work", b, solved=(3, 5))
    res = wt.merge_batch_files([pa, pb], str(tmp_path / "m.work"))
    out = wt.read_batch(str(tmp_path / "m.work"))
    for i in (1, 3, 5):
        assert res.status[i] == 1 and out.solved[i] and out.privs[i] == ANSWERS[i]
    assert res.status[9] == 2 and res.privs[9] == ANSWERS[9]
    assert (res.solved_in_inputs, res.solved_by_merge, res.left, res.already_solved, res.solving) == (3, 1, 60, 1, 1)
    assert [i for i in range(64) if out.solved[i]] == [1, 3, 5, 9]
    assert [out.privs[i] for i in (1, 3, 5, 9)] == [ANSWERS[i] for i in (1, 3, 5, 9)]


def test_the_merge_finds_a_key_and_leaves_solved_ones_alone(tmp_path):
    a, b = work(tame=(11, 22, 33)), work(dp=10, count=200, time=2.0, tame=(44,))
    collision_pair(a, b, 6)                                # key 6: unsolved in both
    collision_pair(a, b, 2, d_t=0x777)                     # key 2: solved in a
    collision_pair(b, a, 40, d_t=0x999)                    # key 40: wild in a, tame in b
    pa = write_batch(tmp_path / "a.work", a, solved=(2,))
    pb = write_batch(tmp_path / "b.work", b)
    dest = str(tmp_path / "m.work")
    rc, out = tool(["merge", pa, pb, "-o", dest])
    assert rc == 0, out
    assert privs(out) == {6: ANSWERS[6], 40: ANSWERS[40]}, out
    assert "2 solved by the merge" in out and "1 solved in the inputs" in out
    blk = wt.read_batch(dest)
    assert [i for i in range(64) if blk.solved[i]] == [2, 6, 40]
    assert [blk.privs[i] for i in (2, 6, 40)] == [ANSWERS[2], ANSWERS[6], ANSWERS[40]]
    res = wt.merge_batch_files([pa, pb], str(tmp_path / "again.work"))
    assert (res.collisions, res.solving, res.already_solved, res.no_key, res.same_herd) == (3, 2, 1, 0, 0)
    h, d1, d2 = res.solved_by[6]
    assert d2 == (0x1234567 | TYPE_BIT) and d1 == ANSWERS[6] - START + 0x1234567
    assert res.status[2] == 1 and res.solved_by[2] is None
    assert wt.check(dest).ok


@pytest.mark.parametrize("what", ["order", "fewer", "plain", "range", "range+fewer", "conflict", "tampered"])
def test_refusals_on_the_device_write_nothing(tmp_path, what):
    inputs, match = refusal_inputs(tmp_path, what)
    tmp = str(tmp_path / "m.work.tmp")
    for order in (inputs, inputs[::-1])[:1 if what == "plain" else 2]:     # a plain file first is refused by read_batch
        with pytest.raises(ValueError, match=match):
            wt.merge_batch_files(order, tmp)
        assert not os.path.exists(tmp)
    dest = str(tmp_path / "m.work")
    assert wt.main(["merge"] + inputs + ["-o", dest]) == 2
    assert not os.path.exists(dest) and not os.path.exists(dest + ".tmp")


@needs_ingest
def test_batch_resume_of_the_merged_file_solves_the_rest(runs, tmp_path):
    dest = str(tmp_path / "m.work")
    rc, out = tool(["merge"] + runs + ["-o", dest])
    assert rc == 0, out[-3000:]
    b = wt.read_batch(dest)
    rc, out = solver(["--batch-keys", "--batch-resume", dest, "--seed", "9", "--grid", "32,128"])
    assert rc == 0, out[-3000:]
    assert "%d of 64 keys solved in the file" % sum(b.solved) in out, out[-3000:]
    assert privs(out) == dict(enumerate(ANSWERS)), out[-3000:]


def test_merge_dir_equals_the_explicit_list(tmp_path):
    """three batch files of different sizes; the tame and the wild entry of key 6 sit in two of them, so the order decides
    which entry the table keeps"""
    d = tmp_path / "d"
    d.mkdir()
    big, mid, small = work(tame=range(100, 112)), work(tame=range(200, 205)), work(tame=(300,))
    collision_pair(small, big, 6)
    write_batch(d / "big.work", big, solved=(2,))
    write_batch(d / "mid.work", mid, solved=(2, 4))
    write_batch(d / "small.work", small)
    files = wt.dir_inputs(str(d))
    assert [os.path.basename(f) for f in files] == ["big.work", "mid.work", "small.work"]
    rc, out = tool(["merge", "--dir", str(d), "-o", str(tmp_path / "dir.work")])
    assert rc == 0, out[-3000:]
    assert privs(out) == {6: ANSWERS[6]}, out
    rc, out = tool(["merge"] + files + ["-o", str(tmp_path / "list.work")])
    assert rc == 0, out[-3000:]
    got = open(str(tmp_path / "dir.work"), "rb").read()
    assert got == open(str(tmp_path / "list.work"), "rb").read()
    rc, out = tool(["merge"] + files[::-1] + ["-o", str(tmp_path / "rev.work")])
    assert rc == 0, out[-3000:]
    assert open(str(tmp_path / "rev.work"), "rb").read() != got
    blk = wt.read_batch(str(tmp_path / "dir.work"))
    assert [i for i in range(64) if blk.solved[i]] == [2, 4, 6]
