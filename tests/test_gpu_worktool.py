"""-m gpu: the work-file tools on the device (kgx_work_*, python -m kangaroo_b200.worktool): the comb, the check kernel on
crafted entries and kangaroos, check and merge on reference-written files, and a merge of two solver runs that finds the key."""
import json
import os
import random
import shutil
import subprocess
import sys

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200 import worktool as wt
from tests.worktool_util import GOLD, REFBIN, ROOT, Work, crafted_pair, golden, merge_model, tagged

pytestmark = pytest.mark.gpu
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources)")


def key48():
    from tests.golden import make_work_golden as g
    return ec.mul(g.PRIV), g.START, g.PRIV - g.START


def tool(args, timeout=900):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.worktool"] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    return p.returncode, p.stdout + p.stderr


def test_comb_table_is_j_times_16_to_the_w_times_G():
    tab = wt.comb_table()
    for (w, j), pt in tab.items():
        assert pt == ec.mul(j << (4 * w)), (w, j)


def expected_entry(mag, wild, neg, K):
    s = ec.mul(mag)
    if neg:
        s = ec.neg(s)
    return ec.add(s, K) if wild else s


def test_check_kernel_on_crafted_entries():
    pub, start, k = key48()
    K = ec.add(pub, ec.neg(ec.mul(start)))
    rnd = random.Random(7)
    mags = [0, 1, 2, (1 << 126) - 1, k]
    for w in (1, 2, 7, 16, 31):
        mags += [(1 << (4 * w)) - 1, 1 << (4 * w), (1 << (4 * w)) + 1]
    mags += [rnd.getrandbits(126) for _ in range(40)]
    cases = []                                               # (tagged d, x 256-bit or None, entry meant to be wrong)
    for m in mags:
        for wild in (False, True):
            for neg in (False, True):
                cases.append((m, wild, neg))
    recs, hs, want = [], [], []
    for i, (m, wild, neg) in enumerate(cases):
        s = expected_entry(m, wild, neg, K)
        x = s[0] if s is not None else rnd.getrandbits(256)
        bad = s is None or i % 5 == 3                        # every fifth entry gets a wrong x
        if s is not None and i % 5 == 3:
            x ^= 1 << (i % 128)
        d = tagged(m, wild, neg)
        recs.append([x & ((1 << 64) - 1), (x >> 64) & ((1 << 64) - 1), d & ((1 << 64) - 1), d >> 64])
        hs.append((x >> 128) & 0x3FFFF)
        want.append(int(bad))
    # S = +-K: m = k, wild.  +k*G + K = 2K (a doubling, OK); -k*G + K = infinity (wrong)
    i_dbl = cases.index((k, True, False)); i_inf = cases.index((k, True, True))
    assert want[i_inf] == 1 and (want[i_dbl] == 0 or i_dbl % 5 == 3)
    assert expected_entry(k, True, False, K) == ec.add(K, K)
    got = wt.check_records(0, np.array(recs, dtype=np.uint64), hs, pub, start)
    assert got.tolist() == want
    # a bucket one off is wrong too
    hs2 = list(hs); hs2[0] ^= 1
    assert wt.check_records(0, np.array(recs, dtype=np.uint64), hs2, pub, start)[0] == 1


def test_check_kernel_batch_groups_with_one_wrong_entry_each():
    """2500 entries (not a multiple of the 1024 a block takes): in every thread's group of 8 one entry is wrong -- a wrong x,
    a tame entry of magnitude 0 (infinity, left out of the product) or a wrong bucket -- and the others stay OK"""
    pub, start, k = key48()
    K = ec.add(pub, ec.neg(ec.mul(start)))
    n = 2500
    rnd = random.Random(11)
    recs, hs, want = [], [], []
    for i in range(n):
        t = i % 1024
        g, th = divmod(t, 128)
        m = rnd.getrandbits(40) + 1
        wild = bool(i & 1)
        s = expected_entry(m, wild, False, K)
        x, h, bad = s[0], (s[0] >> 128) & 0x3FFFF, 0
        if g == th % 8:                                      # this thread's wrong one
            bad = 1
            kind = th % 3
            if kind == 0:
                x ^= 1 << 70
            elif kind == 1:
                m, wild, x = 0, False, rnd.getrandbits(256)
            else:
                h ^= 0x100
        d = tagged(m, wild)
        recs.append([x & ((1 << 64) - 1), (x >> 64) & ((1 << 64) - 1), d & ((1 << 64) - 1), d >> 64])
        hs.append(h)
        want.append(bad)
    got = wt.check_records(0, np.array(recs, dtype=np.uint64), hs, pub, start)
    assert got.tolist() == want


def test_check_kernel_on_crafted_kangaroos():
    pub, start, k = key48()
    K = ec.add(pub, ec.neg(ec.mul(start)))
    rnd = random.Random(3)
    recs, want = [], []

    def rec(pt, d):
        x, y = pt
        return [(v >> (64 * j)) & ((1 << 64) - 1) for v in (x, y, d) for j in range(4)]
    for i in range(200):
        d = rnd.getrandbits(100) if i % 4 else ec.N - rnd.getrandbits(60) - 1      # some wrapped below zero mod n
        wild = bool(i & 1)
        pt = ec.add(K, ec.mul(d)) if wild else ec.mul(d)
        kind = 2 if wild else 1
        if i % 7 == 3:
            pt = (pt[0], (pt[1] + 1) % ec.P); kind = 0
        recs.append(rec(pt, d)); want.append(kind)
    recs.append(rec(ec.mul(1 << 130), 1 << 130)); want.append(0)                   # magnitude >= 2^128
    recs.append(rec(K, 0)); want.append(2)                                          # wild at distance 0
    recs.append(rec(ec.mul(5), ec.N + 5)); want.append(0)                           # d >= n
    got = wt.check_records(1, np.array(recs, dtype=np.uint64), None, pub, start)
    assert got.tolist() == want


def test_check_reference_fixture_is_all_ok(tmp_path):
    path = golden("ref_work48.work.gz", tmp_path)
    r = wt.check(path, chunk=1000)                                                  # buckets span chunks
    assert r.entries == Work.read(path).entries() and r.wrong_entries == 0
    assert (r.walks, r.walks_tame, r.walks_wild, r.wrong_walks, r.has_walk_count) == (1024, 512, 512, 0, 1)
    rc, out = tool(["check", path])
    assert rc == 0 and "[100.000% OK]" in out and "DP Wrong: 0" in out and "tame OK 512, wild OK 512, wrong 0" in out, out


def test_check_corrupted_fixture_gives_the_reference_count(tmp_path):
    want = json.load(open(os.path.join(GOLD, "merge_golden.json")))["ref_work48_bad_wrong"]
    path = golden("ref_work48_bad.work.gz", tmp_path)
    r = wt.check(path)
    assert r.wrong_entries == want and r.wrong_walks == 0
    assert len(r.wrong_entry_positions) == want and r.wrong_entry_positions == sorted(r.wrong_entry_positions)
    rc, out = tool(["check", path])
    assert rc == 1 and "DP Wrong: %d" % want in out, out
    if os.path.exists(REFBIN):
        ref = subprocess.run([REFBIN, "-t", "2", "-wcheck", path], capture_output=True, text=True, timeout=300).stdout
        assert "DP Wrong: %d" % want in ref


def test_check_refuses_keys_off_the_curve(tmp_path):
    """kgx_work_check's key refusals in their order: the header key first, in a plain or a batch file, and before a damaged
    batch block is reported; then the keys of the batch block"""
    from tests.batch_merge_util import PUBS, work, write_batch
    off = (PUBS[0][0], PUBS[0][1] ^ 2)
    head_off = write_batch(tmp_path / "h.work", work(pub0=off))
    good = write_batch(tmp_path / "g.work", work())
    for name, src in (("hd.work", head_off), ("gd.work", good)):                   # the batch block's footer cut short
        (tmp_path / name).write_bytes(open(src, "rb").read()[:-1])
    cases = [(work(pub0=off).write(str(tmp_path / "p.work")), "key1 does not lie on elliptic curve"),
             (head_off, "key1 does not lie on elliptic curve"),
             (str(tmp_path / "hd.work"), "key1 does not lie on elliptic curve"),
             (str(tmp_path / "gd.work"), "no batch block footer"),
             (write_batch(tmp_path / "b.work", work(), pubs=[PUBS[0], off]), "a key of the batch block does not lie on elliptic curve")]
    for path, match in cases:
        with pytest.raises(ValueError, match=match):
            wt.check(path)
    assert wt.check(good).ok


def solver(args, timeout=900):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    out = p.stdout + p.stderr
    assert p.returncode in (0, 1), out[-3000:]
    return out


@needs_ingest
@pytest.mark.parametrize("table", ["host", "device"])
def test_check_solver_file_with_kangaroos(tmp_path, table):
    work = str(tmp_path / "s.work")
    out = solver([os.path.join(GOLD, "in80.txt"), "--max-steps", "6", "--save-work", work, "--dp", "8", "--grid", "8,32", "--seed", "4",
                  "--save-kangaroos", "--dp-table", table] + (["--dp-table-capacity", "1000000"] if table == "device" else []))
    assert os.path.exists(work), out[-2000:]
    r = wt.check(work)
    assert r.ok and r.entries > 1000 and r.walks == 8 * 32 * 128 and r.walks_tame == r.walks_wild == r.walks // 2


def test_merge_golden_pair_equals_reference_output(tmp_path):
    a, b = golden("ref_work48.work.gz", tmp_path), golden("ref_work48b.work.gz", tmp_path)
    ref = open(golden("ref_merge48.work.gz", tmp_path), "rb").read()
    for block in (0, 300):
        dest = str(tmp_path / ("m%d.work" % block))
        rc, out = tool(["merge", a, b, "-o", dest] + (["--block-entries", str(block)] if block else []))
        assert rc == 0 and "Total f1+f2: DP count 2^" in out and "Dead kangaroo:" in out, out
        assert open(dest, "rb").read() == ref + b"\0" * 8
        assert not os.path.exists(dest + ".tmp")
    r = wt.merge_files([a, b], str(tmp_path / "x.work"), block_entries=300)
    assert r.blocks > 1
    # a bucket of more entries than a block is refused, and nothing is left behind
    ta, tb = Work.read(a).table, Work.read(b).table
    big = max(len(ta[h]) + len(tb[h]) for h in range(1 << 18))
    assert big >= 2
    with pytest.raises(ValueError, match="more than a merge block"):
        wt.merge_files([a, b], str(tmp_path / "y.work"), block_entries=big - 1)
    assert not os.path.exists(str(tmp_path / "y.work"))
    # the reference's own checker accepts the merged file, and its -i loads it
    if os.path.exists(REFBIN):
        chk = subprocess.run([REFBIN, "-t", "2", "-wcheck", str(tmp_path / "m0.work")], capture_output=True, text=True, timeout=300).stdout
        assert "[100.000% OK]" in chk, chk[-1500:]
    r = wt.check(str(tmp_path / "m0.work"))
    assert r.ok and r.walks == 0 and r.has_walk_count == 1
    r = wt.check(golden("ref_merge48.work.gz", tmp_path))
    assert r.ok and r.has_walk_count == 0


def test_merge_five_files_equals_the_model(tmp_path):
    a, b = golden("ref_work48.work.gz", tmp_path), golden("ref_work48b.work.gz", tmp_path)
    m = golden("ref_merge48.work.gz", tmp_path)                                     # no kangaroo count
    wa = Work.read(a)
    empty = Work(wa.dp, wa.start, wa.end, wa.key, 5, 0.5).write(str(tmp_path / "empty.work"))
    dups = Work(wa.dp + 1, wa.start, wa.end, wa.key, 7, 0.25)                       # duplicates and collisions of a's entries
    filled = [h for h in range(1 << 18) if wa.table[h]][:40]
    for i, h in enumerate(filled):
        x, d = wa.table[h][0]
        dups.table[h] = [(x, d if i % 2 else d ^ 0x5)]
        dups.maxitem[h] = 4
    dups = dups.write(str(tmp_path / "dups.work"))
    paths = [m, dups, empty, b, a]
    want, dup, coll = merge_model([Work.read(p) for p in paths])
    for block in (0, 257):
        dest = str(tmp_path / ("five%d.work" % block))
        r = wt.merge_files(paths, dest, block_entries=block)
        assert open(dest, "rb").read() == want.to_bytes()
        assert (r.entries, r.duplicates, r.collisions) == (want.entries(), dup, len(coll))
        assert [(h, d1[0] | d1[1] << 64, d2[0] | d2[1] << 64) for h, d1, d2 in r.collision_list] == coll
    assert dup > 0 and len(coll) >= 20
    if os.path.exists(REFBIN):                                                      # -wmdir over the same files
        d = tmp_path / "d"
        os.mkdir(d)
        for p in paths:
            shutil.copy(p, d / os.path.basename(p))
        order = wt.dir_inputs(str(d))
        assert len({os.path.getsize(p) for p in order}) == 5
        out = str(tmp_path / "ref_dir.work")
        subprocess.run([REFBIN, "-wmdir", str(d), out], capture_output=True, text=True, timeout=300)
        dest = str(tmp_path / "tool_dir.work")
        rc, txt = tool(["merge", "--dir", str(d), "-o", dest])
        assert rc == 0, txt
        assert open(dest, "rb").read() == open(out, "rb").read() + b"\0" * 8


def test_merge_refuses_bad_inputs_on_the_device(tmp_path):
    """kgx_work_merge's own checks (the tool checks first; callers of the C ABI rely on these)"""
    pa, pb = crafted_pair(tmp_path)
    w = Work.read(pb)
    w.key = (w.key[0], w.key[1] ^ 2)
    off = w.write(str(tmp_path / "off.work"))
    with pytest.raises(ValueError, match="does not lie on elliptic curve"):
        wt.merge_files([pa, off], str(tmp_path / "o.work"))
    w = Work.read(pb); w.end += 1
    with pytest.raises(ValueError, match="range differs"):
        wt.merge_files([pa, w.write(str(tmp_path / "r.work"))], str(tmp_path / "o.work"))
    w.key = (w.key[0], w.key[1] ^ 2)                                                # off the curve and another range: the curve first
    with pytest.raises(ValueError, match="does not lie on elliptic curve"):
        wt.merge_files([pa, w.write(str(tmp_path / "cr.work"))], str(tmp_path / "o.work"))
    assert not os.path.exists(str(tmp_path / "o.work"))


@needs_ingest
def test_merge_of_the_crafted_pair_finds_the_key(tmp_path):
    from tests.golden import make_work_golden as g
    pa, pb = crafted_pair(tmp_path)
    dest = str(tmp_path / "found.work")
    rc, out = tool(["merge", pa, pb, "-o", dest])
    assert rc == 0 and "Priv: 0x%X" % g.PRIV in out, out
    assert not os.path.exists(dest) and not os.path.exists(dest + ".tmp")


@needs_ingest
@pytest.mark.parametrize("table", ["host", "device"])
def test_two_solver_runs_merged_find_the_key(tmp_path, table):
    """two runs of the in56 key with different seeds, each stopped early; their merge is all OK and either finds the key or is
    resumed by the solver, which finds it"""
    cfg = os.path.join(GOLD, "in56.txt")
    _, _, pubs = ec.parse_config(cfg)
    a, b = str(tmp_path / "a.work"), str(tmp_path / "b.work")
    common = ["--dp", "10", "--grid", "32,128", "--dp-table", table]
    solver([cfg, "--max-steps", "40", "--seed", "1", "--save-work", a] + common)
    solver([cfg, "--max-steps", "30", "--seed", "2", "--save-work", b] + common)
    if not (os.path.exists(a) and os.path.exists(b)):
        pytest.skip("a run found the key before saving")
    dest = str(tmp_path / "m.work")
    rc, out = tool(["merge", a, b, "-o", dest])
    assert rc == 0, out
    if "Priv:" in out:
        assert not os.path.exists(dest)
        return
    r = wt.check(dest)
    assert r.ok and r.entries > 0 and r.walks == 0
    out = solver(["--resume", dest, "--seed", "3", "--max-steps", "100000"] + common)
    assert "Priv: 0x" in out, out[-2000:]
    priv = int(out.split("Priv: 0x")[1].split()[0], 16)
    assert ec.mul(priv) == pubs[0]
