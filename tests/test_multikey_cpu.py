"""CPU: the host side of the solver's --batch-keys (one tame herd shared by every key of the input): the argument checks, the
rule that spreads the wild kangaroos over the unsolved keys and moves them on when a key is solved, and kgi_resolve_multi,
which finds the key of a tame/wild collision among many."""
import os

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200.solver import assign_targets, class_privs, key_classes, main, retarget_targets
from oracle import kgo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
M64 = (1 << 64) - 1


@pytest.mark.parametrize("extra", [["--save-work", "w.work"], ["--save-interval", "5"], ["--save-kangaroos"], ["--resume", "w.work"]])
def test_batch_keys_refuses_work_files(extra, capsys):
    with pytest.raises(SystemExit) as e:
        main([os.path.join(GOLD, "in56_64keys.txt"), "--batch-keys"] + extra)
    assert e.value.code == 2
    assert "--batch-keys cannot be combined" in capsys.readouterr().err


def test_batch_keys_needs_a_config_with_keys(tmp_path, capsys):
    with pytest.raises(SystemExit):
        main(["--batch-keys"])
    cfg = tmp_path / "nokeys.txt"
    cfg.write_text("1000\n2000\n")
    with pytest.raises(SystemExit) as e:
        main([str(cfg), "--batch-keys"])
    assert e.value.code == 2
    assert "at least one public key" in capsys.readouterr().err


def test_batch_keys_refuses_more_keys_than_the_engine_takes(tmp_path, capsys):
    cfg = tmp_path / "many.txt"
    cfg.write_text("1000\n2000\n" + ("04%064X%064X\n" % ec.G) * 65536)
    with pytest.raises(SystemExit) as e:
        main([str(cfg), "--batch-keys"])
    assert e.value.code == 2
    assert "at most 65535 keys" in capsys.readouterr().err


def test_equal_and_opposite_keys_share_one_search():
    """keyToSearch = priv*G - start*G: a key listed twice is one search, and so is a key whose keyToSearch is the negative of
    another's (priv' = 2*start - priv); the first of each class in input order is searched"""
    start = 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD00000000000000
    privs = [start + 0x123456789, start + 0xABCDEF, start + 0x123456789, (2 * start - (start + 0xABCDEF)) % ec.N, start,
             start + 0x555]
    keys = [ec.add(ec.mul(p), ec.neg(ec.mul(start))) for p in privs]
    assert keys[4] is None
    rep, neg = key_classes(keys)
    assert rep == [0, 1, 0, 1, 4, 5] and neg == [False, False, False, True, False, False]
    for i in range(len(privs)):
        if keys[i] is not None:
            assert class_privs(start, privs[rep[i]], neg[i]) == privs[i]


def test_class_members_claim_the_same_keys_as_a_scan_at_65535_keys():
    """BatchSolver._claim gives every key of a solved class its private key through class_members, built once, in place of a
    scan over all keys per class.  At 65535 keys, with keys listed twice, three times and negated mixed in (points stand in as
    (x, y) pairs: key_classes looks only at x and y), both give the same private keys for every class."""
    from kangaroo_b200.solver import BatchSolver, class_members
    n, p = 65535, ec.P
    rng = np.random.default_rng(11)
    xs = [int(v) for v in rng.integers(1, 1 << 62, size=n)]
    keys = [(x, x + 1) for x in xs]
    for i in range(300, n, 257):                                         # a copy of an earlier key, or its negative
        j = int(rng.integers(0, i))
        keys[i] = keys[j] if i % 2 else (keys[j][0], p - keys[j][1])
    keys[n - 1] = keys[n - 2] = (keys[5][0], p - keys[5][1])             # one class across the whole input
    keys[4000] = None                                                     # the point at infinity: a class of its own
    rep, neg = key_classes(keys)
    members = class_members(rep)
    assert sorted(i for m in members.values() for i in m) == list(range(n))
    assert all(rep[i] == r for r, m in members.items() for i in m) and all(m == sorted(m) for m in members.values())
    multi = [r for r, m in members.items() if len(m) > 1]
    assert len(multi) > 100 and any(neg[i] for r in multi for i in members[r]) and members[5] == [5, n - 2, n - 1]

    start = 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD00000000000000
    s = BatchSolver.__new__(BatchSolver)                                 # _claim's state only: no engine
    s.start, s.rep, s.neg, s.members = start, rep, neg, members
    s.priv, s._announce = [None] * n, []
    hits = [(i, start + 1000 + i, 0, 2 * i + 1) for i in range(n)]       # a hit on every key, its class solved by the first
    resets = []
    s._claim(hits, resets)
    assert s._announce == sorted(members) and len(resets) == n - len(members)
    scan, rep_a = [None] * n, np.asarray(rep)                            # the scan over all keys, per class
    for r in multi + [int(v) for v in rng.choice(sorted(members), 40, replace=False)]:
        scan[r] = start + 1000 + r
        for i in np.flatnonzero(rep_a == r).tolist():
            scan[i] = class_privs(start, scan[r], neg[i])
        assert [s.priv[i] for i in members[r]] == [scan[i] for i in members[r]], r
    assert s.priv[n - 1] == (2 * start - (start + 1005)) % ec.N


def test_wilds_are_spread_evenly_over_the_live_keys():
    for n, live in [(2 * 4096, list(range(64))), (12288, [0, 3, 4, 9, 10]), (1000, [7]), (130, list(range(100)))]:
        t = assign_targets(n, live)
        wild = np.arange(n) % 2 == 1
        assert t.dtype == np.uint16 and np.all(t[~wild] == 0)
        counts = np.bincount(t[wild], minlength=max(live) + 1)
        nw = int(wild.sum())
        assert set(np.flatnonzero(counts)) <= set(live)
        assert all(counts[k] in (nw // len(live), -(-nw // len(live))) for k in live), (n, live)


def test_moved_wilds_never_land_on_a_solved_key():
    n, K = 3 * 32 * 128, 64
    live = list(range(K))
    t = assign_targets(n, live)
    rng = np.random.default_rng(5)
    kidx = np.arange(n)
    wild = kidx % 2 == 1
    while len(live) > 1:
        frm = int(rng.choice(live))
        live.remove(frm)
        new = retarget_targets(t, frm, live)
        moved = wild & (t == frm)
        assert moved.any()
        assert np.array_equal(new[~moved], t[~moved])                     # nothing else moves, tame kangaroos least of all
        assert np.array_equal(new[moved], np.asarray(live)[(kidx[moved] >> 1) % len(live)])   # kgx_retarget's rule
        assert not np.isin(new[wild], [k for k in range(K) if k not in live]).any()
        counts = np.bincount(new[wild], minlength=K)[live]
        assert counts.min() > 0 and counts.max() <= 2 * counts.min() + 2  # still spread over every live key
        t = new
    assert np.all(t[wild] == live[0])


# ---- kgi_resolve_multi --------------------------------------------------------------------------------------------------
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")


def tagged(oracle, x, d, ktype):
    _, _, D = oracle.hash_convert(x, d % kgo.N, ktype)
    return D & M64, D >> 64


def signed_mod(v):
    v %= kgo.N
    return v - kgo.N if v > kgo.N // 2 else v


@needs_ingest
def test_resolve_multi_finds_the_key_among_64(oracle):
    from kangaroo_b200.ingest import DPTable
    start = 0x49DCCFD96DC5DF56487436F5A1B18C4F5D34F65DDB48CB5E0000000000000000
    rng = np.random.default_rng(64)
    ks = [int(rng.integers(1, 1 << 62)) for _ in range(64)]                        # keyToSearch = k*G, priv = start + k
    keys = [oracle.ec_mul_g(k) for k in ks]
    table = DPTable.key_table(keys)
    t = DPTable(threads=1)
    cases = 0
    for idx in (0, 1, 31, 62, 63):
        k = ks[idx]
        for ctype in range(4):
            for sign in (1, -1):
                # CheckKey's candidate `ctype` is (+-Td) + (+-Wd); make it sign * k, i.e. key or -key
                td = int(rng.integers(1, 1 << 61))
                s1 = -1 if ctype & 1 else 1
                s2 = -1 if ctype & 2 else 1
                wd = signed_mod(s2 * (sign * k - s1 * td))
                assert (s1 * td + s2 * wd - sign * k) % kgo.N == 0
                tame = oracle.ec_mul_g(td % kgo.N)
                wild = oracle.ec_add(keys[idx], oracle.ec_mul_g(wd % kgo.N))
                # the four cases a walk makes (wild = +-tame) have the same x; the others exercise the algebra alone
                assert (tame[0] == wild[0]) == (sign == (1 if ctype >= 2 else -1))
                dt, dw = tagged(oracle, tame[0], td, 0), tagged(oracle, tame[0], wd, 1)
                for d_old, d_new in ((dt, dw), (dw, dt)):                           # either side may be the stored entry
                    got = t.resolve_multi(d_old, d_new, table, start)
                    assert got == (idx, start + k), (idx, ctype, sign)
                    assert oracle.ec_mul_g(got[1] - start) == keys[idx]
                    assert t.resolve(d_old, d_new, keys[idx], start) == got[1]
                    assert t.resolve_multi(d_old, d_new, keys, start) == got       # a list of points works the same
                cases += 1
    assert cases == 40
    # a pair that matches none of the keys, and two kangaroos of one herd
    td, wd = int(rng.integers(1, 1 << 61)), int(rng.integers(1, 1 << 61))
    x = oracle.ec_mul_g(td)[0]
    assert t.resolve_multi(tagged(oracle, x, td, 0), tagged(oracle, x, wd, 1), table, start) is None
    assert t.resolve_multi(tagged(oracle, x, td, 0), tagged(oracle, x, wd, 0), table, start) is None
    # the first matching key wins when the table lists a key twice
    dup = DPTable.key_table([keys[5]] + keys)
    k = ks[5]
    td = 12345
    wd = td - k
    x = oracle.ec_mul_g(td)[0]
    assert t.resolve_multi(tagged(oracle, x, td, 0), tagged(oracle, x, wd, 1), dup, start) == (0, start + k)
    t.close()


def test_key_table_of_the_point_at_infinity():
    from kangaroo_b200.ingest import DPTable
    kt = DPTable.key_table([None, ec.G])
    assert kt.shape == (2, 8) and kt.dtype == np.uint64 and not kt[0].any()
    assert [int(v) for v in kt[1]] == [(ec.G[c] >> (64 * w)) & M64 for c in (0, 1) for w in range(4)]
