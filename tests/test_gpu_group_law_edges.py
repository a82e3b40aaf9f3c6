"""-m gpu: the group law and the mod-n edges where the multi-key and checkpoint code call it, at the points and distances that
random herds and solver-written files never produce (inputs and model: tests/group_law_model.py):
  - the batch work-file check (wt_check_entries_multi_kernel, the tg path of wt_check_walks_kernel) against the model, and a
    one-key batch file against the single-key check, on keys at infinity, equal and opposite keys, S = +-K, |d| = 0;
  - kgx_retarget where the moved point equals the difference of the keys or its negative, and where that difference is a
    doubling, on every kernel;
  - herd_import_kernel / herd_export_kernel at n - 1, n, n + 1, 2^128 - 1, 2^128 and the wild offset +-1."""
import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200 import worktool as wt
from tests import group_law_model as gm

pytestmark = pytest.mark.gpu
N = gm.N


def limbs(v, n):
    return [(v >> (64 * k)) & gm.M64 for k in range(n)]


def ints(a):
    return [sum(int(r[k]) << (64 * k) for k in range(a.shape[1])) for r in a]


def chunk_for(n):
    """a check chunk that does not divide n records and gives an odd number of chunks, at least 3.  The check alternates two
    buffers, so the last chunk then sits in the first buffer and the one before it in the second: the wrong records of both
    must still come out in file order."""
    return next(c for c in range(max(2, n // 7), n) if n % c and (-(-n // c)) % 2 == 1)


def classes_at(w, positions, entries):
    """the crafted classes of the entries at (bucket, index) positions, for a failure message"""
    by = {}
    for e in entries:
        by.setdefault((e.h, e.x, e.d), set()).add(e.cls)
    return sorted({c for h, i in positions for c in by[(h, *w.table[h][i])]})


# ---- A. the batch work-file check -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_keys", [1, 7, 8, 9, 17])
def test_batch_check_of_crafted_entries_equals_the_model(tmp_path, n_keys):
    kk = gm.key_scalars(n_keys)
    keys = [gm.key_point(k) for k in kk]
    ents = gm.batch_entries(kk)
    w = gm.work_of(ents, gm.pub_of(kk[0]))
    path = tmp_path / "b.work"
    path.write_bytes(gm.file_bytes(w, kk))
    n = w.entries()
    want = gm.wrong_positions(w, keys)
    r = wt.check(str(path), chunk=chunk_for(n), cap=n)
    assert r.n_keys == n_keys and r.entries == n and r.walks == 0
    got = r.wrong_entry_positions
    assert got == want, "wrong only on the device: %s; wrong only in the model: %s" % (
        classes_at(w, sorted(set(got) - set(want)), ents), classes_at(w, sorted(set(want) - set(got)), ents))
    assert r.wrong_entries == len(want) and 0 < len(want) < n
    r = wt.check(str(path), chunk=chunk_for(n), cap=len(want) - 1)                  # the first cap of them
    assert r.wrong_entry_positions == want[:-1] and r.wrong_entries == len(want)


def test_one_key_batch_file_is_the_single_key_check(tmp_path):
    """for every key of the 17 (one at infinity, two equal, two opposite): the entries in a one-key batch file, in the same file
    without its block and through kgx_work_check_records with that key give the model's wrong entries"""
    kk = gm.key_scalars(17)
    ents = gm.batch_entries(kk)
    recs = np.array([limbs(e.x, 2) + limbs(e.d, 2) for e in ents], dtype=np.uint64)
    hs = [e.h for e in ents]
    w = gm.work_of(ents, gm.pub_of(kk[0]))
    n = w.entries()
    chunk = chunk_for(n)
    body = gm.file_bytes(w, [kk[0]], block=False)[len(w.header_bytes()):]   # the table and a kangaroo count of 0
    for k, sk in enumerate(kk):
        K = [gm.key_point(sk)]
        pub = gm.pub_of(sk)
        assert (sk == 0) == (pub == ec.mul(gm.START))
        single = wt.check_records(0, recs, hs, pub, gm.START)
        assert single.tolist() == [int(not gm.entry_ok(e.h, e.x, e.d, K)) for e in ents], k
        w.key = pub
        plain = w.header_bytes() + body
        want = gm.wrong_positions(w, K)
        got = []
        for block in (True, False):
            path = tmp_path / ("k%d_%d.work" % (k, block))
            blk = wt.batch_block(wt.BatchBlock([pub], [False], [None], []), len(plain)).tobytes() if block else b""
            path.write_bytes(plain + blk)
            r = wt.check(str(path), chunk=chunk, cap=n)
            assert r.n_keys == (1 if block else 0)
            got.append((r.wrong_entries, r.wrong_entry_positions))
        assert got[0] == got[1], (k, classes_at(w, sorted(set(got[0][1]) ^ set(got[1][1])), ents))
        assert got[0][1] == want, (k, classes_at(w, sorted(set(got[0][1]) ^ set(want)), ents))


@pytest.mark.parametrize("n_keys", [9, 17])
def test_batch_check_of_crafted_kangaroos_equals_the_model(tmp_path, n_keys):
    """records checked against their own target (the tg path): the last key, the key at infinity, distance 0, a right point
    under a wrong target, in walk chunks that do not divide the record count"""
    kk = gm.key_scalars(n_keys)
    keys = [gm.key_point(k) for k in kk]
    walks = gm.batch_walks(kk)
    ents = gm.batch_entries(kk)[:5]
    w = gm.work_of(ents, gm.pub_of(kk[0]))
    path = tmp_path / "w.work"
    path.write_bytes(gm.file_bytes(w, kk, walks))
    kinds = [gm.walk_kind(v.x, v.y, v.d, keys[v.target]) for v in walks]
    wrong = [i for i, k in enumerate(kinds) if k == 0]
    wchunk = next(c for c in range(len(walks) // 5, len(walks)) if len(walks) % c and (-(-len(walks) // c)) % 2 == 0)
    assert wrong[-1] >= len(walks) - len(walks) % wchunk > wrong[-2] >= len(walks) - len(walks) % wchunk - wchunk
    for cap in (len(walks), len(wrong) - 1):
        # the check takes chunk / 3 records at a time; with the table's chunk an odd number of chunks, the last two hold wrong
        # records, in the two buffers in the order that the final drain has to undo
        r = wt.check(str(path), chunk=3 * wchunk, cap=cap)
        assert (r.walks, r.walks_tame, r.walks_wild, r.wrong_walks) == (len(walks), kinds.count(1), kinds.count(2), len(wrong))
        assert r.wrong_walk_indices == wrong[:cap], [(v.cls, k) for v, k in zip(walks, kinds)]


# ---- B. retargeting at degenerate points ------------------------------------------------------------------------------------
def test_retarget_at_degenerate_points(oracle, kernel):
    from kangaroo_b200 import GPUEngine, random_herd_arrays
    from kangaroo_b200.solver import retarget_targets
    rp, n = 64, 3 * 32 * 128                                              # 12288: padded last tile on every kernel
    wdiv2 = ((1 << rp) - 1) >> 1
    case = gm.retarget_case(n)
    ks, to = case["ks"], case["to"]
    keys = [ec.mul(k) for k in ks]
    t0 = np.random.default_rng(2).integers(0, len(ks), size=n).astype(np.uint16)
    t0[0::2] = 0
    sc, d128 = random_herd_arrays(n, rp, wdiv2, np.random.default_rng(1))
    for s, (kind, d, b) in case["special"].items():
        t0[s] = 0
        sc[s] = limbs(d, 4)
        d128[s] = limbs((d + wdiv2) % N, 2)

    def engine():
        e = GPUEngine(3, 32, 0, 1 << 17, **kernel)
        e.SetWildOffset(wdiv2)
        e.SetParams(oracle.dp_mask(10), *oracle.create_jump_table(rp))
        e.CreateHerdMulti(sc, d128, keys, t0)
        return e

    a, c = engine(), engine()
    assert a.nbKangaroo == n
    a.Retarget(0, to)
    a.sync()
    want = retarget_targets(t0, 0, to)
    assert np.array_equal(a.Targets(), want)
    ra, rc = a.GetKangaroosRaw(), c.GetKangaroosRaw()
    moved = (np.arange(n) % 2 == 1) & (t0 == 0)
    assert np.array_equal(ra[2], rc[2])                                   # every distance kept
    for u, v in zip(ra[:2], rc[:2]):
        assert np.array_equal(u[~moved], v[~moved])                       # the others untouched
    scal = ints(sc)
    gx, gy = ints(ra[0]), ints(ra[1])
    for s in np.flatnonzero(moved).tolist():
        k = (ks[int(want[s])] + scal[s]) % N                              # keys[b] + d*G
        exp = (0, 0) if k == 0 else oracle.ec_mul_g(k)
        assert (gx[s], gy[s]) == exp, (s, case["special"].get(s))
    for s, (kind, d, b) in case["special"].items():
        assert want[s] == b
        p = ec.add(keys[b], ec.mul(d))
        assert (gx[s], gy[s]) == ((0, 0) if kind == "p_neg_delta" else p) and (p is None) == (kind == "p_neg_delta"), (s, kind)
    assert (want[moved] == 1).sum() > 100                                 # keys[1] = -keys[0]: the delta is a doubling
    a.close(); c.close()


# ---- C. the checkpoint conversion -----------------------------------------------------------------------------------------
def garbage(eng, seed):
    n = eng.nbKangaroo
    rng = np.random.default_rng(seed)
    ax, ay, ad = (rng.integers(0, 1 << 63, size=(n, k), dtype=np.uint64) for k in (4, 4, 2))
    eng.SetKangaroosRaw(ax, ay, ad)


def same_state(eng, state):
    for u, v in zip(eng.GetKangaroosRaw(), state):
        assert np.array_equal(u, v)


def test_import_at_the_reduction_edges(kernel):
    from kangaroo_b200 import GPUEngine
    eng = GPUEngine(2, 16, 0, 65536, **kernel)
    n = eng.nbKangaroo
    rng = np.random.default_rng(5)
    garbage(eng, 1)
    for wo in gm.WILD_OFFSETS:
        eng.SetWildOffset(wo)
        items = [(wild, d) for wild in (False, True) for d in gm.import_distances(wo, wild)]
        fits = [(wild, d) for wild, d in items if gm.biased(d, wo, wild) <= gm.M128]
        bad = [(wild, d) for wild, d in items if gm.biased(d, wo, wild) > gm.M128]
        assert fits and bad

        def records(placed, count):
            """records with distance d at slot s ({s: d}), d = 0 (which fits at every offset) elsewhere"""
            recs = np.zeros((count, 12), dtype=np.uint64)
            recs[:, :8] = rng.integers(0, 1 << 63, size=(count, 8), dtype=np.uint64)
            for s, d in placed.items():
                recs[s, 8:] = limbs(d, 4)
            return recs

        slots = {}
        for q, (wild, d) in enumerate(fits):                              # slot parity = the herd
            slots[2 * q + int(wild)] = d
        recs = records(slots, 2 * len(fits) + 2)
        before = eng.GetKangaroosRaw()
        assert eng.ImportKangaroos(recs, (1, 2), verify=False) == 0
        ax, ay, ad = eng.GetKangaroosRaw()
        m = recs.shape[0]
        assert np.array_equal(ax[:m], recs[:, :4]) and np.array_equal(ay[:m], recs[:, 4:8])
        assert ints(ad[:m]) == [gm.biased(ints(recs[i:i + 1, 8:])[0], wo, i % 2 == 1) for i in range(m)]
        for s, d in slots.items():
            assert ints(ad[s:s + 1])[0] == gm.biased(d, wo, s % 2 == 1)
        assert np.array_equal(ax[m:], before[0][m:]) and np.array_equal(ad[m:], before[2][m:])
        # every record that does not fit fails the call, names its index and changes nothing
        state = eng.GetKangaroosRaw()
        for q, (wild, d) in enumerate(bad):
            s = 2 * (37 * q % 500) + int(wild)
            with pytest.raises(RuntimeError, match=r"record %d: distance does not fit" % s):
                eng.ImportKangaroos(records({s: d}, s + 5), (1, 2), verify=False)
            same_state(eng, state)
        # several bad records over different blocks of the import: the lowest index is named
        high = [2 * (n // 2 - 1 - 163 * q) + int(wild) for q, (wild, d) in enumerate(bad)]
        placed = dict(zip(high, [d for _, d in bad]))
        placed.update({s: d for s, d in list(slots.items())[:4]})
        with pytest.raises(RuntimeError, match=r"record %d: distance does not fit" % min(high)):
            eng.ImportKangaroos(records(placed, n), (1, 2), verify=False)
        same_state(eng, state)
    eng.close()


def test_export_at_the_wild_offset_and_round_trip(kernel):
    from kangaroo_b200 import GPUEngine
    eng = GPUEngine(2, 16, 0, 65536, **kernel)
    n = eng.nbKangaroo
    rng = np.random.default_rng(6)
    for wo in gm.WILD_OFFSETS:
        eng.SetWildOffset(wo)
        ax, ay = (rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64) for _ in range(2))
        ad = rng.integers(0, 1 << 63, size=(n, 2), dtype=np.uint64)
        crafted = gm.export_biased(wo)
        for q, b in enumerate(crafted):                                   # each at an even and an odd kIdx, at both ends
            for s in (2 * q, 2 * q + 1, n - 2 - 2 * q, n - 1 - 2 * q):
                ad[s] = limbs(b, 2)
        eng.SetKangaroosRaw(ax, ay, ad)
        state = eng.GetKangaroosRaw()
        eng.SnapshotBegin()
        recs = eng.SnapshotExport(0, n)
        want = [gm.exported(b, wo, i % 2 == 1) for i, b in enumerate(ints(state[2]))]
        assert ints(recs[:, 8:]) == want
        assert np.array_equal(recs[:, :4], state[0]) and np.array_equal(recs[:, 4:8], state[1])
        for q, b in enumerate(crafted):
            assert ints(recs[2 * q:2 * q + 2, 8:]) == [b, (b - wo) % N]
        garbage(eng, 2)
        assert eng.ImportKangaroos(recs, (1, 2), verify=False) == 0
        same_state(eng, state)                                            # bit for bit
    eng.close()


def test_import_verification_of_points_at_infinity():
    """records whose position herd_kernel stores as (0, 0) -- tame d = 0, wild d*G = -K -- and a wild at d = 0 (the key
    itself) pass verification; with one y bit flipped each fails and nothing changes"""
    from kangaroo_b200 import GPUEngine
    eng = GPUEngine(2, 16, 0, 65536, kernel="stream")
    k = 0x5EED1234567890ABCDEF
    K = ec.mul(k)
    wo = 1 << 100
    eng.SetWildOffset(wo)
    garbage(eng, 3)
    g5 = ec.mul(5)
    rows = [(0, 0, 0), (0, 0, N - k), (g5[0], g5[1], 5), (K[0], K[1], 0)]   # tame 0, wild -K, tame 5G, wild K + 0*G
    recs = np.array([limbs(x, 4) + limbs(y, 4) + limbs(d, 4) for x, y, d in rows], dtype=np.uint64)
    assert eng.ImportKangaroos(recs, K) == 0
    ax, ay, ad = eng.GetKangaroosRaw()
    assert [(a, b) for a, b in zip(ints(ax[:4]), ints(ay[:4]))] == [(x, y) for x, y, _ in rows]
    assert ints(ad[:4]) == [0, wo - k, 5, wo]
    state = eng.GetKangaroosRaw()
    flipped = recs.copy()
    for i in (0, 1, 3):
        flipped[i, 4] ^= np.uint64(1)
    assert eng.ImportKangaroos(flipped, K) == 3
    same_state(eng, state)
    assert eng.ImportKangaroos(recs, ec.mul(k + 1)) == 2                   # another key: both wild records fail
    eng.close()
