"""-m gpu: the multi-key herd at the key limit, 65535 keys (KGX_MAX_KEYS, the engine's uint16 targets).

The other multi-key tests use at most 64 keys and 8 retarget destinations, so every target they write has a high byte of 0
and every kgx_retarget fits in one RetargetChunk of 1024 destinations.  These tests cover what only a large batch reaches:
  - herd_kernel's keys + 16 * targets[i] at targets 255, 256, ... 65534, on a herd that gives every key wilds;
  - kgx_retarget with destination lists of 1023 to 65534 entries: chunks past the first, a partial last chunk, the
    infinity flag (a destination equal to the source) and a doubling delta (one equal to its negative) past index 1024;
  - the key table grown under an engine that already has one (kgx_create_herd_multi, kgx_import_multi);
  - kgx_snapshot_export_targets of a herd whose targets are above 255.
Every key has a known scalar, and every point is checked against the oracle: d*G for tame kangaroos, keys[target] + d*G for
wild ones."""
import os
import re
import shutil
import subprocess
import sys
import time

import numpy as np
import pytest

from oracle import kgo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = kgo.N

NK = 65535                       # KGX_MAX_KEYS
FROM = 300                       # the key every retarget here moves wilds from
SAME, NEG = 40000, 65534         # keys[SAME] == keys[FROM], keys[NEG] == -keys[FROM]
FORCED = [255, 256, 257, 511, 512, 1023, 1024, 4095, 4096, 65279, 65280, 65534]
GRID = (87, 94)                  # 87 x 94 x 128 = 1,046,784 kangaroos, 8 wilds per key: the last tile is padded on every
                                 # kernel (tiles of 896, 1792, 4096 and 16384 kangaroos)
RP = 64
WDIV2 = ((1 << RP) - 1) >> 1
N_TO = [1023, 1024, 1025, 2048, 2049, 65534]


@pytest.fixture(scope="module")
def many(oracle):
    """the 65535 keys: random 63-bit scalars, with keys[SAME] = keys[FROM] and keys[NEG] = -keys[FROM]"""
    rng = np.random.default_rng(21)
    ks = [int(v) | (1 << 62) for v in rng.integers(1, 1 << 62, size=NK)]
    ks[SAME], ks[NEG] = ks[FROM], N - ks[FROM]
    t = time.perf_counter()
    keys = [oracle.ec_mul_g(k) for k in ks]
    print("\n[many keys] %d keys from their scalars in %.1f s" % (NK, time.perf_counter() - t))
    assert len({k[0] for k in keys}) == NK - 2 and keys[NEG] == (keys[FROM][0], (kgo.P - keys[FROM][1]) % kgo.P)
    return dict(keys=keys, table=oracle.create_jump_table(RP))


def engine(oracle, many, kernel, targets, keys=None, seed=1):
    from kangaroo_b200 import GPUEngine, random_herd_arrays
    eng = GPUEngine(GRID[0], GRID[1], 0, 1 << 16, **kernel)
    eng.SetWildOffset(WDIV2)
    eng.SetParams(oracle.dp_mask(14), *many["table"])
    sc, d128 = random_herd_arrays(eng.nbKangaroo, RP, WDIV2, np.random.default_rng(seed))
    eng.CreateHerdMulti(sc, d128, many["keys"] if keys is None else keys, targets)
    return eng


def herd_size():
    return GRID[0] * GRID[1] * 128


def all_key_targets():
    from kangaroo_b200.solver import assign_targets
    return assign_targets(herd_size(), list(range(NK)))


def val(row):
    return sum(int(v) << (64 * k) for k, v in enumerate(row))


def check_points(oracle, keys, targets, raw, idx):
    """kangaroos idx of a GetKangaroosRaw() against the oracle: d*G (tame, even kIdx) or keys[target] + d*G (wild)"""
    ax, ay, ad = raw
    for i in sorted(set(int(v) for v in idx)):
        d = val(ad[i])
        if i % 2:
            d = (d - WDIV2) % N
        p = oracle.ec_mul_g(d)
        want = oracle.ec_add(keys[int(targets[i])], p) if i % 2 else p
        assert (val(ax[i]), val(ay[i])) == want, (i, int(targets[i]))


def spread_sample(n, k=200):
    """evenly spread kangaroos, and the last 64: the padded last tile of every kernel"""
    return np.unique(np.concatenate([np.arange(0, n, n // k), np.arange(n - 64, n)]))


# ---- the herd -------------------------------------------------------------------------------------------------------------
def test_herd_at_65535_keys_matches_the_oracle(oracle, many, kernel):
    n = herd_size()
    t = all_key_targets()
    forced = []
    for m, f in enumerate(FORCED):                                       # each forced target twice: early and in the last tile
        for s in (2 * (5000 + 17 * m) + 1, n - 1 - 2 * m):
            t[s] = f
            forced.append(s)
    assert set(t[1::2].tolist()) == set(range(NK))
    eng = engine(oracle, many, kernel, t)
    assert np.array_equal(eng.Targets(), t)
    raw = eng.GetKangaroosRaw()
    high = np.flatnonzero((np.arange(n) % 2 == 1) & (t > 255))[::2617]   # wilds of ordinary keys above 255
    check_points(oracle, many["keys"], t, raw, np.concatenate([spread_sample(n), forced, high]))
    eng.close()


# ---- retargeting ----------------------------------------------------------------------------------------------------------
def destinations(n_to):
    """the destination list of n_to entries, never FROM: every other key for 65534 (SAME at index 39999, NEG at 65533), else
    distinct keys chosen at random with SAME and NEG as the last two"""
    if n_to == NK - 1:
        return [k for k in range(NK) if k != FROM]
    pool = np.array([k for k in range(NK) if k not in (FROM, SAME, NEG)])
    to = np.random.default_rng(n_to).choice(pool, n_to - 2, replace=False).tolist()
    return to + [SAME, NEG]


def checked_js(n_to, to):
    """destination indices with at least one moved wild checked against the oracle"""
    return sorted({j for j in (0, 1023, 1024, 2047, 2048, n_to - 1) if j < n_to} | {to.index(SAME), to.index(NEG)})


def retarget_herd(n_to, to):
    """the targets of a herd over every key, with wilds of FROM forced where (kIdx >> 1) % n_to hits each checked index: the
    first such wild and the last, which for small n_to is in the padded last tile"""
    n = herd_size()
    t = all_key_targets()
    for j in checked_js(n_to, to):
        t[2 * j + 1] = FROM
        t[2 * (j + ((n // 2 - 1 - j) // n_to) * n_to) + 1] = FROM
    return t


@pytest.mark.parametrize("n_to", N_TO)
def test_retarget_across_chunks(oracle, many, kernel, n_to):
    """The moved wilds of every checked destination index sit at keys[to[j]] + d*G, Targets() is the host mirror's, distances
    are kept and every other kangaroo is bit-identical to a twin never retargeted.  With 65534 destinations the retarget is
    issued while a launch is in flight, and equals one issued after a sync."""
    from kangaroo_b200.solver import retarget_targets
    keys = many["keys"]
    to = destinations(n_to)
    assert len(to) == n_to and len(set(to)) == n_to and FROM not in to
    t0 = retarget_herd(n_to, to)
    n = herd_size()
    in_flight = n_to == NK - 1
    engs = [engine(oracle, many, kernel, t0) for _ in range(3 if in_flight else 2)]
    t_launch = time.perf_counter()
    if in_flight:
        for e in engs:
            e.set_jumps_per_launch(1024)
            e.callKernel()
    a, c = engs[0], engs[-1]                                             # retargeted, never retargeted
    t = time.perf_counter()
    a.Retarget(FROM, to)
    call_ms = 1e3 * (time.perf_counter() - t)
    since_launch_ms = 1e3 * (time.perf_counter() - t_launch)
    for e in engs:
        e.sync()
    if in_flight:             # a's launch, issued first, was still running when the call returned: it lasted twice as long
        assert since_launch_ms < 0.5 * a.last_launch_ms(), (since_launch_ms, a.last_launch_ms())
    want = retarget_targets(t0, FROM, to)
    assert np.array_equal(a.Targets(), want)
    ra, rc = a.GetKangaroosRaw(), c.GetKangaroosRaw()
    if in_flight:
        b = engs[1]
        b.Retarget(FROM, to)
        assert np.array_equal(b.Targets(), want)
        for u, v in zip(ra, b.GetKangaroosRaw()):
            assert np.array_equal(u, v)
    kidx = np.arange(n)
    moved = (kidx % 2 == 1) & (t0 == FROM)
    j_of = (kidx >> 1) % n_to
    assert set(checked_js(n_to, to)) <= set(j_of[moved].tolist())
    assert np.array_equal(ra[2], rc[2])                                  # every distance kept
    for u, v in zip(ra[:2], rc[:2]):
        assert np.array_equal(u[~moved], v[~moved])                      # the others untouched
    same = moved & (want == SAME)
    assert same.any() and (moved & (want == NEG)).any()
    assert np.array_equal(ra[0][same], rc[0][same]) and np.array_equal(ra[1][same], rc[1][same])   # infinity flag: kept
    other = moved & ~same
    assert (ra[0][other] != rc[0][other]).any(axis=1).all()
    check_points(oracle, keys, want, ra, np.flatnonzero(moved))
    print("\n[retarget %s] n_to = %d: %d wilds moved, call %.2f ms%s" % (
        a.kernel, n_to, int(moved.sum()), call_ms, " (%.2f ms after a %.2f ms launch began)" % (since_launch_ms, a.last_launch_ms())
        if in_flight else ""))
    for e in engs:
        e.close()


# ---- the key table grown under an engine that has one ----------------------------------------------------------------------
STREAM128 = dict(kernel="stream", stream_g=128)


def test_key_table_grows_from_9_to_65535_keys(oracle, many):
    """kgx_create_herd_multi with 65535 keys on an engine whose herd had 9, then a retarget across chunks: bit-identical to a
    fresh engine given the same two calls"""
    from kangaroo_b200 import random_herd_arrays
    from kangaroo_b200.solver import assign_targets
    to = destinations(2049)
    t0 = retarget_herd(2049, to)
    grown = engine(oracle, many, STREAM128, assign_targets(herd_size(), list(range(9))), keys=many["keys"][:9], seed=5)
    fresh = engine(oracle, many, STREAM128, t0)
    sc, d128 = random_herd_arrays(grown.nbKangaroo, RP, WDIV2, np.random.default_rng(1))
    mem = grown.GetMemory()
    grown.CreateHerdMulti(sc, d128, many["keys"], t0)
    assert grown.GetMemory() == fresh.GetMemory() > mem
    for e in (grown, fresh):
        e.Retarget(FROM, to)
    assert np.array_equal(grown.Targets(), fresh.Targets())
    for u, v in zip(grown.GetKangaroosRaw(), fresh.GetKangaroosRaw()):
        assert np.array_equal(u, v)
    grown.close()
    fresh.close()


def test_export_of_65535_keys_imports_into_an_engine_of_9(oracle, many):
    """A snapshot of a 65535-key herd, with a retarget queued behind it: its targets are the cut's.  Its records and targets,
    imported with verification into an engine whose herd had 9 keys, give the source's state and targets; a retarget across
    chunks then agrees on both engines, and so do the DPs of the next 3 launches."""
    from kangaroo_b200.solver import assign_targets, retarget_targets
    to = destinations(2049)
    t0 = retarget_herd(2049, to)
    src = engine(oracle, many, STREAM128, t0)
    dst = engine(oracle, many, STREAM128, assign_targets(herd_size(), list(range(9))), keys=many["keys"][:9], seed=5)
    n = src.nbKangaroo
    src.set_jumps_per_launch(64)
    src.callKernel()
    src.sync()
    cut = src.GetKangaroosRaw()
    src.SnapshotBegin()
    src.Retarget(FROM, to)                                               # after the snapshot: not in its targets
    want = retarget_targets(t0, FROM, to)
    tg = np.concatenate([src.SnapshotExportTargets(0, 1000), src.SnapshotExportTargets(1000, n - 1000)])
    recs = src.SnapshotExport(0, n)
    assert np.array_equal(tg, t0) and (tg[1::2] > 255).mean() > 0.99
    assert np.array_equal(src.Targets(), want)
    assert dst.ImportKangaroosMulti(recs, many["keys"], tg, verify=True) == 0
    assert np.array_equal(dst.Targets(), t0)
    for u, v in zip(dst.GetKangaroosRaw(), cut):
        assert np.array_equal(u, v)
    dst.Retarget(FROM, to)
    assert np.array_equal(dst.Targets(), want)
    for u, v in zip(dst.GetKangaroosRaw(), src.GetKangaroosRaw()):
        assert np.array_equal(u, v)
    check_points(oracle, many["keys"], want, src.GetKangaroosRaw(), np.flatnonzero(t0 == FROM)[::3])
    ndp = 0
    for e in (src, dst):
        e.set_jumps_per_launch(64)
    for _ in range(3):
        got = []
        for e in (src, dst):
            e.callKernel()
            got.append(sorted((it.x, it.d, it.kIdx) for it in e.Launch(relaunch=False)))
        assert got[0] == got[1]
        ndp += len(got[0])
        for x, d, k in got[0][::max(1, len(got[0]) // 50)]:
            p = oracle.ec_mul_g(d)
            assert x == (oracle.ec_add(many["keys"][int(want[k])], p) if k % 2 else p)[0], k
    assert ndp > 1000
    src.close()
    dst.close()


# ---- the batch work-file check at 65535 keys --------------------------------------------------------------------------------
INF = 65533                      # the check's key at infinity (pub = start*G)


def test_batch_check_at_65535_keys_equals_the_model(oracle, tmp_path):
    """worktool check of a 65535-key batch file: wild entries that match key 0, 7, 8, 65528 (the first key of the last batch
    of KB = 8, which holds 7 keys), 65534 and no key; S = +K (a doubling) at key 65530, S = -K at 65529, S through the key at
    infinity; kangaroo records whose targets are above 255, one of them a right point under a byte-swapped target.  The counts
    and the listed wrong records equal the model of tests/group_law_model.py.  The check costs entries x keys: few entries."""
    from kangaroo_b200 import ecmath as ec
    from kangaroo_b200 import worktool as wt
    from tests import group_law_model as gm
    rnd = np.random.default_rng(31)
    kk = [int(v) << 38 | int(w) for v, w in zip(rnd.integers(1 << 61, 1 << 62, size=NK), rnd.integers(0, 1 << 38, size=NK))]
    kk[INF] = 0
    K = [None if k == 0 else oracle.ec_mul_g(k) for k in kk]
    pubs = [oracle.ec_mul_g((k + gm.START) % N) for k in kk]
    mag = lambda: int(rnd.integers(1, 1 << 62)) << 30 | int(rnd.integers(0, 1 << 30))

    ents = []

    def add(cls, key, pt, d):
        h, x = gm.hx(pt) if pt is not None else (int(rnd.integers(0, 1 << 18)), int(rnd.integers(1, 1 << 62)) << 64 | 12345)
        ents.append(gm.Entry(cls, key, None, h, x, d))

    for j, neg in ((0, False), (7, True), (8, False), (65528, False), (65528, True), (65534, True)):
        d = gm.tagged(mag(), True, neg)
        add("match", j, oracle.ec_add(gm.s_point(d), K[j]), d)
    add("none", None, None, gm.tagged(mag(), True, False))
    m, neg = gm.signed_mag(kk[65530])
    add("dbl", 65530, ec.add(K[65530], K[65530]), gm.tagged(m, True, neg))         # the oracle's ec_add does not double
    m, neg = gm.signed_mag(N - kk[65529])
    add("opp", 65529, None, gm.tagged(m, True, neg))
    d = gm.tagged(mag(), True, True)
    add("inf_key", INF, gm.s_point(d), d)
    d = gm.tagged(mag(), False, False)
    add("tame", None, gm.s_point(d), d)
    e = ents[3]
    ents.append(e._replace(cls="bad_x", x=e.x ^ (1 << 77)))
    w = gm.work_of(ents, pubs[0])

    walks = []
    for i, t in enumerate((256, 257, 4096, 65279, 65280, 65528, 65534, 511)):
        dd = int(rnd.integers(1, 1 << 62))
        p = oracle.ec_add(K[t], oracle.ec_mul_g(dd))
        walks.append(gm.Walk("wild", p[0], p[1], dd, t))
        p = oracle.ec_mul_g(dd + 1)
        walks.append(gm.Walk("tame", p[0], p[1], dd + 1, 65000 + i))
    p = oracle.ec_add(K[1], oracle.ec_mul_g(99))
    walks.append(gm.Walk("byte_swap", p[0], p[1], 99, 0x0100))           # key 1's point under target 256: wrong
    p = oracle.ec_add(K[0x0102], oracle.ec_mul_g(98))
    walks.append(gm.Walk("truncated", p[0], p[1], 98, 0x0202))           # key 258's point under 514: wrong
    w.walks = gm.walk_bytes(walks)
    plain = w.to_bytes()
    path = tmp_path / "max.work"
    path.write_bytes(plain + wt.batch_block(wt.BatchBlock(pubs, [False] * NK, [None] * NK, [v.target for v in walks]),
                                            len(plain)).tobytes())

    t = time.perf_counter()
    want = gm.wrong_positions(w, K)
    t_model = time.perf_counter() - t
    kinds = [gm.walk_kind(v.x, v.y, v.d, K[v.target]) for v in walks]
    wrong_walks = [i for i, k in enumerate(kinds) if k == 0]
    by = {(e.h, e.x, e.d): e.cls for e in ents}
    assert sorted(by[(h, *w.table[h][i])] for h, i in want) == ["bad_x", "none", "opp"]
    assert wrong_walks == [len(walks) - 2, len(walks) - 1]
    t = time.perf_counter()
    r = wt.check(str(path), cap=64)
    t_check = time.perf_counter() - t
    assert r.n_keys == NK and r.entries == len(ents) and r.walks == len(walks)
    assert r.wrong_entry_positions == want, [by[(h, *w.table[h][i])] for h, i in r.wrong_entry_positions]
    assert r.wrong_entries == len(want)
    assert (r.walks_tame, r.walks_wild, r.wrong_walks) == (kinds.count(1), kinds.count(2), len(wrong_walks))
    assert r.wrong_walk_indices == wrong_walks
    print("\n[batch check] %d keys: %d entries, %d kangaroos checked in %.2f s (the model: %.1f s)"
          % (NK, len(ents), len(walks), t_check, t_model))



# ---- the solver: more keys solved in one step than one control broadcast announces ------------------------------------------
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")


@pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")
def test_batch_solver_queues_what_one_broadcast_cannot_announce(oracle, tmp_path):
    """2048 keys of a 2^34 range on a herd of 131,072 kangaroos (32 wilds per key): hundreds of keys are solved in one step, so
    keys wait in the announcement queue (MAX_SOLVED per step).  Every key is found with its private key; no step announces more
    than MAX_SOLVED classes and each class is announced once; after every step the engine's targets are the host mirror's and
    no wild sits on an announced key.  A --batch-save-interval save whose cut has keys waiting passes `worktool check`, shows
    solved exactly the keys announced up to its cut, keeps the waiting keys unsolved with their wilds on them (DESIGN §4), and
    --batch-resume of it finds every key."""
    from kangaroo_b200 import solver as S
    from kangaroo_b200 import worktool
    nk, start, grid = 2048, 0x5A5A5A5A5A5A5A5A0000000000, (8, 128)
    end = start + (1 << 34) - 1
    rng = np.random.default_rng(41)
    privs = [start + int(v) for v in rng.choice(1 << 34, size=nk, replace=False)]
    pubs = [oracle.ec_mul_g(p) for p in privs]
    path, copy = str(tmp_path / "q.work"), str(tmp_path / "copy.work")
    steps, cuts, saved = [], [], []

    class Watch(S.BatchSolver):
        def _solved(self, solved):
            queued = list(self._announce)                  # step() has taken this step's announcements off the queue
            done = super()._solved(solved)
            steps.append((list(solved), queued))
            assert np.array_equal(self.eng.Targets(), self.targets)
            if not done:                                   # (the last key solved has nowhere to send its wilds)
                assert not set(self.targets[1::2].tolist()) & self.announced
            if queued and not any(q for _, q in cuts) and not self._saving and not self._save_due:
                self.save_interval = 1e-6                  # the next step takes a save, its cut while keys wait (if they still do)
            return done

        def _save_start(self, kangaroos, chunks):
            self.save_interval = 1e9
            super()._save_start(kangaroos, chunks)

        def _on_saved(self, p, mb, seconds, err):          # writer thread, saves in cut order
            assert err is None
            k = len(saved)
            saved.append(p)
            if cuts[k][1] and not os.path.exists(copy):
                shutil.copy(p, copy)

    s = Watch(start, end, pubs, 8, grid, seed=12, save_work=path, save_interval=1e9)
    snap = s.eng.SnapshotBegin

    def snapshot():                                        # the cut: the classes announced, and the keys still queued
        cuts.append((set(s.announced), list(s._announce)))
        snap()

    s.eng.SnapshotBegin = snapshot
    t = time.perf_counter()
    s.run(600, verbose=False)
    s.close()
    per_step = [len(a) for a, _ in steps]
    st = np.array(s._step_times) * 1e3
    print("\n[batch queue] %d keys in %d steps, %.1f s (step median %.1f ms, max %.1f ms); most announced in one step %d, longest "
          "queue %d, %d saves" % (nk, len(steps), time.perf_counter() - t, np.median(st), st.max(), max(per_step),
                                   max(len(q) for _, q in steps), len(saved)))
    assert s.priv == privs
    announced = [r for a, _ in steps for r in a]
    assert sorted(announced) == list(range(nk))                           # every class once
    assert max(per_step) == S.MAX_SOLVED and any(q for _, q in steps)

    assert os.path.exists(copy), [len(q) for _, q in cuts]
    done_at_cut, queued_at_cut = next(c for c in cuts if c[1])
    b = worktool.read_batch(copy)
    assert [i for i, v in enumerate(b.solved) if v] == sorted(done_at_cut)
    assert all(b.privs[i] == privs[i] for i in done_at_cut)
    wild = set(b.targets[1::2].tolist())
    assert not wild & done_at_cut and set(queued_at_cut) <= wild and not any(b.solved[i] for i in queued_at_cut)
    r = worktool.check(copy)
    assert r.ok and r.n_keys == nk and r.walks == grid[0] * grid[1] * 128, vars(r)
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver", "--batch-keys", "--batch-resume", copy, "--seed", "13",
                        "--grid", "%d,%d" % grid], capture_output=True, text=True, timeout=900, cwd=ROOT)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out[-3000:]
    got = {int(i): int(v, 16) for i, v in re.findall(r"Key#\s*(\d+) Pub:\s+0x[0-9A-F]+\s+Priv: 0x([0-9A-F]+)", out)}
    assert got == dict(enumerate(privs)), out[-3000:]
    assert "%d of %d keys solved in the file" % (len(done_at_cut), nk) in out, out[-3000:]
