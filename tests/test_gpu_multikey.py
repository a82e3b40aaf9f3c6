"""-m gpu: the multi-key herd (kgx_create_herd_multi / kgx_retarget / kgx_targets) on every kernel, and the solver's
--batch-keys, which solves every key of an input in one run with one tame herd."""
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from oracle import kgo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")

RP = 64
WDIV2 = ((1 << RP) - 1) >> 1
NKEYS = 9


def key_points(oracle, n=NKEYS, seed=17):
    rng = np.random.default_rng(seed)
    return [oracle.ec_mul_g(int(rng.integers(1, 1 << 62)) | (1 << 62)) for _ in range(n)]


def multi_engine(oracle, kernel, keys, targets, seed=1, grid=(3, 32)):
    """3 x 32 x 128 = 12288 kangaroos: padded tiles on every kernel"""
    from kangaroo_b200 import GPUEngine, random_herd_arrays
    eng = GPUEngine(grid[0], grid[1], 0, 1 << 17, **kernel)
    eng.SetWildOffset(WDIV2)
    eng.SetParams(oracle.dp_mask(10), *oracle.create_jump_table(RP))
    sc, d128 = random_herd_arrays(eng.nbKangaroo, RP, WDIV2, np.random.default_rng(seed))
    eng.CreateHerdMulti(sc, d128, keys, targets)
    return eng


def random_targets(n, nkeys, seed=2):
    t = np.random.default_rng(seed).integers(0, nkeys, size=n).astype(np.uint16)
    t[0::2] = 0
    return t


def sample(n, k=160):
    return np.unique(np.concatenate([np.arange(0, n, n // k), np.arange(n - 32, n)]))


def expected_point(oracle, keys, targets, kidx, d):
    p = oracle.ec_mul_g(d % kgo.N)
    return p if kidx % 2 == 0 else oracle.ec_add(keys[int(targets[kidx])], p)


def test_multi_key_herd_matches_the_oracle(oracle, kernel):
    keys = key_points(oracle)
    n = 3 * 32 * 128
    targets = random_targets(n, NKEYS)
    eng = multi_engine(oracle, kernel, keys, targets)
    assert np.array_equal(eng.Targets(), targets)
    assert sorted(set(targets[1::2].tolist())) == list(range(NKEYS))
    gx, gy, gd = eng.GetKangaroos()
    for i in sample(n):
        assert (gx[i], gy[i]) == expected_point(oracle, keys, targets, i, gd[i]), i
    eng.close()


def test_multi_key_herd_refusals(oracle):
    from kangaroo_b200 import GPUEngine, random_herd_arrays
    keys = key_points(oracle, 3)
    eng = GPUEngine(2, 16, 0, 65536, kernel="stream")
    n = eng.nbKangaroo
    sc, d128 = random_herd_arrays(n, RP, WDIV2, np.random.default_rng(3))
    mem = eng.GetMemory()
    with pytest.raises(RuntimeError, match="no key table"):
        eng.Retarget(0, [1])
    with pytest.raises(RuntimeError, match="no key table"):
        eng.Targets()
    with pytest.raises(RuntimeError, match="n_keys must be"):
        eng.CreateHerdMulti(sc, d128, [], np.zeros(n, np.uint16))
    bad = np.zeros(n, np.uint16)
    bad[777] = 3
    with pytest.raises(RuntimeError, match="target 3 of kangaroo 777"):
        eng.CreateHerdMulti(sc, d128, keys, bad)
    eng.CreateHerdMulti(sc, d128, keys, random_targets(n, 3))
    assert eng.GetMemory() >= mem + 2 * n + 3 * 132
    with pytest.raises(RuntimeError, match="not below n_keys"):
        eng.Retarget(3, [0])
    with pytest.raises(RuntimeError, match="to\\[1\\] = 5"):
        eng.Retarget(0, [1, 5])
    with pytest.raises(RuntimeError, match="n_to"):
        eng.Retarget(0, [])
    eng.CreateHerdRaw(sc, d128, keys[0])                                  # a single-key herd drops the table
    with pytest.raises(RuntimeError, match="no key table"):
        eng.Retarget(0, [1])
    eng.CreateHerdMulti(sc, d128, keys, random_targets(n, 3))
    eng.SetSymmetry("symclass")                                           # so does symmetric mode
    for call in (lambda: eng.Retarget(0, [1]), eng.Targets):
        with pytest.raises(RuntimeError, match="symmetric"):
            call()
    eng.close()
    sym = GPUEngine(2, 16, 0, 65536, kernel="resident")
    sym.SetSymmetry("symclass")
    with pytest.raises(RuntimeError, match="symmetric"):
        sym.CreateHerdMulti(sc, d128, keys, random_targets(n, 3))
    sym.close()


def test_retarget_in_flight(oracle, kernel):
    """Retarget while a launch is in flight equals retarget after it (twin engine); moved wilds sit at keys[new] + d*G with
    their distance kept, every other kangaroo is bit-identical to an engine never retargeted, and the DPs of the next launches
    are on the right trails."""
    from kangaroo_b200.solver import retarget_targets
    keys = key_points(oracle)
    keys[7] = keys[3]                                                     # the same key twice: a move that keeps the point
    n = 3 * 32 * 128
    t0 = random_targets(n, NKEYS)
    frm, to = 3, [0, 1, 2, 4, 5, 6, 7, 8]
    engs = [multi_engine(oracle, kernel, keys, t0) for _ in range(3)]     # in flight, after a sync, never retargeted
    for e in engs:
        e.set_jumps_per_launch(2048)
        e.callKernel()
    a, b, c = engs
    t = time.perf_counter()
    a.Retarget(frm, to)
    host_ms = 1e3 * (time.perf_counter() - t)
    for e in engs:
        e.sync()
    launch_ms = a.last_launch_ms()
    b.Retarget(frm, to)
    want = retarget_targets(t0, frm, to)
    assert np.array_equal(a.Targets(), want) and np.array_equal(b.Targets(), want)
    ra, rb, rc = a.GetKangaroosRaw(), b.GetKangaroosRaw(), c.GetKangaroosRaw()
    for u, v in zip(ra, rb):
        assert np.array_equal(u, v)
    moved = (np.arange(n) % 2 == 1) & (t0 == frm)
    assert moved.sum() > 500 and (want[moved] == 7).any()
    assert np.array_equal(ra[2], rc[2])                                   # every distance kept
    for u, v in zip(ra[:2], rc[:2]):
        assert np.array_equal(u[~moved], v[~moved])                       # the others untouched
        assert not np.array_equal(u[moved & (want != 7)], v[moved & (want != 7)])
    assert np.array_equal(ra[0][moved & (want == 7)], rc[0][moved & (want == 7)])   # key 7 == key 3: the point stays
    gx, gy, gd = a.GetKangaroos()
    for i in sorted(set(sample(n)) | set(np.flatnonzero(moved)[::8].tolist())):
        assert (gx[i], gy[i]) == expected_point(oracle, keys, want, i, gd[i]), i
    print("\n[retarget] %s kernel: host %.3f ms while a %.2f ms launch ran" % (a.kernel, host_ms, launch_ms))
    assert host_ms < 0.5 * launch_ms                                      # the call did not wait for the launch
    # the next launches: each DP lies on d*G (tame) or keys[target] + d*G (wild)
    a.set_jumps_per_launch(64)
    ndp = 0
    for _ in range(3):
        a.callKernel()
        items = a.Launch(relaunch=False)
        assert a.lastFound <= a.maxFound
        for it in items[::max(1, len(items) // 150)]:
            assert it.x == expected_point(oracle, keys, want, it.kIdx, it.d)[0], it
            ndp += 1
    assert ndp > 300
    for e in engs:
        e.close()


# ---- the solver ---------------------------------------------------------------------------------------------------------
def solver(args, timeout=900, prefix=None):
    p = subprocess.run((prefix or [sys.executable]) + ["-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT)
    return p.returncode, p.stdout + p.stderr


def privs(out):
    return {int(i): int(v, 16) for i, v in re.findall(r"Key#\s*(\d+) Pub:\s+0x[0-9A-F]+\s+Priv: 0x([0-9A-F]+)", out)}


def batch_jumps(out):
    m = re.search(r"Batch: (\d+)/(\d+) keys solved, (\d+) jumps", out)
    assert m, out[-3000:]
    return int(m.group(1)), int(m.group(2)), int(m.group(3))


ANSWERS = [int(v, 16) for v in open(os.path.join(GOLD, "in56_64keys.answers.txt")).read().split()]
SEQUENTIAL_MODEL = 64 * 2.08 * 2 ** 28                                   # 64 single-key runs of 2.08 sqrt(N) jumps


@needs_ingest
def test_batch_solves_64_keys_in_one_run():
    rc, out = solver([os.path.join(GOLD, "in56_64keys.txt"), "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "3"])
    assert rc == 0, out[-3000:]
    assert privs(out) == dict(enumerate(ANSWERS)), out[-3000:]
    solved, total, jumps = batch_jumps(out)
    assert solved == total == 64
    print("\n[batch-keys] 64 keys of 2^56: %d jumps = %.3f x the sequential model (%.3g), %.2f sqrt(N) per key"
          % (jumps, jumps / SEQUENTIAL_MODEL, SEQUENTIAL_MODEL, jumps / 64 / 2 ** 28))
    assert jumps < 0.5 * SEQUENTIAL_MODEL


@needs_ingest
def test_batch_reports_a_key_outside_the_range(tmp_path):
    lines = open(os.path.join(GOLD, "in56_64keys.txt")).read().split()
    outside = ec.mul(int(lines[0], 16) + (0xC0FFEE << 160))              # 2^183 past the range start: out of reach
    cfg = tmp_path / "three.txt"
    cfg.write_text("\n".join(lines[:3] + ["04%064X%064X" % outside, lines[3]]) + "\n")
    rc, out = solver([str(cfg), "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "4", "--max-steps", "400"])
    assert rc == 1, out[-3000:]
    assert privs(out) == {0: ANSWERS[0], 2: ANSWERS[1]}, out[-3000:]
    assert "Key# 1 not found" in out
    assert batch_jumps(out)[:2] == (2, 3)


@needs_ingest
def test_batch_solves_a_key_listed_twice_and_its_negative(tmp_path):
    """A key listed twice, and the key whose keyToSearch is the negative of another's (2*start - priv, below the range), are
    searched once with the first of their class and all reported."""
    lines = open(os.path.join(GOLD, "in56_64keys.txt")).read().split()
    start = int(lines[0], 16)
    mirror = (2 * start - ANSWERS[1]) % ec.N
    cfg = tmp_path / "dup.txt"
    cfg.write_text("\n".join(lines[:4] + [lines[2], "04%064X%064X" % ec.mul(mirror), lines[4]]) + "\n")
    rc, out = solver([str(cfg), "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "6", "--max-steps", "4000"])
    assert rc == 0, out[-3000:]
    assert privs(out) == {0: ANSWERS[0], 1: ANSWERS[1], 2: ANSWERS[0], 3: mirror, 4: ANSWERS[2]}, out[-3000:]
    assert batch_jumps(out)[:2] == (5, 5)
    assert "Batch time: set-up" in out


@needs_ingest
def test_batch_on_two_gpus():
    """two GPUs, or two ranks sharing one over gloo"""
    from tests.ranks_util import solver_on
    rc, out = solver_on(2, [os.path.join(GOLD, "in56_64keys.txt"), "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "5"])
    assert rc == 0, out[-3000:]
    assert privs(out) == dict(enumerate(ANSWERS)), out[-3000:]
    assert batch_jumps(out)[:2] == (64, 64)
