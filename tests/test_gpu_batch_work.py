"""-m gpu: checkpoint and resume of a multi-key herd (the targets in kgx_snapshot_begin / kgx_snapshot_export_targets,
kgx_import_multi) on every kernel, and the solver's batch work files (--batch-keys --batch-save / --batch-resume) checked by
the work-file tool."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from tests.test_gpu_multikey import ANSWERS, GOLD, NKEYS, batch_jumps, expected_point, key_points, multi_engine, needs_ingest, \
    privs, random_targets, sample, solver

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG64 = os.path.join(GOLD, "in56_64keys.txt")
N = 3 * 32 * 128
GRID = ["--dp", "8", "--grid", "32,128"]
PER_STEP = 32 * 128 * 128 * 64


def export_all(eng, chunk=5000):
    """records and targets of the pending snapshot, in chunks that do not divide n (targets first: the last record chunk
    releases the snapshot)"""
    n = eng.nbKangaroo
    tg = eng.SnapshotExportTargets(0, n)
    recs = np.empty((n, 12), dtype=np.uint64)
    for first in range(0, n, chunk):
        c = min(chunk, n - first)
        eng.SnapshotExport(first, c, recs[first:first + c])
    return recs, tg


def test_snapshot_holds_the_targets_of_the_cut(oracle, kernel):
    keys = key_points(oracle)
    t0 = random_targets(N, NKEYS)
    eng = multi_engine(oracle, kernel, keys, t0)
    eng.set_jumps_per_launch(256)
    eng.callKernel()
    eng.SnapshotBegin()                                                   # after the launch in flight
    cut = eng.Targets()
    eng.Retarget(3, [0, 1, 2, 4, 5, 6, 7, 8])                             # queued after the snapshot
    after = eng.Targets()
    assert np.array_equal(cut, t0) and not np.array_equal(after, cut)
    assert np.array_equal(eng.SnapshotExportTargets(0, N), cut)
    assert np.array_equal(eng.SnapshotExportTargets(777, 1000), cut[777:1777])
    _, tg = export_all(eng)
    assert np.array_equal(tg, cut)
    with pytest.raises(RuntimeError, match="no snapshot pending"):
        eng.SnapshotExportTargets(0, 1)
    eng.sync()
    eng.close()


def test_import_multi_restores_the_herd_bit_for_bit(oracle, kernel):
    from kangaroo_b200 import GPUEngine
    keys = key_points(oracle)
    src = multi_engine(oracle, kernel, keys, random_targets(N, NKEYS))
    src.callKernelAndWait()
    src.Retarget(5, [0, 1, 2, 3, 4, 6, 7, 8])
    src.SnapshotBegin()
    recs, tg = export_all(src)
    src.sync()
    dst = GPUEngine(3, 32, 0, 1 << 17, **kernel)                          # a fresh engine: no herd, no key table
    dst.SetWildOffset(src.wildOffset)
    dst.SetParams(src.dpMask, *oracle.create_jump_table(64))
    assert dst.ImportKangaroosMulti(recs, keys, tg) == 0
    for a, b in zip(dst.GetKangaroosRaw(), src.GetKangaroosRaw()):
        assert np.array_equal(a, b)
    assert np.array_equal(dst.Targets(), src.Targets())
    for _ in range(3):                                                    # the next launches find the same DPs
        dps = []
        for e in (src, dst):
            e.callKernel()
            dps.append(sorted((it.x, it.d, it.kIdx) for it in e.Launch(relaunch=False)))
        assert dps[0] == dps[1] and len(dps[0]) > 10
    dst.Retarget(1, [0, 2])                                               # the key table is installed
    src.Retarget(1, [0, 2])
    assert np.array_equal(dst.Targets(), src.Targets())
    for a, b in zip(dst.GetKangaroosRaw(), src.GetKangaroosRaw()):
        assert np.array_equal(a, b)
    src.close(); dst.close()


def test_import_multi_verification_changes_nothing_on_a_mismatch(oracle, kernel):
    keys = key_points(oracle)
    src = multi_engine(oracle, kernel, keys, random_targets(N, NKEYS))
    src.SnapshotBegin()
    recs, tg = export_all(src)
    dst = multi_engine(oracle, kernel, keys, random_targets(N, NKEYS, seed=9), seed=4)
    state, targets = dst.GetKangaroosRaw(), dst.Targets()

    def unchanged():
        for a, b in zip(dst.GetKangaroosRaw(), state):
            assert np.array_equal(a, b)
        assert np.array_equal(dst.Targets(), targets)

    wrong = tg.copy()
    for i in (1, 3, 4001, N - 1):                                         # wild records given another key
        wrong[i] = (wrong[i] + 1) % NKEYS
    wrong[2] = 5                                                          # a tame record's target is not used
    assert dst.ImportKangaroosMulti(recs, keys, wrong) == 4
    unchanged()
    others = key_points(oracle, seed=99)                                  # another key set: every wild fails
    assert dst.ImportKangaroosMulti(recs, others, tg) == N // 2
    unchanged()
    bad = tg.copy()
    bad[7] = NKEYS
    with pytest.raises(RuntimeError, match="target 9 of record 7"):
        dst.ImportKangaroosMulti(recs, keys, bad)
    unchanged()
    # a partial import: records 0..999 replace the herd's, the rest keeps its state and targets
    assert dst.ImportKangaroosMulti(recs[:1000], keys, tg[:1000]) == 0
    ax, ay, ad = dst.GetKangaroosRaw()
    got = dst.Targets()
    assert np.array_equal(got[:1000], tg[:1000]) and np.array_equal(got[1000:], targets[1000:])
    assert np.array_equal(ax[1000:], state[0][1000:]) and np.array_equal(ad[1000:], state[2][1000:])
    gx, gy, gd = dst.GetKangaroos()
    for i in sample(N):
        assert (gx[i], gy[i]) == expected_point(oracle, keys, got, i, gd[i]), i
    src.close(); dst.close()


# ---- the solver ---------------------------------------------------------------------------------------------------------
def resume_line(out):
    m = re.search(r"Resume .*: (\d+) DPs, count 2\^[\d.]+, (\d+) kangaroos in the file for \d+ in the herd, (\d+) of (\d+) keys solved "
                  r"in the file, (\d+) keys left to search", out)
    assert m, out[-3000:]
    return [int(v) for v in m.groups()]


@pytest.fixture(scope="module")
def stopped_run(tmp_path_factory):
    """one GPU, 64 keys of 2^56, stopped with --max-steps after some keys were solved and saved with --batch-save"""
    path = str(tmp_path_factory.mktemp("batch") / "stop.work")
    rc, out = solver([CFG64, "--batch-keys", "--seed", "3", "--max-steps", "120", "--batch-save", path] + GRID)
    assert os.path.exists(path), out[-3000:]
    return path, out


@needs_ingest
@pytest.mark.parametrize("table", ["host", "device"])
def test_batch_resume_finishes_the_keys(stopped_run, table, tmp_path):
    from kangaroo_b200.worktool import read_batch
    path, out1 = stopped_run
    solved1, _, j1 = batch_jumps(out1)
    block = read_batch(path)
    k = sum(block.solved)
    assert 0 < k < 64 and k <= solved1, out1[-3000:]
    for i, done in enumerate(block.solved):
        if done:
            assert block.privs[i] == ANSWERS[i]
    rc, out2 = solver(["--batch-keys", "--batch-resume", path, "--seed", "4", "--dp-table", table, "--grid", "32,128"])
    assert rc == 0, out2[-3000:]
    dps, nwalk, ksolved, nkeys, left = resume_line(out2)
    assert (nwalk, ksolved, nkeys, left) == (32 * 128 * 128, k, 64, 64 - k)   # solved keys are not searched again
    assert "%d kangaroos imported and verified" % nwalk in out2
    assert privs(out2) == dict(enumerate(ANSWERS)), out2[-3000:]          # those of the file printed with the others
    solved2, total, j2 = batch_jumps(out2)
    assert solved2 == total == 64
    assert j2 > j1 and (j2 - j1) % PER_STEP == 0                          # the count goes on from the file's


@needs_ingest
def test_batch_resume_with_the_config_and_on_two_gpus(stopped_run):
    path, _ = stopped_run
    rc, out = solver([CFG64, "--batch-keys", "--batch-resume", path, "--seed", "5", "--grid", "32,128", "--max-steps", "2"])
    assert resume_line(out)[1] == 32 * 128 * 128 and "imported and verified" in out, out[-3000:]
    from tests.ranks_util import solver_on                              # two GPUs, or two ranks sharing one over gloo
    rc, out = solver_on(2, ["--batch-keys", "--batch-resume", path, "--seed", "5", "--grid", "16,128"])
    assert rc == 0, out[-3000:]
    assert privs(out) == dict(enumerate(ANSWERS)), out[-3000:]
    assert out.count("kangaroos imported and verified") == 2


@needs_ingest
def test_interval_save_while_keys_are_solved_passes_the_check(tmp_path):
    """a --batch-save-interval save taken while keys are being solved: every DP and every kangaroo (against its own target)
    checks OK; no wild sits on a key the file shows solved, every unsolved key keeps wilds; one corrupted target fails it"""
    from kangaroo_b200 import solver as S
    from kangaroo_b200 import worktool
    start, end, pubs = ec.parse_config(CFG64)
    path = str(tmp_path / "iv.work")
    copies = []

    class Keep(S.BatchSolver):
        """takes one interval save once a key is announced solved, and keeps a copy of it"""
        def _solved(self, solved):
            done = super()._solved(solved)
            if self.announced and not copies and self.save_interval > 1:
                self.save_interval = 1e-6                      # the next step's save decision takes it
            return done

        def _save_start(self, kangaroos, chunks):
            self.save_interval = 1e9
            super()._save_start(kangaroos, chunks)

        def _on_saved(self, p, mb, seconds, err):              # on the writer thread, right after the rename
            assert err is None
            if not copies:
                shutil.copy(p, str(tmp_path / "copy.work"))
                copies.append(p)

    s = Keep(start, end, pubs, 8, (32, 128), seed=11, save_work=path, save_interval=1e9)
    s.run(200, verbose=False)
    s.close()
    assert copies
    f = str(tmp_path / "copy.work")
    b = worktool.read_batch(f)
    assert 0 < sum(b.solved) < 64, sum(b.solved)
    r = worktool.check(f)
    assert r.ok and r.n_keys == 64 and r.walks == b.nb_walk == 32 * 128 * 128, vars(r)
    assert r.walks_wild == r.walks // 2 and r.entries > 1000
    wild = b.targets[1::2]
    solved = {i for i, v in enumerate(b.solved) if v}
    assert not solved & set(wild.tolist())                                # a solved key has no wild left on it
    assert set(range(64)) - solved <= set(wild.tolist())                  # every unsolved key has wilds
    bad = str(tmp_path / "bad.work")
    raw = bytearray(open(f, "rb").read())
    pos = b.offset + 24 + 64 * 104 + 2 * 4001                             # kangaroo 4001 (wild): another key
    raw[pos] ^= 1
    open(bad, "wb").write(bytes(raw))
    r2 = worktool.check(bad)
    assert not r2.ok and r2.wrong_walks == 1 and r2.wrong_walk_indices == [4001] and r2.wrong_entries == 0
    assert worktool.main(["check", bad]) == 1
    with pytest.raises(ValueError, match="batch work file"):
        worktool.merge_files([f, f], str(tmp_path / "m.work"))
