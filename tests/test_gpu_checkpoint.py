"""-m gpu: the herd as work-file records on the device (kgx_snapshot_export / kgx_import) and the stand-alone solver's
checkpoint / resume (--save-work --save-kangaroos --save-interval --resume)."""
import gzip
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
DROPIN = os.path.join(ROOT, "build", "kangaroo_b200")
GOLD = os.path.join(ROOT, "tests", "golden")
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")


def rec_ints(recs):
    return [tuple(sum(int(r[4 * k + j]) << (64 * j) for j in range(4)) for k in range(3)) for r in recs]


def garbage_engine(kernel, wo, seed=1):
    """3 x 32 x 128 = 12288 kangaroos (padded tiles on every kernel) with random coordinates and biased distances, many of
    the wild ones below the wild offset (they wrap below zero mod n on export)."""
    from kangaroo_b200 import GPUEngine
    eng = GPUEngine(3, 32, 0, 65536, **kernel)
    n = eng.nbKangaroo
    rng = np.random.default_rng(seed)
    ax = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64)
    ay = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.uint64)
    ad = rng.integers(0, 1 << 63, size=(n, 2), dtype=np.uint64)
    ad[::3, 1] = 0                                                     # small: below the offset
    eng.SetWildOffset(wo)
    eng.SetKangaroosRaw(ax, ay, ad)
    return eng


def test_export_equals_get_kangaroos_and_import_restores_the_state(oracle, kernel):
    wo = (1 << 100) + 12345
    eng = garbage_engine(kernel, wo)
    n = eng.nbKangaroo
    eng.SetParams(oracle.dp_mask(8), *oracle.create_jump_table(64))
    eng.callKernel()
    eng.SnapshotBegin()                                                # stream order: after the launch in flight
    recs = np.empty((n, 12), dtype=np.uint64)
    for first in range(0, n, 5000):                                    # chunks that do not divide n
        c = min(5000, n - first)
        eng.SnapshotExport(first, c, recs[first:first + c])
    eng.sync()
    gx, gy, gd = eng.GetKangaroos()
    assert rec_ints(recs) == list(zip(gx, gy, gd))
    assert any(d > (1 << 128) for d in gd[1::2])                       # wild distances that wrapped below zero mod n
    raw = eng.GetKangaroosRaw()
    # scramble the herd with more launches, then import the export: the state is back bit for bit
    eng.callKernelAndWait()
    assert eng.ImportKangaroos(recs, (1, 2), verify=False) == 0
    for a, b in zip(eng.GetKangaroosRaw(), raw):
        assert np.array_equal(a, b)
    # a distance that does not fit the biased 128-bit form fails the call and changes nothing
    eng.callKernelAndWait()
    before = eng.GetKangaroosRaw()
    bad = recs.copy()
    bad[4097, 10] = 1                                                  # d >= 2^128 (a wild kangaroo)
    with pytest.raises(RuntimeError, match="record 4097"):
        eng.ImportKangaroos(bad, (1, 2), verify=False)
    for a, b in zip(eng.GetKangaroosRaw(), before):
        assert np.array_equal(a, b)
    eng.close()


def test_import_verification_and_partial_import(oracle):
    from kangaroo_b200 import GPUEngine
    from kangaroo_b200.engine import random_herd_arrays
    rp = 80
    wdiv2 = ((1 << rp) - 1) >> 1
    key = oracle.ec_mul_g(0x1D0C8E2F4A5B6C7D8E9F0A1B2C3D4E5F60718293A4B5C6D7E8F9)
    other = oracle.ec_mul_g(0x777)
    eng = GPUEngine(2, 16, 0, 65536, kernel="stream")
    n = eng.nbKangaroo
    eng.SetWildOffset(wdiv2)
    sc, d128 = random_herd_arrays(n, rp, wdiv2, np.random.default_rng(3))
    eng.CreateHerdRaw(sc, d128, key)
    eng.SnapshotBegin()
    recs = eng.SnapshotExport(0, n)
    assert eng.ImportKangaroos(recs, key) == 0
    flipped = recs.copy()
    for i in (3, 100, n - 1):
        flipped[i, 1] ^= np.uint64(1 << 17)                           # one bit of x
    state = eng.GetKangaroosRaw()
    assert eng.ImportKangaroos(flipped, key) == 3
    for a, b in zip(eng.GetKangaroosRaw(), state):                     # a failed verification changes nothing
        assert np.array_equal(a, b)
    # against another key every wild kangaroo (key + d*G) fails; tame ones (d*G) do not depend on the key
    assert eng.ImportKangaroos(recs, other) == n // 2
    # a herd built for the other key: its kangaroos 0..999 replace ours, the rest stays
    eng2 = GPUEngine(2, 16, 0, 65536, kernel="stream")
    eng2.SetWildOffset(wdiv2)
    sc2, d2 = random_herd_arrays(n, rp, wdiv2, np.random.default_rng(4))
    eng2.CreateHerdRaw(sc2, d2, other)
    eng2.SnapshotBegin()
    recs2 = eng2.SnapshotExport(0, n)
    assert eng.ImportKangaroos(recs2[:1000], key) == 500
    assert eng.ImportKangaroos(recs2[:1000], other) == 0
    ax, ay, ad = eng.GetKangaroosRaw()
    bx, by, bd = eng2.GetKangaroosRaw()
    assert np.array_equal(ax[:1000], bx[:1000]) and np.array_equal(ad[:1000], bd[:1000])
    assert np.array_equal(ax[1000:], state[0][1000:]) and np.array_equal(ad[1000:], state[2][1000:])
    eng.close(); eng2.close()


def test_symmetric_mode_refuses_both():
    from kangaroo_b200 import GPUEngine
    eng = GPUEngine(2, 16, 0, 65536, kernel="resident")
    eng.SetSymmetry("symclass")
    eng.SetKangaroosRaw(np.ones((eng.nbKangaroo, 4), np.uint64), np.ones((eng.nbKangaroo, 4), np.uint64), np.ones((eng.nbKangaroo, 2), np.uint64))
    eng.SnapshotBegin()
    with pytest.raises(RuntimeError, match="symmetric"):
        eng.SnapshotExport(0, 10)
    eng.SnapshotRead()
    with pytest.raises(RuntimeError, match="symmetric"):
        eng.ImportKangaroos(np.zeros((10, 12), np.uint64), (1, 2), verify=False)
    eng.close()


# ---- the solver --------------------------------------------------------------------------------------------------------
def solver(args, timeout=900):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    out = p.stdout + p.stderr
    assert p.returncode in (0, 1), out[-3000:]
    return out


def split(path):
    from kangaroo_b200.ingest import DPTable
    t = DPTable(threads=1)
    w = t.load_work_ex(path)
    t.close()
    raw = open(path, "rb").read()
    return raw[:140], w.total_count, raw[156:w.walk_offset], raw[w.walk_offset:], w


COMMON = ["--dp", "8", "--grid", "8,32", "--seed", "5", "--save-kangaroos"]


@needs_ingest
def test_resume_continues_the_straight_run_bit_for_bit(tmp_path):
    cfg = os.path.join(GOLD, "in80.txt")
    a, a2, b = (str(tmp_path / f) for f in ("a.work", "a2.work", "b.work"))
    K = 20
    out_a = solver([cfg, "--max-steps", str(K), "--save-work", a] + COMMON)
    out_a2 = solver(["--resume", a, "--max-steps", str(K), "--save-work", a2] + COMMON)
    out_b = solver([cfg, "--max-steps", str(2 * K + 1), "--save-work", b] + COMMON)
    for out in (out_a, out_a2, out_b):
        assert " 0 dead kangaroos re-created" in out, out[-2000:]
    assert "imported and verified" in out_a2, out_a2[-2000:]
    ha, ca, ta, ka, wa = split(a2)
    hb, cb, tb, kb, wb = split(b)
    assert wa.nb_walk == wb.nb_walk == 8 * 32 * 128
    assert ca == cb == 42 * 8 * 32 * 128 * 64                           # (K+1) + (K+1) launches == 2K+2
    assert ha == hb and ta == tb and ka == kb
    # the reference's own checker accepts every DP of the solver's file
    if os.path.exists(DROPIN):
        chk = subprocess.run([DROPIN, "-wcheck", a2], capture_output=True, text=True, timeout=600, cwd=ROOT).stdout
        assert "[100.000% OK]" in chk and "Wrong" not in chk, chk[-1500:]


@needs_ingest
def test_mid_run_save_is_the_end_save_of_a_shorter_run(tmp_path):
    """A --save-interval save equals, byte for byte past the header's time, the end-of-run save of a straight run stopped at
    that file's count."""
    from kangaroo_b200 import solver as S
    start, end, pubs = ec.parse_config(os.path.join(GOLD, "in80.txt"))
    path = str(tmp_path / "m.work")
    copies = []

    class Keep(S.Solver):
        def _on_saved(self, p, mb, seconds, err):              # on the writer thread, right after the rename
            assert err is None
            copies.append(open(p, "rb").read())

    s = Keep(start, end, pubs[0], 8, (8, 32), seed=9, save_work=path, save_interval=1e-6, save_kangaroos=True)
    s.run(12, verbose=False)
    s.close()
    assert len(copies) >= 3 and s.same_herd == 0
    mid = str(tmp_path / "mid.work")
    open(mid, "wb").write(copies[len(copies) // 2])
    hm, cm, tm, km, _ = split(mid)
    launches = cm // (8 * 32 * 128 * 64)
    straight = str(tmp_path / "s.work")
    out = solver([os.path.join(GOLD, "in80.txt"), "--max-steps", str(launches - 1), "--save-work", straight, "--dp", "8",
                  "--grid", "8,32", "--seed", "9", "--save-kangaroos"])
    assert " 0 dead kangaroos re-created" in out
    hs, cs, ts, ks, _ = split(straight)
    assert cs == cm and hm == hs and tm == ts and km == ks


@needs_ingest
def test_resume_the_reference_written_fixture_finds_the_key(tmp_path):
    from tests.golden import make_work_golden as g
    path = str(tmp_path / "ref.work")
    with gzip.open(os.path.join(GOLD, "ref_work48.work.gz"), "rb") as src, open(path, "wb") as dst:
        shutil.copyfileobj(src, dst)
    out = solver(["--resume", path, "--grid", "8,32", "--seed", "1", "--dp", "10", "--max-steps", "20000"], timeout=600)
    assert "1024 kangaroos imported and verified" in out, out[-2000:]
    assert "Priv: 0x%X" % g.PRIV in out, out[-2000:]


@needs_ingest
@pytest.mark.skipif(not os.path.exists(DROPIN), reason="build/kangaroo_b200 not built")
def test_reference_program_resumes_a_solver_file(tmp_path):
    work = str(tmp_path / "s56.work")
    out = solver([os.path.join(GOLD, "in56.txt"), "--max-steps", "4", "--save-work", work] + COMMON)
    assert os.path.exists(work), out[-2000:]
    p = subprocess.run([DROPIN, "-t", "0", "-gpu", "-g", "16,128", "-i", work], capture_output=True, text=True, timeout=900, cwd=ROOT)
    out2 = p.stdout + p.stderr
    assert "CD612C0F05F3DA03" in out2.upper().replace(" ", ""), out2[-2000:]


@needs_ingest
def test_two_gpu_checkpoint_resumes_on_one_gpu(tmp_path):
    """two GPUs, or two ranks sharing one over gloo"""
    from tests.ranks_util import solver_on
    work = str(tmp_path / "two.work")
    rc, out = solver_on(2, [os.path.join(GOLD, "in56.txt"), "--max-steps", "4", "--save-work", work] + COMMON)
    assert os.path.exists(work), out[-2000:]
    out = solver(["--resume", work, "--grid", "16,32", "--seed", "2"])
    assert "%d kangaroos imported and verified" % (2 * 8 * 32 * 128) in out, out[-2000:]
    assert "Priv: 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD612C0F05F3DA03" in out, out[-2000:]


@needs_ingest
@pytest.mark.skipif(not os.path.exists(DROPIN), reason="build/kangaroo_b200 not built")
def test_solver_resumes_a_reference_program_file(tmp_path):
    """`build/kangaroo_b200 -w f -wi 1 -ws` (the reference's SaveWork with kangaroos) -> `solver --resume f`: every kangaroo
    verifies and the puzzle-110 key is found."""
    work = str(tmp_path / "d.work")
    cfg = os.path.join(GOLD, "puzzle110_window72.txt")
    out1 = ""
    for attempt in range(3):                                          # a lucky run may solve before the first save
        p = subprocess.run([DROPIN, "-t", "0", "-gpu", "-g", "32,128", "-d", "14", "-w", work, "-wi", "1", "-ws", "-m", "0.25", cfg],
                           capture_output=True, text=True, timeout=600, cwd=ROOT)
        out1 = p.stdout + p.stderr
        if os.path.exists(work) and "Aborted" in out1:
            break
    assert os.path.exists(work) and "Aborted" in out1, out1[-2000:]
    n = 32 * 128 * 128
    out = solver(["--resume", work, "--grid", "32,128", "--seed", "3"])
    assert "%d kangaroos imported and verified" % n in out, out[-2000:]
    assert "Priv: 0x35C0D7234DF7DEB0F20CF7062444" in out, out[-2000:]


@needs_ingest
def test_failed_save_is_reported_and_leaves_no_tmp(tmp_path):
    plain = tmp_path / "plain"
    plain.write_bytes(b"x")
    work = str(plain / "w.work")                                     # ENOTDIR
    out = solver([os.path.join(GOLD, "in80.txt"), "--max-steps", "5", "--save-work", work, "--save-interval", "1e-6"] + COMMON)
    assert "SaveWork %s failed" % work in out and "work file NOT written" in out, out[-2000:]
    assert os.listdir(str(tmp_path)) == ["plain"]
