"""-m gpu: --dp-table sharded.  The partition kernel (kgx_dp_partition) against tests/shard_model.py on crafted records; W
range-limited tables on one GPU fed the partition of tests/dptable_model.py's record streams, against one full table and the
model (events, counts, work-file pieces, loads); and the solver with --dp-table sharded on one GPU and, where two are visible,
on two."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from kangaroo_b200 import worktool as wt
from tests import dptable_model as dm
from tests import shard_model as sm
from tests.ranks_util import solver_on
from tests.worktool_util import NB, ROOT

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")
PRIV56 = "Priv: 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD612C0F05F3DA03"
CAP = 4096


# ---- 1: the partition kernel ------------------------------------------------------------------------------------------------
def run_partition(recs, world, stride=0, skew=0):
    """kgx_dp_partition on the GPU -> (groups, malformed count).  skew: bytes the input and the output start past a 256-byte
    boundary (4: where kgx_convert_dps's records start, after its u32 count)"""
    import torch
    from kangaroo_b200 import load_library
    lib = load_library()
    n = len(recs)
    raw = torch.zeros(skew + max(n, 1) * 40, dtype=torch.uint8)
    raw[skew:skew + 40 * n] = torch.from_numpy(np.ascontiguousarray(recs, np.uint64).view(np.uint8).reshape(-1))
    src = raw.cuda()[skew:]
    rows = world * stride if stride else max(n, 1)
    out = torch.full((skew + rows * 40,), 0xEE, dtype=torch.uint8, device="cuda")[skew:]
    counts = torch.zeros(world + 1, dtype=torch.int32, device="cuda")
    scratch = torch.empty(int(lib.kgx_dp_partition_scratch_bytes(n, world)), dtype=torch.uint8, device="cuda")
    rc = lib.kgx_dp_partition(ctypes.c_void_p(src.data_ptr()), n, world, stride, ctypes.c_void_p(out.data_ptr()),
                              ctypes.c_void_p(counts.data_ptr()), ctypes.c_void_p(scratch.data_ptr()), scratch.numel(),
                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    c = counts.cpu().tolist()
    o = np.frombuffer(out.cpu().numpy().tobytes(), np.uint64).reshape(-1, 5)
    if stride:
        groups = [o[r * stride:r * stride + c[r]] for r in range(world)]
        for r in range(world):                                      # nothing written past a group
            assert (o[r * stride + c[r]:(r + 1) * stride] == np.uint64(0xEEEEEEEEEEEEEEEE)).all()
    else:
        pre = np.concatenate([[0], np.cumsum(c[:world])])
        groups = [o[pre[r]:pre[r + 1]] for r in range(world)]
    return groups, c[world]


def crafted(rng, world, n):
    """n records: random buckets, every boundary's lo-1, lo, hi-1, hi, malformed h, in random order"""
    b = sm.owner_bounds(world)
    edges = sorted({v + d for v in b for d in (-1, 0) if 0 <= v + d < NB})
    h = np.concatenate([rng.integers(0, NB, size=n // 2, dtype=np.uint64), rng.choice(np.asarray(edges, np.uint64), size=n - n // 2 - n // 50),
                        np.uint64(NB) + rng.integers(0, 1 << 31, size=n // 50, dtype=np.uint64)])
    rng.shuffle(h)
    out = rng.integers(0, 1 << 63, size=(n, 5), dtype=np.uint64)
    out[:, 0] = (h << np.uint64(32)) | np.arange(n, dtype=np.uint64)
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 8, 256])
def test_partition_kernel_matches_the_model(world):
    rng = np.random.default_rng(world)
    for n in (0, 1, 255, 256, 257, 1000, 77777):
        recs = crafted(rng, world, n)
        want, bad = sm.partition(recs, world)
        for stride, skew in ((0, 0), (n + 3, 0), (0, 4), (n + 1, 4)):
            got, gbad = run_partition(recs, world, stride, skew)
            assert gbad == bad
            assert [g.tobytes() for g in got] == [w.tobytes() for w in want], (n, stride, skew)
    one = crafted(rng, world, 5000)                                  # every record to one owner
    r = world // 2
    lo, hi = owner_ranges_of(world, r)
    one[:, 0] = (rng.integers(lo, hi, size=len(one), dtype=np.uint64) << np.uint64(32)) | (one[:, 0] & np.uint64(0xFFFFFFFF))
    got, bad = run_partition(one, world)
    assert bad == 0 and got[r].tobytes() == one.tobytes() and all(len(g) == 0 for i, g in enumerate(got) if i != r)


def owner_ranges_of(world, r):
    b = sm.owner_bounds(world)
    return b[r], b[r + 1]


# ---- 2: W shards on one GPU against one table -----------------------------------------------------------------------------
def upload(segments, stride):
    import torch
    flat = np.zeros((max(1, len(segments) * stride), 5), np.uint64)
    for r, seg in enumerate(segments):
        flat[r * stride:r * stride + len(seg)] = seg
    return torch.from_numpy(flat.view(np.uint8).reshape(-1)).cuda()


def ev_tuples(evs, n):
    raw = ctypes.string_at(ctypes.addressof(evs), 48 * n)
    w32, w64 = np.frombuffer(raw, np.uint32).reshape(n, 12).tolist(), np.frombuffer(raw, np.uint64).reshape(n, 6).tolist()
    return [(a[0], a[1], a[2], a[3], (b[2], b[3]), (b[4], b[5])) for a, b in zip(w32, w64)]


def add(table, segments):
    stride = max(len(s) for s in segments) + 1
    buf = upload(segments, stride)
    rc, n, evs = table.add_raw(buf.data_ptr(), [len(s) for s in segments], stride)
    assert rc == 0
    return ev_tuples(evs, n)


def file_of_pieces(shards, path):
    """the pieces of the shards at their offsets under one header, as the solver assembles a work file"""
    from kangaroo_b200 import solver as S
    a = dm.save_args()
    with open(path, "wb") as f:
        f.write(S.work_header(a["dp_bits"], a["range_start"], a["range_end"], a["pubkey"], a["total_count"], a["total_time"]))
    offs = S.piece_offsets([s.piece_bytes() for s in shards])
    for s, o in zip(shards, offs):
        s.save_piece(path, o)
    with open(path, "r+b") as f:
        f.seek(offs[-1])
        f.write(np.uint64(0).tobytes())
    return open(path, "rb").read()


@pytest.mark.parametrize("world", [2, 3, 8])
def test_emulated_shards_equal_one_table(world, tmp_path):
    from kangaroo_b200.ingest import DeviceDPTable
    adv = dm.Adversary(world, CAP)
    bounds = sm.owner_bounds(world)
    full = DeviceDPTable(CAP, max_events=1 << 14)
    shards = [DeviceDPTable(CAP, max_events=1 << 14, buckets=(bounds[r], bounds[r + 1])) for r in range(world)]
    model = dm.HashTableModel()
    recs = np.concatenate([r for _, r in adv.classes()] + [adv.random(300)])
    for segments in adv.calls(recs, ncalls=4, nsegs=world + 1):
        want, skipped = model.add(segments)
        assert skipped == 0
        got_full = add(full, segments)
        assert got_full == want
        got = []
        for d, segs in enumerate(sm.arrivals(segments, world)):
            if sum(len(s) for s in segs):
                got += add(shards[d], segs)
            assert len(shards[d]) == sum(len(b) for h, b in model.ent.items() if bounds[d] <= h < bounds[d + 1])
        assert sorted(got) == sorted(want)
        assert sum(len(s) for s in shards) == len(full) == len(model)
    one = str(tmp_path / "full.work")
    full.save_work(one, **dm.save_args())
    raw = open(one, "rb").read()
    assert raw == model.to_work().to_bytes()
    assert file_of_pieces(shards, str(tmp_path / "pieces.work")) == raw
    again = [DeviceDPTable(CAP, buckets=(bounds[r], bounds[r + 1])) for r in range(world)]
    for s in again:
        w = s.load_piece(one, CAP)
        assert w.nb_walk == 0 and w.walk_offset == len(raw)
    assert [len(s) for s in again] == [len(s) for s in shards]
    assert file_of_pieces(again, str(tmp_path / "again.work")) == raw
    from kangaroo_b200.ingest import TableFull
    biggest = int(np.argmax([len(s) for s in shards]))
    with pytest.raises(TableFull, match="hold more than"):
        again[biggest].load_piece(one, len(shards[biggest]) - 1)
    for t in [full] + shards + again:
        t.close()


# ---- 3: the solver ----------------------------------------------------------------------------------------------------------
def solver(args, timeout=900, prefix=None):
    p = subprocess.run((prefix or [sys.executable]) + ["-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT)
    return p.returncode, p.stdout + p.stderr


SH = ["--dp-table", "sharded"]


@needs_ingest
def test_solver_sharded_in56_and_puzzle110_window():
    rc, out = solver([os.path.join(GOLD, "in56.txt"), "--dp", "8", "--grid", "32,128", "--seed", "7", "--dp-table-capacity",
                      str(1 << 24)] + SH)
    assert rc == 0 and PRIV56 in out, out[-2000:]
    assert "dp table: sharded over 1 GPUs, 16777216 entries in all" in out and "sharded table" in out, out[-2000:]
    rc, out = solver([os.path.join(GOLD, "puzzle110_window56.txt"), "--dp", "8", "--grid", "32,128", "--seed", "11"] + SH)
    assert rc == 0 and "Priv: 0x35C0D7234DF7DEB0F20CF7062444" in out, out[-2000:]


def batch_ok(rc, out):
    answers = [int(v, 16) for v in open(os.path.join(GOLD, "in56_64keys.answers.txt")).read().split()]
    assert rc == 0, out[-3000:]
    privs = {int(i): int(v, 16) for i, v in re.findall(r"Key#\s*(\d+) Pub:\s+0x[0-9A-F]+\s+Priv: 0x([0-9A-F]+)", out)}
    assert privs == dict(enumerate(answers)), out[-3000:]


@needs_ingest
def test_solver_sharded_batch_keys():
    rc, out = solver([os.path.join(GOLD, "in56_64keys.txt"), "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "3"] + SH)
    batch_ok(rc, out)


COMMON = ["--dp", "8", "--grid", "8,32", "--seed", "5", "--save-kangaroos"]


@needs_ingest
def test_solver_sharded_resumes_host_files_and_host_resumes_its_files(tmp_path):
    cfg = os.path.join(GOLD, "in56.txt")
    host, sh = str(tmp_path / "host.work"), str(tmp_path / "sh.work")
    rc, out = solver([cfg, "--max-steps", "4", "--save-work", host] + COMMON)
    assert os.path.exists(host), out[-2000:]
    rc, out = solver([cfg, "--max-steps", "4", "--save-work", sh] + COMMON + SH + ["--dp-table-capacity", str(1 << 22)])
    assert os.path.exists(sh) and "work file written" in out, out[-2000:]
    rh, rs = open(host, "rb").read(), open(sh, "rb").read()
    assert rh[:140] == rs[:140]
    if " 0 dead kangaroos re-created" in out:
        assert rh[156:] == rs[156:]                                 # the same file past the header's run time
    r = wt.check(sh)
    assert r.ok and r.walks == 8 * 32 * 128
    rc, out = solver(["--resume", host, "--grid", "16,32", "--seed", "2"] + SH)
    assert "imported and verified" in out and PRIV56 in out, out[-2000:]
    rc, out = solver(["--resume", sh, "--grid", "16,32", "--seed", "2"])
    assert "imported and verified" in out and PRIV56 in out, out[-2000:]


@needs_ingest
def test_saves_of_a_herd_of_several_chunks_beside_the_steps(tmp_path):
    """a save on every step of a herd of two gather chunks (2^18 kangaroos each): the chunks move as rank 0's writer frees its
    buffers, during the run and in the end-of-run drain, while that writer waits for the pieces' offsets"""
    f = str(tmp_path / "c.work")
    rc, out = solver([os.path.join(GOLD, "in80.txt"), "--max-steps", "8", "--save-work", f, "--save-interval", "1e-6", "--dp", "8",
                      "--grid", "32,128", "--seed", "5", "--save-kangaroos", "--dp-table-capacity", str(1 << 23)] + SH)
    assert "work file written" in out and out.count("SaveWork") >= 2 and "failed" not in out, out[-2000:]
    r = wt.check(f)
    assert r.ok and r.walks == 32 * 128 * 128 and r.walks_tame == r.walks_wild


@needs_ingest
def test_a_full_shard_stops_the_run_with_kangaroos_in_its_file(tmp_path):
    """a capacity a few launches above the headroom: the run stops at the headroom and writes the normal end-of-run cut, with
    kangaroos, that the check passes and a larger table or the host table resume to the key"""
    cfg = os.path.join(GOLD, "in56.txt")
    a = str(tmp_path / "full.work")
    per_launch = 8 * 32 * 128 * 64 // 256                          # DPs of one launch at dp 8, on average
    cap = 2 * (1 << 17) + 4 * per_launch
    rc, out = solver([cfg, "--save-work", a, "--dp-table-capacity", str(cap)] + COMMON + SH)
    assert rc == 1 and "DP table shard full, run stopped: shard 0 of 1" in out and "of its capacity %d" % cap in out, out[-2000:]
    assert "work file written" in out, out[-2000:]
    r = wt.check(a)
    assert r.ok and r.walks == 8 * 32 * 128 and 0 < r.entries <= cap
    rc, out = solver(["--resume", a, "--grid", "8,32", "--seed", "2"] + SH)
    assert "imported and verified" in out and PRIV56 in out, out[-2000:]
    rc, out = solver(["--resume", a, "--grid", "8,32", "--seed", "2"])
    assert "imported and verified" in out and PRIV56 in out, out[-2000:]


@needs_ingest
def test_resume_file_too_large_for_the_shard_is_refused(tmp_path):
    cfg = os.path.join(GOLD, "in80.txt")
    a = str(tmp_path / "a.work")
    solver([cfg, "--max-steps", "3", "--save-work", a] + COMMON)
    r = wt.check(a)
    cap = 2 * (1 << 17) + r.entries - 1
    rc, out = solver(["--resume", a, "--grid", "8,32", "--seed", "2", "--max-steps", "5", "--dp-table-capacity", str(cap)] + SH)
    assert rc != 0 and "of shard 0 hold more than its capacity %d less the stop headroom" % cap in out, out[-2000:]
    assert "imported and verified" not in out and "MJump/s" not in out


# ---- 4: two ranks: two GPUs, or two ranks sharing one over gloo (tests/ranks_util.py) ----------------------------------------
@needs_ingest
def test_two_shards_solve_and_their_files_cross_tables(tmp_path):
    rc, out = solver_on(2, [os.path.join(GOLD, "puzzle110_window56.txt"), "--dp", "8", "--grid", "32,128", "--seed", "11",
                            "--dp-table-capacity", str(1 << 24)] + SH)
    assert rc == 0 and "Priv: 0x35C0D7234DF7DEB0F20CF7062444" in out and "GPUs: 2" in out, out[-3000:]
    rc, out = solver_on(2, [os.path.join(GOLD, "in56_64keys.txt"), "--batch-keys", "--dp", "8", "--grid", "32,128", "--seed", "3",
                            "--dp-table-capacity", str(1 << 25)] + SH)
    batch_ok(rc, out)
    cfg = os.path.join(GOLD, "in56.txt")
    sh, host = str(tmp_path / "sh.work"), str(tmp_path / "host.work")
    rc, out = solver_on(2, [cfg, "--max-steps", "40", "--save-work", sh, "--save-interval", "0.05", "--dp-table-capacity",
                            str(1 << 22)] + COMMON + SH)
    assert os.path.exists(sh) and "SaveWork" in out, out[-3000:]
    r = wt.check(sh)
    assert r.ok and r.walks == 2 * 8 * 32 * 128
    rc, out = solver(["--resume", sh, "--grid", "16,32", "--seed", "2"])
    assert "imported and verified" in out and PRIV56 in out, out[-2000:]
    solver([cfg, "--max-steps", "4", "--save-work", host] + COMMON)
    rc, out = solver_on(2, ["--resume", host, "--grid", "16,32", "--seed", "2", "--dp-table-capacity", str(1 << 24)] + SH)
    assert "imported and verified" in out and PRIV56 in out, out[-3000:]
    from kangaroo_b200.ingest import DeviceDPTable
    t = DeviceDPTable(1 << 22)
    w = t.load_work_ex(sh)
    again = str(tmp_path / "again.work")
    t.save_work(again, w.dp_bits, w.range_start, w.range_end, w.key, w.total_count, w.total_time, 0)
    t.close()
    raw, ref = open(again, "rb").read(), open(sh, "rb").read()
    assert raw[156:-8] == ref[156:w.walk_offset - 8]               # the same table bytes
