"""-m gpu: the multi-rank solver on one GPU.  W = 2, 3, 4 ranks share device 0 over gloo (tests/ranks_util.py), so every path
that crosses ranks runs: the DP gather to rank 0, the sharded table's exchange, per-step blocks and stop, work-file pieces
written by every rank at their offsets, the herd gather of a save, the resume scatter, per-rank range loads of a file written
at another world size, and the control broadcast that sends dead kangaroos back to their owners.  The reference's HashTable
(build/libkgx_ingest.so, --dp-table host) is the yardstick: the device and sharded tables promise its events and its file
bytes.  Every multi-rank run passes --dp-table-capacity: ranks sharing a GPU would otherwise each size a table from the free
memory of that one device."""
import os
import re
import struct
import subprocess
import sys

import numpy as np
import pytest

from kangaroo_b200 import worktool as wt
from kangaroo_b200.dist import owner_ranges
from tests.ranks_util import ROOT, run_ranks

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
IN56, IN80 = os.path.join(GOLD, "in56.txt"), os.path.join(GOLD, "in80.txt")
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")
PRIV56 = "Priv: 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD612C0F05F3DA03"
HERD = 8 * 32 * 128                     # kangaroos of one rank at --grid 8,32
MAX_FOUND = 1 << 17
SH = ["--dp-table", "sharded"]
DEAD = re.compile(r"(\d+) dead kangaroos re-created \((\d+) reported by the table, at most (\d+) in one step\)")


def headroom(world):
    return 2 * world * MAX_FOUND        # solver.shard_headroom


def cap(n):
    return ["--dp-table-capacity", str(n)]


def ranks(world, args, timeout=400):
    """the solver on W ranks sharing device 0 (one plain process for W = 1) -> (exit codes, outputs) in rank order"""
    if world == 1:
        p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True, timeout=timeout,
                           cwd=ROOT)
        return [p.returncode], [p.stdout + p.stderr]
    return run_ranks(world, args, timeout)


def stepped(rcs):
    """a run that ends at --max-steps: rank 0 exits 1 (key not found) or 0 (found), every other rank 0"""
    return rcs[0] in (0, 1) and rcs[1:] == [0] * (len(rcs) - 1)


def show(outs):
    return "".join("--- rank %d ---\n%s" % (r, o[-2500:]) for r, o in enumerate(outs))


def clean(outs):
    """no rank reported malformed records or a failed table"""
    for o in outs:
        assert "malformed" not in o and "DP table failed" not in o and "Traceback" not in o, show(outs)


def table_end(raw):
    """-> (the offset where a HEADW file's table ends, entries per bucket)"""
    sizes, o = np.zeros(1 << 18, np.int64), 156
    for h in range(1 << 18):
        n = struct.unpack_from("<I", raw, o)[0]
        sizes[h] = n
        o += 8 + 32 * n
    return o, sizes


def shard_entries(path, world):
    """entries of each rank's buckets in the file's table"""
    _, sizes = table_end(open(path, "rb").read())
    return [int(sizes[lo:hi].sum()) for lo, hi in owner_ranges(world)]


def dead(out):
    m = DEAD.search(out)
    assert m, out[-2500:]
    return tuple(int(v) for v in m.groups())          # (re-created on every rank, reported, most in one step)


# ---- a: the sharded and device tables against the reference table, on W ranks ----------------------------------------------
@needs_ingest
@pytest.mark.parametrize("world", [2, 3, 4])
def test_shards_write_the_reference_tables_file(world, tmp_path):
    """one seed, three tables: the files agree from byte 156 on (the table, the kangaroo count, every rank's herd in rank
    order); W = 3 splits the 2^18 buckets unevenly"""
    files = {}
    for table, extra in (("host", []), ("device", cap(1 << 21)), ("sharded", cap(1 << 21))):
        f = files[table] = str(tmp_path / ("%s.work" % table))
        rcs, outs = ranks(world, [IN80, "--dp", "10", "--grid", "8,32", "--seed", "21", "--max-steps", "6", "--save-work", f,
                                  "--save-kangaroos", "--dp-table", table] + extra)
        assert stepped(rcs), show(outs)
        clean(outs)
        assert "GPUs: %d" % world in outs[0] and "work file written" in outs[0], show(outs)
        assert dead(outs[0])[:2] == (0, 0), outs[0][-2500:]
    raw = {t: open(f, "rb").read() for t, f in files.items()}
    assert raw["host"][:140] == raw["device"][:140] == raw["sharded"][:140]
    assert raw["host"][156:] == raw["device"][156:] == raw["sharded"][156:]
    r = wt.check(files["sharded"])
    assert r.ok and r.walks == world * HERD and r.walks_tame == r.walks_wild and r.entries > 0


# ---- b: a save on every step of three shards --------------------------------------------------------------------------------
@needs_ingest
def test_three_shards_save_on_every_step(tmp_path):
    from kangaroo_b200.ingest import DeviceDPTable
    f = str(tmp_path / "every.work")
    rcs, outs = ranks(3, [IN80, "--dp", "10", "--grid", "8,32", "--seed", "4", "--max-steps", "12", "--save-work", f,
                          "--save-interval", "1e-6", "--save-kangaroos"] + SH + cap(1 << 21))
    assert stepped(rcs), show(outs)
    clean(outs)
    assert outs[0].count("SaveWork %s:" % f) >= 3 and "failed" not in outs[0] and "work file written" in outs[0], show(outs)
    assert sorted(os.listdir(str(tmp_path))) == ["every.work"]                 # no FILE.tmp left
    r = wt.check(f)
    assert r.ok and r.walks == 3 * HERD and r.walks_tame == r.walks_wild
    t = DeviceDPTable(1 << 21)                                                 # the table again, through one device table
    w = t.load_work_ex(f)
    again = str(tmp_path / "again.work")
    t.save_work(again, w.dp_bits, w.range_start, w.range_end, w.key, w.total_count, w.total_time, 0)
    t.close()
    a, ref = open(again, "rb").read(), open(f, "rb").read()
    assert a[156:-8] == ref[156:w.walk_offset - 8]


# ---- c: a full shard stops every rank -----------------------------------------------------------------------------------------
@needs_ingest
def test_a_full_shard_stops_every_rank_and_its_file_resumes(tmp_path):
    """W = 4.  A short run's file gives each shard's entries after K + 1 launches; a capacity of the headroom plus the largest
    of them less one stops exactly that shard (not rank 0 at this seed) at step K + 1, before any other"""
    K, seed = 3, "6"
    args = [IN56, "--dp", "8", "--grid", "8,32", "--seed", seed, "--save-kangaroos"] + SH
    probe = str(tmp_path / "probe.work")
    rcs, outs = ranks(4, args + ["--max-steps", str(K), "--save-work", probe] + cap(1 << 22))
    assert stepped(rcs), show(outs)
    per = shard_entries(probe, 4)
    full = int(np.argmax(per))
    assert full != 0 and sorted(per)[-2] < per[full] - 1, per                  # pinned: one shard, not rank 0's, is the largest
    c = headroom(4) + per[full] - 1
    f = str(tmp_path / "full.work")
    rcs, outs = ranks(4, args + ["--save-work", f] + cap(c))
    assert rcs[0] == 1 and rcs[1:] == [0, 0, 0], show(outs)                     # every rank exits
    clean(outs)
    assert "DP table shard full, run stopped: shard %d of 4 (buckets [%d, %d))" % ((full,) + owner_ranges(4)[full]) in outs[0], show(outs)
    assert "of its capacity %d" % c in outs[0] and "work file written" in outs[0], show(outs)
    r = wt.check(f)
    assert r.ok and r.walks == 4 * HERD and 0 < r.entries <= c, vars(r)
    assert struct.unpack_from("<Q", open(f, "rb").read(), 140)[0] == (K + 2) * 4 * HERD * 64  # stopped at step K + 1
    rcs, outs = ranks(2, ["--resume", f, "--grid", "16,32", "--seed", "2"] + SH + cap(1 << 22))
    assert rcs == [0, 0] and "imported and verified" in outs[1] and PRIV56 in outs[0], show(outs)
    rcs, outs = ranks(1, ["--resume", f, "--grid", "32,32", "--seed", "2"])
    assert rcs == [0] and "%d kangaroos imported and verified" % (4 * HERD) in outs[0] and PRIV56 in outs[0], show(outs)


# ---- d, e: files across world sizes ----------------------------------------------------------------------------------------
W3_SEED = "8"


@pytest.fixture(scope="module")
def w3_file(tmp_path_factory):
    """in56 on three shards, 5 launches, with its herds"""
    if not os.path.exists(INGEST):
        pytest.skip("build/libkgx_ingest.so not built")
    f = str(tmp_path_factory.mktemp("w3") / "w3.work")
    rcs, outs = ranks(3, [IN56, "--dp", "8", "--grid", "8,32", "--seed", W3_SEED, "--max-steps", "4", "--save-work", f,
                          "--save-kangaroos"] + SH + cap(1 << 22))
    assert stepped(rcs) and "work file written" in outs[0], show(outs)
    clean(outs)
    return f


@needs_ingest
def test_range_loads_at_other_world_sizes_reassemble_the_table(w3_file, tmp_path):
    """the W = 3 file loaded by the shards of W = 2 and W = 4, whose bucket boundaries differ from the writers': their pieces
    at their offsets are the file's table byte for byte"""
    from kangaroo_b200 import solver as S
    from kangaroo_b200.ingest import DeviceDPTable
    raw = open(w3_file, "rb").read()
    end, _ = table_end(raw)
    for world in (2, 4):
        shards = [DeviceDPTable(1 << 20, buckets=b) for b in owner_ranges(world)]
        for s in shards:
            s.load_piece(w3_file, 1 << 20)
        assert [len(s) for s in shards] == shard_entries(w3_file, world)
        path = str(tmp_path / ("w%d.work" % world))
        open(path, "wb").write(raw[:156])
        offs = S.piece_offsets([s.piece_bytes() for s in shards])
        for s, o in zip(shards, offs):
            s.save_piece(path, o)
        assert offs[-1] == end and open(path, "rb").read()[156:] == raw[156:end]
        for s in shards:
            s.close()


@needs_ingest
@pytest.mark.parametrize("world,grid,table", [(2, "12,32", SH + cap(1 << 22)), (4, "6,32", SH + cap(1 << 22)),
                                              (1, "24,32", ["--dp-table", "device"] + cap(1 << 23))])
def test_three_shard_file_resumes_at_other_world_sizes(w3_file, world, grid, table):
    rcs, outs = ranks(world, ["--resume", w3_file, "--grid", grid, "--seed", "2"] + table)
    assert rcs == [0] * world, show(outs)
    clean(outs)
    assert sum(int(m) for o in outs for m in re.findall(r"rank \d+: (\d+) kangaroos imported and verified", o)) == 3 * HERD, show(outs)
    assert PRIV56 in outs[0], show(outs)


@needs_ingest
def test_one_rank_host_file_resumes_on_three_shards(tmp_path):
    f = str(tmp_path / "host.work")
    rcs, outs = ranks(1, [IN56, "--dp", "8", "--grid", "24,32", "--seed", "3", "--max-steps", "4", "--save-work", f,
                          "--save-kangaroos"])
    assert stepped(rcs) and "work file written" in outs[0], outs[0][-2500:]
    rcs, outs = ranks(3, ["--resume", f, "--grid", "8,32", "--seed", "2"] + SH + cap(1 << 22))
    assert rcs == [0, 0, 0], show(outs)
    clean(outs)
    assert all("%d kangaroos imported and verified" % HERD in o for o in outs) and PRIV56 in outs[0], show(outs)


@needs_ingest
def test_resume_too_large_for_one_shard_is_refused_on_every_rank(tmp_path):
    """a capacity at which only the largest shard's buckets pass the load limit (shard 1 at this seed: 40764, 41012 and 40913
    entries): every rank exits non-zero, none waits in a collective, none starts stepping"""
    f = str(tmp_path / "e.work")
    rcs, outs = ranks(3, [IN56, "--dp", "8", "--grid", "8,32", "--seed", "13", "--max-steps", "4", "--save-work", f,
                          "--save-kangaroos"] + SH + cap(1 << 22))
    assert stepped(rcs) and "work file written" in outs[0], show(outs)
    per = shard_entries(f, 3)
    big = int(np.argmax(per))
    assert big != 0 and sorted(per)[-2] < per[big] - 1, per
    c = headroom(3) + per[big] - 1
    rcs, outs = ranks(3, ["--resume", f, "--grid", "8,32", "--seed", "2", "--max-steps", "5"] + SH + cap(c), timeout=300)
    assert all(rc != 0 for rc in rcs), show(outs)
    msg = "of shard %d hold more than its capacity %d less the stop headroom" % (big, c)
    assert all(msg in o for o in outs), show(outs)
    assert not any("MJump/s" in o or "imported and verified" in o for o in outs), show(outs)


# ---- f: --batch-keys on several ranks --------------------------------------------------------------------------------------
@needs_ingest
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("table", ["host", "sharded"])
def test_batch_keys_on_several_ranks(world, table):
    answers = [int(v, 16) for v in open(os.path.join(GOLD, "in56_64keys.answers.txt")).read().split()]
    extra = SH + cap(1 << 25) if table == "sharded" else []
    rcs, outs = ranks(world, [os.path.join(GOLD, "in56_64keys.txt"), "--batch-keys", "--dp", "8", "--grid", "16,128", "--seed", "3"]
                      + extra)
    assert rcs == [0] * world, show(outs)
    clean(outs)
    privs = {int(i): int(v, 16) for i, v in re.findall(r"Key#\s*(\d+) Pub:\s+0x[0-9A-F]+\s+Priv: 0x([0-9A-F]+)", outs[0])}
    assert privs == dict(enumerate(answers)), show(outs)
    if table == "sharded":
        hits = [int(v) for v in re.search(r"Hits resolved per shard: ([\d ]+)", outs[0]).group(1).split()]
        assert len(hits) == world and sum(hits) >= 64, hits
        if world == 3:
            assert sum(hits[1:]) > hits[0], hits                                # most on the shards of other ranks


# ---- g: more than 255 dead kangaroos in one step ---------------------------------------------------------------------------
@needs_ingest
@pytest.mark.parametrize("world,table", [(1, "host"), (2, "host"), (2, "sharded")])
def test_every_dead_kangaroo_is_re_created(world, table, tmp_path):
    """A herd made to re-walk its own trail: the table of a run to step k under the herd of the same run at step j < k.  Every
    DP the resumed herd makes before it passes step k is already in the table with its x and its distance, a dead kangaroo;
    one launch of 8 x 32 x 128 kangaroos per rank at dp 11 makes about a thousand per rank, far over the 255 one control
    broadcast carries.  Every one the table reports is re-created, on the gather path and the sharded one alike."""
    base = [IN80, "--dp", "11", "--grid", "8,32", "--seed", "12", "--save-kangaroos"]
    fj, fk, mix = (str(tmp_path / n) for n in ("j.work", "k.work", "mix.work"))
    for steps, f in (("2", fj), ("3", fk)):
        rcs, outs = ranks(world, base + ["--max-steps", steps, "--save-work", f])
        assert stepped(rcs) and dead(outs[0])[1] == 0, show(outs)
    n = world * HERD * 96
    raw_j, raw_k = open(fj, "rb").read(), open(fk, "rb").read()
    open(mix, "wb").write(raw_k[:len(raw_k) - n] + raw_j[len(raw_j) - n:])     # F_k's header and table, F_j's kangaroos
    extra = SH + cap(1 << 21) if table == "sharded" else []
    rcs, outs = ranks(world, ["--resume", mix, "--grid", "8,32", "--seed", "2", "--max-steps", "24"] + extra)
    assert stepped(rcs), show(outs)
    clean(outs)
    recreated, reported, most = dead(outs[0])
    assert most > 255 and reported > 400 * world, outs[0][-2500:]
    assert recreated == reported, outs[0][-2500:]
