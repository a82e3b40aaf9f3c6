"""-m gpu: the device DP table with its entries in pinned host memory (DeviceDPTable(entries="host"), KGX_DPT_HOST_ENTRIES)
against the table with everything on the device and the HashTable model fed the same records: events, counts, return codes
and work files byte for byte, add_resolve, a full table, saves and loads of 2^26 entries over several select passes, pieces
of shards, and the solver and the server with --dp-table-entries host."""
import ctypes
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import dptable_model as dm
from tests.test_gpu_server_shards import engine_recs, messages, outcome, same_file, serve, tame, worktool_check  # noqa: F401
from tests.test_gpu_server import write_cfg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
NB = 1 << 18
TYPE = np.uint64(1 << 62)


def upload(segments, stride):
    import torch
    flat = np.zeros((max(len(segments) * stride, 1), 5), dtype=np.uint64)
    for r, seg in enumerate(segments):
        flat[r * stride:r * stride + len(seg)] = seg
    return torch.from_numpy(flat.view(np.uint8).reshape(-1)).cuda()


def ev_tuples(evs, n, size=48):
    raw = ctypes.string_at(ctypes.addressof(evs), size * n)
    return [raw[i * size:(i + 1) * size] for i in range(n)]


def add_both(tables, segments, gap=3, resolver=None):
    """one call with the same rank segments (stride = the longest + gap) into every table -> [(rc, n, events as bytes)]"""
    stride = max([len(s) for s in segments] + [1]) + gap
    buf = upload(segments, stride)
    out = []
    for t in tables:
        try:
            rc, n, evs = t.add_raw(buf.data_ptr(), [len(s) for s in segments], stride, resolver=resolver)
        except Exception as e:                                      # TableFull: the same refusal on every layout
            out.append((type(e).__name__, len(t), None))
            continue
        out.append((rc, n, ev_tuples(evs, min(n, t._cap), 48 if resolver is None else 96), len(t)))
    return out


def batch(rng, n, seen, bad=0):
    """n random records, 5 % exact copies and 5 % same x with another d (either herd) of records seen before, `bad` with h >= 2^18"""
    a = rng.integers(0, 1 << 63, size=(n, 5), dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=(n, 5), dtype=np.uint64)
    a[:, 0] = (a[:, 0] & np.uint64(0xFFFFFFFF)) | (rng.integers(0, NB, size=n, dtype=np.uint64) << np.uint64(32))
    if len(seen):
        k = n // 20
        a[:k] = seen[rng.integers(0, len(seen), size=k)]
        b = seen[rng.integers(0, len(seen), size=k)].copy()
        b[:, 3] = rng.integers(0, 1 << 63, size=k, dtype=np.uint64)
        b[:, 4] = (b[:, 4] & TYPE) ^ (rng.integers(0, 2, size=k, dtype=np.uint64) << np.uint64(62)) | \
            (rng.integers(0, 1 << 62, size=k, dtype=np.uint64) & ~TYPE)
        a[k:2 * k] = b
    if bad:
        a[-bad:, 0] = (a[-bad:, 0] & np.uint64(0xFFFFFFFF)) | (rng.integers(NB, 1 << 32, size=bad, dtype=np.uint64) << np.uint64(32))
    return a[rng.permutation(n)]


def model_event(raw):
    """a kgx_dp_event's 48 bytes as HashTableModel.add's event tuple"""
    k, r, i, h = (int(v) for v in np.frombuffer(raw[:16], np.uint32))
    o0, o1, n0, n1 = (int(v) for v in np.frombuffer(raw[16:48], np.uint64))
    return (k, r, i, h, (o0, o1), (n0, n1))


def digest(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def pair(capacity, max_events=1 << 16, buckets=None):
    from kangaroo_b200.ingest import DeviceDPTable
    return [DeviceDPTable(capacity, max_events=max_events, buckets=buckets, entries=e) for e in ("device", "host")]


# ---- the calls ------------------------------------------------------------------------------------------------------------
def test_layout_and_memory():
    from kangaroo_b200.ingest import DeviceDPTable
    dev, host = pair(1 << 20)
    assert dev.host_bytes() == 0 and host.host_bytes() == 32 << 20
    assert dev.memory_bytes() - host.memory_bytes() == 32 << 20
    assert DeviceDPTable.bytes_for_ex(1 << 20, "host") == (DeviceDPTable.bytes_for(1 << 20) - (32 << 20), 32 << 20)
    for t in (dev, host):
        t.close()
    with pytest.raises(ValueError):
        DeviceDPTable(1000, entries="disk")


@pytest.mark.parametrize("ranks", [1, 3, 256])
def test_adds_equal_the_device_layout_and_the_model(ranks, tmp_path):
    rng = np.random.default_rng(ranks)
    tables = pair(1 << 20, max_events=1 << 14)
    model = dm.HashTableModel()
    seen = np.zeros((0, 5), np.uint64)
    for call in range(4):
        recs = batch(rng, 3000 if ranks < 256 else 20000, seen, bad=5 if call == 2 else 0)
        cut = np.sort(rng.choice(np.arange(1, len(recs)), size=ranks - 1, replace=False)) if ranks > 1 else []
        segments = np.split(recs, cut)
        if ranks > 2:
            segments[1] = segments[1][:0]                          # an empty rank
        want, skipped = model.add(segments)
        a, b = add_both(tables, segments, gap=int(rng.integers(0, 5)))
        assert a == b
        assert a[0] == (-1 if skipped else 0) and a[1] == len(want) <= 1 << 14 and a[3] == len(model)
        assert sorted(model_event(e) for e in a[2]) == sorted(want)
        seen = np.concatenate([seen, recs[(recs[:, 0] >> np.uint64(32)) < np.uint64(NB)]])
    paths = [str(tmp_path / ("%d.work" % i)) for i in range(2)]
    for t, p in zip(tables, paths):
        t.save_work(p, **dm.save_args())
        t.close()
    assert open(paths[0], "rb").read() == open(paths[1], "rb").read() == model.to_work().to_bytes()


def test_add_resolve_equals_the_device_layout():
    from kangaroo_b200 import ecmath as ec
    from kangaroo_b200.ingest import DeviceResolver, DPTable
    start = 1 << 60
    r = DeviceResolver(DPTable.key_table([ec.mul(12345)]), start)
    rng = np.random.default_rng(7)
    tables = pair(1 << 18, max_events=1 << 12)
    seen, events = np.zeros((0, 5), np.uint64), 0
    for _ in range(3):
        recs = batch(rng, 4000, seen)
        a, b = add_both(tables, [recs[:1500], recs[1500:]], resolver=r)
        assert a == b
        events += a[1]
        seen = np.concatenate([seen, recs])
    assert events >= 2 * 400                                       # the copies of earlier records
    for t in tables:
        t.close()
    r.close()


def test_a_full_table_refuses_the_call_and_changes_nothing(tmp_path):
    rng = np.random.default_rng(11)
    tables = pair(5000)
    recs = batch(rng, 4000, np.zeros((0, 5), np.uint64))
    assert add_both(tables, [recs])[0][0] == 0
    paths = [str(tmp_path / ("%d.work" % i)) for i in range(4)]
    for t, p in zip(tables, paths):
        t.save_work(p, **dm.save_args())
    a, b = add_both(tables, [batch(rng, 1001, recs)])
    assert a == b == ("TableFull", 4000, None)
    for t, p in zip(tables, paths[2:]):
        t.save_work(p, **dm.save_args())
        t.close()
    assert len({digest(p) for p in paths}) == 1


# ---- saves and loads at 2^26 entries: 8 select passes of 2^23 ----------------------------------------------------------
def fill_large(tables, n, seed=5, step=1 << 22):
    """n distinct random entries in batches of step records, generated on the GPU, into every table"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    for i in range(0, n, step):
        k = min(step, n - i)
        r = torch.randint(-(1 << 63), (1 << 63) - 1, (k, 5), dtype=torch.int64, device="cuda", generator=g)
        h = torch.randint(0, NB, (k,), dtype=torch.int64, device="cuda", generator=g)
        r[:, 0] = (h << 32) | torch.arange(i, i + k, device="cuda", dtype=torch.int64)
        for t in tables:
            rc, _, _ = t.add_raw(r.data_ptr(), [k], k)
            assert rc == 0
        del r
    torch.cuda.synchronize()


def test_save_and_load_2_26_entries_across_layouts(tmp_path):
    n = 1 << 26
    dev, host = pair(n)
    fill_large([dev, host], n - 12345)
    assert len(dev) == len(host) and len(dev) > n - 12345 - 100
    a, b = str(tmp_path / "dev.work"), str(tmp_path / "host.work")
    dev.save_work(a, **dm.save_args())
    host.save_work(b, **dm.save_args())
    assert os.path.getsize(a) == os.path.getsize(b) and digest(a) == digest(b)
    want = digest(a)
    os.remove(b)
    count = len(dev)
    dev.load_work_ex(a)                                            # device -> device, as before
    host.load_work_ex(a)                                           # the device layout's file into the host layout
    assert len(host) == len(dev) == count
    host.save_work(b, **dm.save_args())
    assert digest(b) == want
    dev.load_work_ex(b)                                            # and back
    os.remove(a)
    dev.save_work(a, **dm.save_args())
    assert digest(a) == want
    for t in (dev, host):
        t.close()


# ---- pieces ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 3, 8])
def test_pieces_of_host_entry_shards_equal_the_single_table(world, tmp_path):
    from kangaroo_b200 import solver as S
    from kangaroo_b200.dist import owner_ranges
    from kangaroo_b200.ingest import DeviceDPTable
    rng = np.random.default_rng(world)
    single = DeviceDPTable(1 << 20)
    shards = [DeviceDPTable(1 << 18, buckets=rg, entries="host") for rg in owner_ranges(world)]
    seen = np.zeros((0, 5), np.uint64)
    for _ in range(3):
        recs = batch(rng, 20000, seen)
        add_both([single], [recs])
        for s in shards:
            buf = upload([recs], len(recs))
            s.add_raw(buf.data_ptr(), [len(recs)], len(recs))
        seen = np.concatenate([seen, recs])
    assert sum(len(s) for s in shards) == len(single)
    one = str(tmp_path / "one.work")
    single.save_work(one, **dm.save_args())

    def assemble(path):
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

    want = open(one, "rb").read()
    assert assemble(str(tmp_path / "pieces.work")) == want
    counts = [len(s) for s in shards]
    for s in shards:
        s.load_piece(one, s.capacity)
    assert [len(s) for s in shards] == counts
    assert assemble(str(tmp_path / "again.work")) == want
    for t in shards + [single]:
        t.close()


# ---- the solver ----------------------------------------------------------------------------------------------------------
def solver(args, timeout=900):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver"] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    return p.returncode, p.stdout + p.stderr


RUN = [os.path.join(GOLD, "in56.txt"), "--dp", "8", "--grid", "8,32", "--seed", "5", "--max-steps", "4", "--save-kangaroos"]
CAP = ["--dp-table-capacity", str(1 << 22)]
PRIV56 = "Priv: 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD612C0F05F3DA03"


def test_solver_host_entries_save_equal_and_resume_across_layouts(tmp_path):
    a, b = str(tmp_path / "dev.work"), str(tmp_path / "host.work")
    rc, out = solver(RUN + ["--save-work", a, "--dp-table", "device"] + CAP)
    assert "work file written" in out, out[-2000:]
    rc, out2 = solver(RUN + ["--save-work", b, "--dp-table", "device", "--dp-table-entries", "host"] + CAP)
    assert "work file written" in out2 and "entries in pinned host memory" in out2, out2[-2000:]
    assert open(a, "rb").read()[156:] == open(b, "rb").read()[156:]
    rc, out = solver(["--resume", b, "--grid", "16,32", "--seed", "2", "--dp-table", "device"] + CAP)
    assert rc == 0 and "imported and verified" in out and PRIV56 in out, out[-2000:]
    rc, out = solver(["--resume", a, "--grid", "16,32", "--seed", "2", "--dp-table", "device", "--dp-table-entries", "host"] + CAP)
    assert rc == 0 and "imported and verified" in out and PRIV56 in out, out[-2000:]


def test_sharded_two_ranks_host_entries_equal_device_layout(tmp_path):
    from tests.ranks_util import run_ranks
    files = []
    for e in ("device", "host"):
        f = str(tmp_path / ("%s.work" % e))
        rcs, outs = run_ranks(2, RUN + ["--save-work", f, "--dp-table", "sharded", "--dp-table-entries", e] + CAP)
        assert "work file written" in outs[0], "".join(outs)[-3000:]
        files.append(open(f, "rb").read())
    assert files[0][156:] == files[1][156:]
    rcs, outs = run_ranks(2, ["--resume", str(tmp_path / "device.work"), "--grid", "16,32", "--seed", "2", "--dp-table", "sharded",
                              "--dp-table-entries", "host"] + CAP)
    assert "imported and verified" in outs[0] and PRIV56 in outs[0], "".join(outs)[-3000:]


# ---- the server ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("devices", [None, "0,0"])
def test_server_host_entries_equal_device_entries(tmp_path, tame, devices):  # noqa: F811
    cfg = write_cfg(tmp_path / "c.txt")
    msgs, _ = messages(tame)
    extra = ["--devices", devices] if devices else []
    base = [cfg, "--dp", 8, "--dp-table-capacity", 1 << 20] + extra
    rcd, d = serve(tmp_path, "dev", base + ["--save-work", tmp_path / "dev.work"], msgs)
    rch, h = serve(tmp_path, "host", base + ["--save-work", tmp_path / "host.work", "--dp-table-entries", "host"], msgs)
    assert rcd == rch == 1 and "entries in pinned host memory" in h
    assert outcome(d) == outcome(h)
    same_file(tmp_path / "dev.work", tmp_path / "host.work")
    worktool_check(tmp_path / "host.work")
    rc, r = serve(tmp_path, "resumed", ["--resume", tmp_path / "dev.work", "--save-work", tmp_path / "r.work",
                                        "--dp-table-capacity", 1 << 20, "--dp-table-entries", "host"] + extra, [])
    assert rc == 1 and "Resume %s" % (tmp_path / "dev.work") in r
    same_file(tmp_path / "dev.work", tmp_path / "r.work")
