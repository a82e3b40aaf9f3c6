"""CPU: work files with kangaroos (Kangaroo::SaveWork -ws / LoadWork / FetchWalks, Backup.cpp:149-231, 449-572) through the
ingest library: a file the reference's own CPU program wrote, a write/read round trip, and write errors."""
import gzip
import os
import shutil

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_work48.work.gz")
pytestmark = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")


def _limbs_to_int(row):
    return sum(int(v) << (64 * k) for k, v in enumerate(row))


def golden_work(tmp_path):
    path = str(tmp_path / "ref_work48.work")
    with gzip.open(GOLDEN, "rb") as src, open(path, "wb") as dst:
        shutil.copyfileobj(src, dst)
    return path


def test_reference_written_work_file_loads_with_its_kangaroos(tmp_path):
    from tests.golden import make_work_golden as g
    from kangaroo_b200.ingest import DPTable, read_work_header
    path = golden_work(tmp_path)
    t = DPTable(threads=2)
    w = t.load_work_ex(path)
    pub = ec.mul(g.PRIV)
    assert (w.dp_bits, w.range_start, w.range_end, w.key) == (g.DP_BITS, g.START, g.START + (1 << g.RANGE_BITS) - 1, pub)
    assert w.total_count > 0 and w.total_time > 0 and len(t) > 0
    assert w.nb_walk == 1024                                              # one CPU thread: CPU_GRP_SIZE kangaroos
    assert os.path.getsize(path) == w.walk_offset + 96 * w.nb_walk
    assert read_work_header(path) == (w.dp_bits, w.range_start, w.range_end, w.key, w.total_count, w.total_time)
    assert read_work_header(path).version == 0                            # Kangaroo::SaveHeader writes version 0
    key = ec.add(pub, ec.neg(ec.mul(g.START)))                            # Kangaroo::InitSearchKey: P - start*G
    recs = w.walks()
    for i in list(range(8)) + list(range(1016, 1024)) + [101, 502, 777]:
        x, y, d = (_limbs_to_int(recs[i, 4 * k:4 * k + 4]) for k in range(3))
        assert d < ec.N
        want = ec.add(key, ec.mul(d)) if i & 1 else ec.mul(d)            # wild kangaroos: key + d*G (odd positions)
        assert (x, y) == want, i
    assert np.array_equal(w.walks(100, 5), recs[100:105])
    t.close()


def _table(seed, n):
    from kangaroo_b200.ingest import DPTable
    rng = np.random.default_rng(seed)
    raw = np.zeros((n, 10), dtype=np.uint32)
    raw[:, 0] = np.arange(n)
    raw[:, 2:10] = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint32)
    raw[:, 1] = raw[:, 6] & 0x3FFFF
    raw[:, 9] &= 0x7FFFFFFF
    t = DPTable(threads=2)
    assert t.add_dp40(raw) == []
    return t


def test_table_and_kangaroos_round_trip_byte_for_byte(tmp_path):
    from kangaroo_b200.ingest import DPTable
    t = _table(5, 20000)
    n = 777
    recs = np.random.default_rng(6).integers(0, 1 << 63, size=(n, 12), dtype=np.uint64)
    start, end = 0x1234 << 100, (0x1234 << 100) + (1 << 80) - 1
    pub = ec.mul(0xC0FFEE)
    a = str(tmp_path / "a.work")
    t.save_work(a, 14, start, end, pub, total_count=123456789, total_time=42.5, total_walk=n)
    with open(a, "ab") as f:
        f.write(recs.tobytes())
    t2 = DPTable(threads=3)
    w = t2.load_work_ex(a)
    assert (w.dp_bits, w.range_start, w.range_end, w.key, w.total_count, w.total_time, w.nb_walk) == (14, start, end, pub, 123456789, 42.5, n)
    assert len(t2) == len(t) == 20000
    assert np.array_equal(w.walks(), recs)
    # the reloaded table writes the same bytes
    b = str(tmp_path / "b.work")
    t2.save_work(b, 14, start, end, pub, total_count=123456789, total_time=42.5, total_walk=n)
    with open(b, "ab") as f:
        f.write(w.walks().tobytes())
    assert open(a, "rb").read() == open(b, "rb").read()
    # a file cut inside its kangaroo block is refused
    c = str(tmp_path / "c.work")
    with open(c, "wb") as f:
        f.write(open(a, "rb").read()[:-50])
    with pytest.raises(RuntimeError):
        DPTable(threads=1).load_work_ex(c)
    # kgi_save_work keeps its meaning: zero kangaroos
    z = str(tmp_path / "z.work")
    t.save_work(z, 14, start, end, pub)
    assert DPTable(threads=1).load_work_ex(z).nb_walk == 0
    t.close(); t2.close()


def test_write_errors_are_reported(tmp_path):
    t = _table(7, 5000)
    pub = ec.mul(3)
    with pytest.raises(RuntimeError, match="No space left"):
        t.save_work("/dev/full", 10, 0, (1 << 64) - 1, pub, total_walk=10)    # ENOSPC
    plain = tmp_path / "plain"
    plain.write_bytes(b"x")
    with pytest.raises(RuntimeError, match="Not a directory"):
        t.save_work(str(plain / "w.work"), 10, 0, (1 << 64) - 1, pub)           # ENOTDIR
    t.close()
