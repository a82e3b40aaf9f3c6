"""CPU: the work-file merge's refusals and a model of its semantics (python -m kangaroo_b200.worktool), checked against the
reference's own -wm / -wmdir output."""
import os
import shutil
import subprocess

import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200 import worktool as wt
from tests.worktool_util import REFBIN, Work, crafted_pair, golden, merge_model, tagged

needs_ref = pytest.mark.skipif(not os.path.exists(REFBIN), reason="oracle/_ref/kangaroo_ref_cpu not built (needs the reference sources)")


def small(tmp_path, name, **kw):
    from tests.golden import make_work_golden as g
    a = dict(dp=16, start=g.START, end=g.START + (1 << g.RANGE_BITS) - 1, key=ec.mul(g.PRIV))
    a.update(kw)
    w = Work(a["dp"], a["start"], a["end"], a["key"], 10, 1.0, a.get("version", 0))
    for i in range(1, 4):
        w.add(ec.mul(31 * i)[0], tagged(31 * i, False))
    return w.write(str(tmp_path / name))


@pytest.mark.parametrize("what,match", [
    ("one", "at least two"), ("range", "range differs"), ("key", "key differs"), ("version", "different version"),
    ("curve", "does not lie on elliptic curve"), ("curve+range", "does not lie on elliptic curve"), ("nothw", "not a HEADW"),
    ("dir", "directory")])
def test_merge_refusals_write_nothing(tmp_path, what, match):
    from tests.golden import make_work_golden as g
    a = small(tmp_path, "a.work")
    if what == "one":
        inputs = [a]
    elif what == "range":
        inputs = [a, small(tmp_path, "b.work", end=g.START + (1 << 40))]
    elif what == "key":
        inputs = [a, small(tmp_path, "b.work", key=ec.mul(g.PRIV + 1))]
    elif what == "version":
        inputs = [a, small(tmp_path, "b.work", version=1)]
    elif what == "curve":
        x, y = ec.mul(g.PRIV)
        inputs = [a, small(tmp_path, "b.work", key=(x, y + 1))]
    elif what == "curve+range":                             # two faults in one input: the curve is refused first
        x, y = ec.mul(g.PRIV)
        inputs = [a, small(tmp_path, "b.work", key=(x, y + 1), end=g.START + (1 << 40))]
    elif what == "nothw":
        (tmp_path / "b.work").write_bytes(b"\x00" * 400)
        inputs = [a, str(tmp_path / "b.work")]
    else:
        os.mkdir(tmp_path / "d")
        inputs = [a, str(tmp_path / "d")]
    dest = str(tmp_path / "dest.work")
    with pytest.raises(ValueError, match=match):
        wt.merge(inputs, dest)
    assert not os.path.exists(dest) and not os.path.exists(dest + ".tmp")
    assert wt.main(["merge"] + inputs + ["-o", dest]) == 2


def test_check_refuses_a_directory(tmp_path):
    with pytest.raises(ValueError, match="directory"):
        wt.check(str(tmp_path))


def test_model_first_input_wins_duplicates_collisions_and_rounding(tmp_path):
    a = Work(14, 0, (1 << 64) - 1, ec.mul(5), 100, 1.25)
    b = Work(12, 0, (1 << 64) - 1, ec.mul(5), 200, 2.5)
    c = Work(16, 0, (1 << 64) - 1, ec.mul(5), 300, 4.0)
    X = lambda i, h: (h << 128) | (i << 64) | 7            # x in bucket h, ordered by i
    a.add(X(1, 5), tagged(10, False)); a.add(X(3, 5), tagged(11, True))
    b.add(X(1, 5), tagged(10, False))                       # duplicate of a's
    b.add(X(2, 5), tagged(12, False)); b.add(X(3, 5), tagged(99, False))   # new, and a tame/wild collision with a's
    c.add(X(2, 5), tagged(13, False))                       # same-herd collision with b's (the first at that x)
    c.add(X(9, 7), tagged(14, True))
    m, dup, coll = merge_model([a, b, c])
    assert (m.dp, m.count, m.time) == (12, 600, 7.75)
    assert m.table[5] == [(X(1, 5) & ((1 << 128) - 1), tagged(10, False)), (X(2, 5) & ((1 << 128) - 1), tagged(12, False)),
                          (X(3, 5) & ((1 << 128) - 1), tagged(11, True))]
    assert m.maxitem[5] == 4 and m.maxitem[7] == 4 and m.maxitem[0] == 0
    assert dup == 1
    assert coll == [(5, tagged(12, False), tagged(13, False)), (5, tagged(11, True), tagged(99, False))]
    # b first: b's entries win
    m2, _, _ = merge_model([b, a])
    assert dict(m2.table[5])[X(3, 5) & ((1 << 128) - 1)] == tagged(99, False)


def test_dir_order_is_largest_first(tmp_path):
    d = tmp_path / "d"
    os.mkdir(d)
    for name, n in (("a.work", 1), ("b.work", 5), ("c.work", 3), ("z.work", 5)):
        w = Work(10, 0, 1 << 40, ec.mul(3))
        for i in range(n):
            w.add(ec.mul(100 + i)[0], tagged(100 + i, False))
        w.write(str(d / name))
    (d / "notes.txt").write_text("not a work file")
    os.mkdir(d / "sub")
    assert [os.path.basename(p) for p in wt.dir_inputs(str(d))] == ["b.work", "z.work", "c.work", "a.work"]


def test_model_equals_the_reference_merge_fixture(tmp_path):
    """ref_merge48 is the reference's -wm output for (ref_work48, ref_work48b): the model gives its bytes plus a zero kangaroo
    count"""
    a, b = golden("ref_work48.work.gz", tmp_path), golden("ref_work48b.work.gz", tmp_path)
    ref = open(golden("ref_merge48.work.gz", tmp_path), "rb").read()
    m, dup, coll = merge_model([Work.read(a), Work.read(b)])
    assert m.to_bytes() == ref + b"\0" * 8
    assert all(not ((c[1] ^ c[2]) >> 126) & 1 for c in coll)  # no tame/wild collision: the pair does not find the key


@needs_ref
def test_model_equals_reference_wm_and_wmdir(tmp_path):
    a, b = golden("ref_work48.work.gz", tmp_path), golden("ref_work48b.work.gz", tmp_path)
    c = small(tmp_path, "c.work")
    pa, pb = crafted_pair(tmp_path)
    out = str(tmp_path / "ref_ab.work")
    subprocess.run([REFBIN, "-wm", a, c, out], capture_output=True, text=True, timeout=300, check=True)
    m, _, _ = merge_model([Work.read(a), Work.read(c)])
    assert m.to_bytes() == open(out, "rb").read() + b"\0" * 8
    # -wmdir over four files of different sizes: largest first, pairwise
    d = tmp_path / "d"
    os.mkdir(d)
    for p in (a, b, c, pb):
        shutil.copy(p, d / os.path.basename(p))
    order = wt.dir_inputs(str(d))
    assert len({os.path.getsize(p) for p in order}) == 4
    out = str(tmp_path / "ref_dir.work")
    r = subprocess.run([REFBIN, "-wmdir", str(d), out], capture_output=True, text=True, timeout=300)
    assert "Priv:" not in r.stdout, r.stdout[-2000:]
    m, _, _ = merge_model([Work.read(p) for p in order])
    assert m.to_bytes() == open(out, "rb").read() + b"\0" * 8
