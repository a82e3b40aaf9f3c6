"""CPU: the model of the reference's HashTable in tests/dptable_model.py against the reference itself -- the host table
(kgi_add) and the reference binary's -wm / -wmdir -- on records and work files built at the keys random records never produce,
and a guard that the model's mirror of the device table's index hash is still the hash in kgx_dptable.cuh."""
import os
import re
import shutil
import subprocess
from collections import Counter

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200 import worktool as wt
from tests import dptable_model as dm
from tests.worktool_util import NB, REFBIN, ROOT, Work, merge_model

INGEST = os.path.join(ROOT, "build", "libkgx_ingest.so")
needs_ingest = pytest.mark.skipif(not os.path.exists(INGEST), reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")
needs_ref = pytest.mark.skipif(not os.path.exists(REFBIN), reason="oracle/_ref/kangaroo_ref_cpu not built (needs the reference sources)")
CUH = os.path.join(ROOT, "kangaroo_b200", "csrc", "kgx_dptable.cuh")


def squeeze(s):
    return re.sub(r"\s+", "", s)


def test_the_mirror_is_the_tables_hash():
    """The crafted index tests build their records with dptable_model's slot_home / slot_tag / slots_for.  If the table's hash
    changed without the mirror, those tests would quietly become random ones: update both together."""
    src = open(CUH).read()
    tag = re.search(r"uint32_t slot_tag\(uint32_t h, uint64_t x1\) \{(.*?)\}", src, re.S).group(1)
    assert squeeze(tag) == "return(h+1)|((uint32_t)(x1>>51)<<19);"
    home = re.search(r"uint64_t slot_home\(uint32_t h, uint64_t x0, uint64_t x1, uint64_t nslots\) \{(.*?)\n\}", src, re.S).group(1)
    assert squeeze(home) == squeeze("uint64_t k = (x0 ^ (x1 * 0x%Xull) ^ ((uint64_t)h << 40)) * 0x%Xull; k ^= k >> 32; "
                                    "return __umul64hi(k, nslots);" % (dm.HOME_MUL_X1, dm.HOME_MUL))
    slots = re.search(r"uint64_t slots_for\(uint64_t capacity\) \{(.*?)\}", src).group(1)
    assert squeeze(slots) == "returncapacity+capacity/2+64;"
    assert re.search(r"SAVE_CHUNK = 1ull << (\d+);", src).group(1) == str(dm.SAVE_CHUNK.bit_length() - 1)
    # the array form is the scalar one
    rng = np.random.default_rng(1)
    h = rng.integers(0, NB, size=2000, dtype=np.uint64)
    x0, x1 = (rng.integers(0, 1 << 63, size=2000, dtype=np.uint64) * np.uint64(2) + np.uint64(1) for _ in range(2))
    for n in (dm.slots_for(1), dm.slots_for(4096), dm.slots_for(1 << 31)):
        got = dm.slot_homes(h, x0, x1, n)
        assert got.tolist() == [dm.slot_home(int(a), int(b), int(c), n) for a, b, c in zip(h, x0, x1)]
        assert int(got.max()) < n


def test_the_records_are_at_the_edges_they_claim():
    adv = dm.Adversary(5)
    again = dm.Adversary(5)
    assert all(np.array_equal(a[1], b[1]) for a, b in zip(adv.classes(), again.classes()))     # seeded
    adv = dm.Adversary(5)
    n = adv.nslots
    a = adv.shared_hi()
    for h in set((a[:, 0] >> np.uint64(32)).tolist()):
        b = a[(a[:, 0] >> np.uint64(32)) == np.uint64(h)]
        assert 30 <= len(b) <= 60 and len(set(b[:, 2].tolist())) == 1 and len(set(b[:, 1].tolist())) == len(b)
        lo = set(b[:, 1].tolist())
        assert set(dm.SPECIAL) <= lo and any(v ^ (1 << k) in lo for v in lo for k in range(64))
    b = adv.shared_lo()
    assert {0, (1 << 63) - 1, 1 << 63, dm.M64} <= set(b[:, 2].tolist())
    c = adv.one_x()
    assert max(Counter(zip(c[:, 1].tolist(), c[:, 2].tolist())).values()) >= 5
    d = adv.same_home()
    hs, x0, x1 = (d[:, 0] >> np.uint64(32)).tolist(), d[:, 1].tolist(), d[:, 2].tolist()
    assert len(set(hs)) == 1 and len({dm.slot_tag(h, v) for h, v in zip(hs, x1)}) == 1
    assert len({dm.slot_home(h, a, b, n) for h, a, b in zip(hs, x0, x1)}) == 1 and len(set(zip(x0, x1))) == len(d)
    assert Counter(x1).most_common(1)[0][1] == len(d) // 2 and Counter(x0).most_common(1)[0][1] == len(d) // 2
    e = adv.wrapping()
    homes = [dm.slot_home(int(r[0]) >> 32, int(r[1]), int(r[2]), n) for r in e]
    assert min(homes) >= n - 4 and len(homes) > 4                       # more records than slots to the end: the chain wraps
    f = adv.contention()
    assert len({int(r[0]) >> 32 for r in f}) == len(f) == 300
    assert len({dm.slot_home(int(r[0]) >> 32, int(r[1]), int(r[2]), n) for r in f}) == 1
    g = adv.copies(a)
    assert sorted(map(tuple, g[:, 1:3].tolist())) == sorted(map(tuple, a[:, 1:3].tolist()))
    assert len({int(r[0]) & 0xFFFFFFFF for r in np.concatenate([a, g])}) == len(a) + len(g)   # every record its own kIdx


def test_the_model_counts_items_like_the_reference():
    """maxItem: 16 on a bucket's first Add, then +4 on every Add that finds nbItem >= maxItem - 1, stored or not"""
    adv = dm.Adversary(2)
    m = dm.HashTableModel()
    r = adv.random(40, buckets=[77])
    ev, bad = m.add([r[:15]])
    assert ev == [] and bad == 0 and m.mx[77] == 16 and len(m) == 15
    ev, _ = m.add([r[:1]])                                             # finds nbItem 15 >= 15: +4, not stored
    assert m.mx[77] == 20 and len(ev) == 1 and ev[0][0] == dm.EV_RESET and ev[0][4] == (0, 0)
    m.add([r[15:19]])                                                  # 15 -> 19 (+0: 15 < 19, 16 < 19, 17 < 19, 18 < 19)
    assert m.mx[77] == 20
    m.add([r[19:20]])                                                  # 19 >= 19: +4
    assert m.mx[77] == 24
    bad = r[20:22].copy()
    bad[0, 0] = np.uint64(NB << 32)
    ev, skipped = m.add([bad])
    assert skipped == 1 and len(m) == 21
    w = m.to_work()
    assert [x for x, _ in w.table[77]] == sorted(int(a) | int(b) << 64 for a, b in np.concatenate([r[:20], r[21:22]])[:, 1:3])


@needs_ingest
def test_the_model_is_the_host_table_on_adversarial_records(tmp_path):
    """every class with copies over several calls and rank segments, then all of them again: the reference's HashTable gives the
    model's events (as a multiset: the host returns them in worker-shard order), count and saved bytes"""
    from kangaroo_b200.ingest import DPTable
    adv = dm.Adversary(17)
    host = DPTable(threads=8, max_events=1 << 16)
    m = dm.HashTableModel()
    everything = np.concatenate([r for _, r in adv.classes()])
    bad = adv.random(3)
    bad[1, 0] = np.uint64((NB + 9) << 32)
    calls = [segs for _, r in adv.classes() for segs in adv.calls(r)] + adv.calls(everything, ncalls=4, nsegs=5) + [[bad]]
    kinds = Counter()
    for segs in calls:
        want, skipped = m.add(segs)
        got, host_bad = dm.host_add(host, segs)
        assert sorted(got) == sorted(want) and host_bad == (skipped > 0)
        assert len(host) == len(m)
        kinds.update(e[0] for e in want)
    assert kinds[dm.EV_RESET] > 300 and kinds[dm.EV_COLLISION] > 100
    path = str(tmp_path / "host.work")
    host.save_work(path, **dm.save_args())
    assert open(path, "rb").read() == m.to_work().to_bytes()
    host.close()


@needs_ref
def test_merge_model_is_the_reference_merge_on_adversarial_files(tmp_path):
    """-wm of two files and -wmdir of four, holding classes (a), (b) and (c) with runs of equal x over the inputs: the model's
    bytes (plus the kangaroo count the reference's merge leaves out)"""
    from tests.golden import make_work_golden as g
    works = dm.Adversary(23).merge_inputs(4, g.START, g.START + (1 << g.RANGE_BITS) - 1, ec.mul(g.PRIV))
    paths = [w.write(str(tmp_path / ("in%d.work" % i))) for i, w in enumerate(works)]
    _, dup, coll = merge_model(works)
    assert dup > 20 and len(coll) > 40
    out = str(tmp_path / "ref_wm.work")
    r = subprocess.run([REFBIN, "-wm", paths[2], paths[0], out], capture_output=True, text=True, timeout=300)
    assert "Priv:" not in r.stdout, r.stdout[-2000:]
    assert merge_model([works[2], works[0]])[0].to_bytes() == open(out, "rb").read() + b"\0" * 8
    d = tmp_path / "d"
    os.mkdir(d)
    for p in paths:
        shutil.copy(p, d / os.path.basename(p))
    order = wt.dir_inputs(str(d))
    assert len({os.path.getsize(p) for p in order}) == 4
    out = str(tmp_path / "ref_dir.work")
    r = subprocess.run([REFBIN, "-wmdir", str(d), out], capture_output=True, text=True, timeout=300)
    assert "Priv:" not in r.stdout, r.stdout[-2000:]
    assert merge_model([Work.read(p) for p in order])[0].to_bytes() == open(out, "rb").read() + b"\0" * 8
