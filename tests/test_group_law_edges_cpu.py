"""CPU: the crafted inputs of tests/test_gpu_group_law_edges.py have the property each class claims (so that a later change
cannot quietly turn them into random ones), and the check model in tests/group_law_model.py agrees with the reference
program's -wcheck on a plain one-key file (needs the reference sources at build time)."""
import os
import re
import subprocess

import pytest

from kangaroo_b200 import ecmath as ec
from tests import group_law_model as gm
from tests.worktool_util import REFBIN

N = gm.N
needs_ref = pytest.mark.skipif(not os.path.exists(REFBIN), reason="oracle/_ref/kangaroo_ref_cpu not built (needs the reference sources)")
SIZES = [1, 7, 8, 9, 17]
OK_CLASSES = {"match", "tame", "max", "zero", "dbl", "shared", "inf_key"}
WRONG_CLASSES = {"zero_tame", "opp", "bad_x", "bad_h"}


@pytest.mark.parametrize("n_keys", SIZES)
def test_the_keys_are_the_points_they_claim(n_keys):
    kk = gm.key_scalars(n_keys)
    assert kk == gm.key_scalars(n_keys)                                   # seeded
    keys = [gm.key_point(k) for k in kk]
    start_g = ec.mul(gm.START)
    for k, K in zip(kk, keys):
        assert ec.add(gm.pub_of(k), ec.neg(start_g)) == K                  # K = pub - start*G
    if n_keys > gm.INF_KEY:
        assert keys[gm.INF_KEY] is None and gm.pub_of(kk[gm.INF_KEY]) == start_g
    assert sum(K is None for K in keys) == (1 if n_keys > gm.INF_KEY else 0)
    same, opp = gm.key_pairs(n_keys)
    for a, b in same:
        assert keys[a] == keys[b] and keys[a] is not None
    for a, b in opp:
        assert keys[a] == ec.neg(keys[b]) and keys[a] != keys[b]
    assert len(same) == len(opp) == (1 if n_keys >= 7 else 0)
    if n_keys >= 7:
        assert any(a // gm.KB == b // gm.KB for a, b in opp) == (n_keys <= 12)   # the opposite pair in one batch of 8, or two
    assert any(k > N // 2 for k in kk if k) == (n_keys > 1)                 # S = +K needs the sign bit for some keys


@pytest.mark.parametrize("n_keys", SIZES)
def test_the_entries_have_the_property_of_their_class(n_keys):
    kk = gm.key_scalars(n_keys)
    keys = [gm.key_point(k) for k in kk]
    ents = gm.batch_entries(kk)
    assert ents == gm.batch_entries(kk)                                   # seeded
    seen = {}
    for e in ents:
        s = gm.s_point(e.d)
        wild, neg = bool(e.d & gm.WILD_BIT), bool(e.d & gm.NEG_BIT)
        seen.setdefault(e.cls, set()).add((wild, neg))
        ok = gm.entry_ok(e.h, e.x, e.d, keys)
        assert ok == (e.cls in OK_CLASSES) and (e.cls in OK_CLASSES) != (e.cls in WRONG_CLASSES), e
        if e.cls in ("match", "max", "zero", "dbl", "shared", "inf_key"):
            assert wild and gm.hx(ec.add(s, keys[e.key])) == (e.h, e.x), e      # the point the entry is built on
        if e.cls == "match":
            assert e.key in gm.match_indices(n_keys)
        elif e.cls == "max":
            assert e.d & gm.MAG == gm.MAG
        elif e.cls in ("zero", "zero_tame"):
            assert e.d & gm.MAG == 0 and s is None
        elif e.cls == "dbl":
            assert s == keys[e.key] is not None                             # S = +K: a doubling
        elif e.cls == "opp":
            assert wild and s == ec.neg(keys[e.key]) and keys[e.key] is not None   # S = -K: infinity
        elif e.cls == "shared":
            assert s[0] == keys[e.other][0] and e.other != e.key and e.key // gm.KB == e.other // gm.KB
            assert not gm.entry_ok(e.h, e.x, e.d, [keys[e.other]]) and keys[e.key] not in (s, ec.neg(s))
        elif e.cls == "inf_key":
            assert keys[e.key] is None and gm.hx(s) == (e.h, e.x)
        elif e.cls == "bad_x":                                              # a right entry with one x bit flipped
            assert any(f.d == e.d and f.h == e.h and bin(f.x ^ e.x).count("1") == 1 for f in ents if f.cls in OK_CLASSES), e
        elif e.cls == "bad_h":                                              # a right entry one bucket off
            assert any(f.d == e.d and f.x == e.x and (f.h - e.h) % (1 << 18) in (1, (1 << 18) - 1) for f in ents if f.cls in OK_CLASSES), e
    # every class, with the sign bit both ways where the class has a free sign
    want = {"match", "tame", "max", "zero", "zero_tame", "dbl", "opp", "bad_x", "bad_h"}
    if n_keys > gm.INF_KEY:
        want |= {"inf_key"}
    if n_keys >= 7:
        want |= {"shared"}
    assert set(seen) == want
    for c in ("match", "tame", "max", "zero", "zero_tame", "inf_key"):
        if c in seen:
            assert len({neg for _, neg in seen[c]}) == 2, c
    assert {neg for _, neg in seen["dbl"]} == ({False, True} if n_keys > 1 else {gm.signed_mag(kk[0])[1]})
    assert {e.key for e in ents if e.cls == "match"} == set(gm.match_indices(n_keys))
    assert {e.key for e in ents if e.cls == "dbl"} == {j for j in range(n_keys) if kk[j]}
    if n_keys == 17:
        assert {0, 7, 8, 9, 15, 16} <= {e.key for e in ents if e.cls == "match"}
        assert {e.other % gm.KB for e in ents if e.cls == "shared"} >= {0, 7}       # the zero factor first and last in its batch


@pytest.mark.parametrize("n_keys", [9, 17])
def test_the_kangaroos_have_the_property_of_their_class(n_keys):
    kk = gm.key_scalars(n_keys)
    keys = [gm.key_point(k) for k in kk]
    kinds = {"tame": 1, "wild": 2, "last": 2, "zero": 2, "same_key_target": 2, "inf_target": 1, "n_minus_1": 1,
             "inf_target_zero": 0, "neg_key_target": 0, "wrong_target": 0, "d_ge_n": 0, "mag_2_128": 0, "bad_y": 0}
    walks = gm.batch_walks(kk)
    assert {v.cls for v in walks} == set(kinds)
    for v in walks:
        assert gm.walk_kind(v.x, v.y, v.d, keys[v.target]) == kinds[v.cls], v
        assert 0 <= v.target < n_keys
    assert {v.target for v in walks if v.cls == "last"} == {n_keys - 1}
    assert all(keys[v.target] is None for v in walks if v.cls.startswith("inf_target"))
    assert all(v.d == 0 for v in walks if v.cls == "zero")
    assert any(v.d > N // 2 for v in walks if v.cls == "tame")             # negative distances too


def test_the_retarget_scalars_give_the_degenerate_points():
    n = 3 * 32 * 128
    case = gm.retarget_case(n)
    ks, to = case["ks"], case["to"]
    K = [ec.mul(k) for k in ks]
    assert K[1] == ec.neg(K[0]) and 1 in to                                 # keys[to] = -keys[from]: the delta is -2 K_0
    assert ec.add(K[1], ec.neg(K[0])) == ec.add(K[1], K[1])
    kinds = set()
    for s, (kind, d, b) in case["special"].items():
        assert s % 2 == 1 and to[(s >> 1) % len(to)] == b                   # a wild kangaroo that the spread rule sends to b
        p = ec.add(K[0], ec.mul(d))                                         # its point
        delta = ec.add(K[b], ec.neg(K[0]))
        assert p == (delta if kind == "p_eq_delta" else ec.neg(delta)), (s, kind)
        assert ec.add(p, delta) == (ec.add(K[b], ec.mul(d)) if kind == "p_eq_delta" else None)
        kinds.add((kind, s >= n - 128))
    assert kinds == {("p_eq_delta", False), ("p_neg_delta", False), ("p_eq_delta", True), ("p_neg_delta", True)}
    assert len(set(to)) < len(to) and 0 not in to


@pytest.mark.parametrize("wo", gm.WILD_OFFSETS)
def test_the_checkpoint_values_sit_at_the_edges(wo):
    for wild in (False, True):
        b = {d: gm.biased(d, wo, wild) for d in gm.import_distances(wo, wild)}
        assert {d for d in b if d >= N} >= {N, N + 1, N + gm.M128, (1 << 256) - 1}   # reduced once by n
        fits = {v for v in b.values() if v <= gm.M128}
        assert 0 in fits and gm.M128 in fits and (1 << 128) in b.values()   # both sides of the 128-bit limit
        if wild:
            assert b[N - wo] == 0 and b[N - wo + gm.M128] == gm.M128 and b[N - wo + (1 << 128)] == 1 << 128
            assert b[N - wo - 1] == N - 1                                   # the add reaching exactly n, and one short of it
    e = gm.export_biased(wo)
    assert {wo, gm.M128} <= set(e) and all(0 <= v <= gm.M128 for v in e)
    if wo:
        assert gm.exported(wo - 1, wo, True) == N - 1                       # the borrow: + n
    for v in e:
        assert gm.biased(gm.exported(v, wo, True), wo, True) == v and gm.exported(v, wo, False) == v


@needs_ref
def test_the_model_agrees_with_the_reference_wcheck(tmp_path):
    """a plain one-key file of the classes the reference can check (no point at infinity or doubling on the way): the
    reference's DP Wrong count is the model's"""
    kk = gm.key_scalars(1)
    ents = [e for e in gm.batch_entries(kk) if e.cls in ("match", "tame", "max", "bad_x", "bad_h")]
    w = gm.work_of(ents, gm.pub_of(kk[0]))
    path = tmp_path / "plain.work"
    path.write_bytes(gm.file_bytes(w, kk, block=False))
    want = gm.wrong_positions(w, [gm.key_point(kk[0])])
    assert 0 < len(want) < w.entries()
    out = subprocess.run([REFBIN, "-t", "1", "-wcheck", str(path)], capture_output=True, text=True, timeout=300).stdout
    m = re.search(r"DP Wrong: (\d+)", out)
    assert m, out[-2000:]
    assert int(m.group(1)) == len(want), out[-2000:]
    assert "DP: %d" % w.entries() in out or str(w.entries()) in out, out[-2000:]
