"""Transcripts of the oracle-vs-reference comparisons (tests/test_oracle_vs_ref.py).

Each function runs one fixed, seeded workload on a back end (oracle.kgo.Oracle or oracle.kgo.Reference, which share
the same method set) and returns the list of every value it produced.  tests/golden/make_ref_golden.py runs them on the
reference's own SECPK1 code and stores a SHA-256 of each transcript (plus its first entries, for diagnosis) in
tests/golden/ref_golden.json; the tests run them on the oracle and compare.  Hashing keeps the stored vectors small while
the comparison stays value for value."""
import hashlib
import json
import random

import numpy as np

from oracle import kgo

P, N = kgo.P, kgo.N
KEY_PRIV = 0x5B3F38AF935A3640D158E871CE6E9666DB862636383386EE510F18CCC3BD72EB
SYM_KEY_PRIV = 0x5B3F38AF935A3640D158E871CE6E9666DB862636383386EE0000000000123000
SYM_RANGE_POWERS = (40, 56, 64, 80, 109, 125)


def _rows(*arrays):
    return [[int(v) for v in a.reshape(-1)] for a in arrays]


def field_ops(be):
    rng = random.Random(3)
    edge = [0, 1, 2, P - 1, P - 2, 0x1000003D1, 2**255, 2**256 - 1 - 0x1000003D1, 2**128 - 1]
    vals = edge + [rng.randrange(P) for _ in range(3000)]
    out = []
    for i in range(len(vals) - 1):
        a, b = vals[i], vals[i + 1]
        out += [be.mod_mul(a, b), be.mod_sqr(a), be.mod_sub(a, b)]
    out += [be.mod_inv(a) for a in vals[:300]]
    return out


def order_ops(be):
    rng = random.Random(4)
    out = []
    for _ in range(500):
        a, b = rng.randrange(N), rng.randrange(N)
        out += [be.order_add(a, b), be.order_sub(a, b)]
    return out


def rng_and_rand(be):
    out = []
    for seed in (0, 1, 0x600DCAFE, 0xFFFFFFFF):
        be.rseed(seed)
        out += [be.rndl() for _ in range(700)]
        out += [be.rand_bits(nbit) for nbit in (1, 31, 32, 33, 64, 65, 128, 255, 256)]
    return out


def scalar_mult_and_add(be):
    rng = random.Random(5)
    ks = [1, 2, 3, 255, 256, 257, 2**64, N - 1, N - 2] + [rng.randrange(1, N) for _ in range(40)]
    pts = [be.ec_mul_g(k) for k in ks]
    out = list(pts)
    for i in range(len(pts) - 1):
        if pts[i][0] != pts[i + 1][0]:
            out.append(be.ec_add(pts[i], pts[i + 1]))
    return out


def jump_tables(be):
    out = []
    for rp in (32, 40, 48, 56, 64, 72, 80, 84, 110, 115, 125, 256):
        out.append(_rows(*be.create_jump_table(rp)) + [be.last_draws])
    return out


def herd_and_jump_loop(be, grp):
    """grp: kangaroos per batch inverse of the back end's SolveKeyCPU loop (the results do not depend on it)."""
    table = be.create_jump_table(64)
    key = be.ec_mul_g(KEY_PRIV)
    out = []
    for first_type in (0, 1):
        be.rseed(42)
        herd = be.create_herd(300, 64, 2**63 - 1, key, first_type)
        out.append(_rows(*herd))
    mask = kgo.Oracle().dp_mask(6)
    dps = be.jump_cpu(*herd, table, 70, mask, grp=grp)
    out.append(_rows(*herd))
    out.append(sorted(dps))
    x, y, d = (kgo.from_limbs(v[7]) for v in be.create_herd(8, 64, 2**63 - 1, key, 0))
    for _ in range(20):
        x, y, d = be.jump_single(x, y, d, table)
    out.append((x, y, d))
    return out


def hash_convert(be):
    rng = random.Random(6)
    out = []
    for _ in range(200):
        x = rng.randrange(P)
        d = rng.randrange(2**126) if rng.random() < 0.5 else N - rng.randrange(1, 2**126)
        t = rng.randrange(2)
        out.append(be.hash_convert(x, d, t))
    return out


def symmetric_jump_table(be, rp):
    rows = _rows(*be.create_jump_table_sym(rp))
    return [list(be.last_uv), be.last_draws] + rows


def symmetric_herd_and_walk(be, grp):
    """-> (transcript, final herd arrays and rule state) for the invariant checks of the test."""
    rp, n = 64, 96
    key = be.ec_mul_g(SYM_KEY_PRIV)
    wdiv4 = ((1 << rp) - 1) >> 2
    table = be.create_jump_table_sym(rp)
    be.rseed(777)
    px, py, d = be.create_herd_sym(n, rp, wdiv4, key, 0)
    out = [_rows(px, py, d)]
    mask = kgo.Oracle().dp_mask(4)
    for rule, init in (("lastjump", 32), ("symclass", 0)):
        state = np.full(n, init, dtype=np.uint8)
        dps = be.jump_sym(px, py, d, state, table, 200, mask, grp=grp, rule=rule)
        out.append(_rows(px, py, d, state))
        out.append(sorted(dps))
    return out, (px, py, d, state)


def digest(transcript):
    return hashlib.sha256(json.dumps(transcript, default=str).encode()).hexdigest()


def head(transcript, k=4):
    """First entries, as text, so that a mismatch shows where the transcripts part."""
    return json.dumps(transcript[:k], default=str)[:2000]
