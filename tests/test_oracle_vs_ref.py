"""Pin oracle/kgx_oracle.c against the reference's own SECPK1 code.  The reference's results on these seeded workloads
are stored in tests/golden/ref_golden.json (tests/golden/make_ref_golden.py); every test recomputes the same transcript
on the oracle and must reproduce it value for value."""
import json
import os

import pytest

from oracle import kgo
from tests import ref_transcripts as rt

P, N = kgo.P, kgo.N
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_golden.json")


def check(name, transcript):
    with open(GOLDEN) as f:
        want = json.load(f)["transcripts"][name]
    assert len(transcript) == want["entries"], name
    assert rt.digest(transcript) == want["sha256"], "%s: oracle %s vs reference %s" % (name, rt.head(transcript), want["head"])


def test_field_ops(oracle):
    check("field_ops", rt.field_ops(oracle))


def test_order_ops(oracle):
    check("order_ops", rt.order_ops(oracle))


def test_rng_and_rand(oracle):
    check("rng_and_rand", rt.rng_and_rand(oracle))


def test_scalar_mult_and_add(oracle):
    check("scalar_mult_and_add", rt.scalar_mult_and_add(oracle))


def test_jump_tables_all_range_powers(oracle):
    check("jump_tables", rt.jump_tables(oracle))


def test_herd_and_jump_loop(oracle):
    """Herds of both types, 70 jumps of the SolveKeyCPU loop (oracle: 128 kangaroos per inverse, reference: 1024) with
    their DPs, and 20 single-AddDirect jumps of the Check.cpp replay."""
    t = rt.herd_and_jump_loop(oracle, grp=128)
    assert len(t[3]) > 200
    check("herd_and_jump_loop", t)


def test_hash_convert(oracle):
    check("hash_convert", rt.hash_convert(oracle))


# ---- USE_SYMMETRY restatement (SURVEY 8f/f4) pinned to the reference's own Int / Secp256K1 code -------------------------
@pytest.mark.parametrize("rp", list(rt.SYM_RANGE_POWERS))
def test_symmetric_jump_table_matches_reference(oracle, rp):
    """Kangaroo.cpp:742-832 USE_SYMMETRY branch: the two primes u, v come from Int::IsProbablePrime, whose Miller-Rabin bases
    are drawn from the same MT19937 stream as the distances -- the oracle reproduces that consumption exactly."""
    check("symmetric_jump_table_%d" % rp, rt.symmetric_jump_table(oracle, rp))
    jd = oracle.create_jump_table_sym(rp)[0]
    u, v = oracle.last_uv
    assert all(int(jd[i, 0]) % u == 0 for i in range(16)) and all(int(jd[i, 0]) % v == 0 for i in range(16, 32))


def test_symmetric_herd_and_walk_match_reference(oracle):
    """CreateHerd (Kangaroo.cpp:670-738, sym branch) and the symmetric walk Check.cpp:534-556 replays (lastJump limiter,
    ModPositiveK1 class switch, d = n - d): oracle (batched inverse, 32 per group) == reference (24 per group), bit for bit."""
    t, (ox, oy, od, lo) = rt.symmetric_herd_and_walk(oracle, grp=32)
    check("symmetric_herd_and_walk", t)
    n = ox.shape[0]
    assert len(t[2]) > 500 and len(t[4]) > 500
    assert set(int(v) for v in lo) == {0, 1}                                  # symclass state after the second walk
    half = (kgo.P - 1) // 2
    assert all(kgo.from_limbs(oy[i]) <= half for i in range(n))
    assert any(kgo.from_limbs(od[i]) > kgo.N // 2 for i in range(n))           # some distances went negative (mod n)
    # invariant of the class walk: tame x == (d*G).x ; wild x == (key + d*G).x or (key - d*G).x -- a class switch negates
    # the whole point, i.e. d AND the key term, which is why CheckKey tries +-key and the four sign pairs (Kangaroo.cpp:218-253)
    key = oracle.ec_mul_g(rt.SYM_KEY_PRIV)
    for i in (0, 1, 2, 3, 50, 95):
        dv = kgo.from_limbs(od[i])
        if i % 2 == 0:
            assert oracle.ec_mul_g(dv)[0] == kgo.from_limbs(ox[i])
        else:
            cands = (oracle.ec_add(key, oracle.ec_mul_g(dv))[0], oracle.ec_add(key, oracle.ec_mul_g(N - dv))[0])
            assert kgo.from_limbs(ox[i]) in cands
