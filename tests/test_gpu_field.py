"""-m gpu: device field arithmetic (kgx_field.cuh, kgx_modinv.h) bit-exact against the oracle through the C ABI, and the
branch-free primitives of the jump, herd and DP-conversion kernels at the values where their branches flip -- values random
walks reach with probability 2^-80 or less -- against plain big-integer references written here."""
import ctypes
import os
import random
import re

import numpy as np
import pytest

import kangaroo_b200
from oracle import kgo

pytestmark = pytest.mark.gpu
P = kgo.P
N = kgo.N
C = 0x1000003D1                  # 2^256 mod p
M256 = 2**256 - 1
M128 = 2**128 - 1
HALF = (P - 1) // 2
ALL = 0xFFFFFFFF
_u64p = ctypes.POINTER(ctypes.c_uint64)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OP = {m.group(1): int(m.group(2))
      for m in re.finditer(r"#define\s+KGX_TF_(\w+)\s+(\d+)", open(os.path.join(ROOT, "include", "kgx.h")).read())}


def run(op, a_vals, b_vals):
    lib = kangaroo_b200.load_library()
    a = kgo.ints_to_array(a_vals); b = kgo.ints_to_array(b_vals)
    out = np.zeros_like(a)
    op = OP[op] if isinstance(op, str) else op
    rc = lib.kgx_test_field(0, op, len(a_vals), a.ctypes.data_as(_u64p), b.ctypes.data_as(_u64p), out.ctypes.data_as(_u64p))
    assert rc == 0, lib.kgx_last_error(None)
    return kgo.array_to_ints(out)


EDGE = [0, 1, 2, 3, P - 1, P - 2, P, P + 1, P + 5, 2**256 - 1, 2**256 - 2, 0x1000003D1, 0x1000003D0, 2**255, 2**128 - 1, 2**128,
        2**32 - 1, 2**32, 2**64 - 1, 2**224 + 1, (P + 1) // 2, 0xFFFFFFFF00000000FFFFFFFF00000000FFFFFFFF00000000FFFFFFFF00000000]


def pairs():
    rng = random.Random(7)
    a = [x for x in EDGE for _ in EDGE] + [rng.randrange(2**256) for _ in range(20000)] + [rng.randrange(P) for _ in range(20000)]
    b = [y for _ in EDGE for y in EDGE] + [rng.randrange(2**256) for _ in range(20000)] + [rng.randrange(P) for _ in range(20000)]
    return a, b


def test_mul_bit_exact(oracle):
    a, b = pairs()
    got = run(0, a, b)
    for x, y, g in zip(a, b, got):
        assert g == oracle.mod_mul(x, y), (hex(x), hex(y))


def test_sqr_bit_exact(oracle):
    a, _ = pairs()
    got = run(1, a, a)
    for x, g in zip(a, got):
        assert g == oracle.mod_sqr(x), hex(x)


def test_sub_bit_exact(oracle):
    a, b = pairs()
    got = run(2, a, b)
    for x, y, g in zip(a, b, got):
        assert g == oracle.mod_sub(x, y), (hex(x), hex(y))


def test_inv_canonical(oracle):
    rng = random.Random(9)
    a = [0, 1, 2, P - 1, P - 2, 2**255, (P + 1) // 2] + [2**k for k in range(0, 256, 3)] + [rng.randrange(1, P) for _ in range(4000)]
    got = run(3, a, a)
    for x, g in zip(a, got):
        assert g == (pow(x, -1, P) if x else 0), hex(x)


# ---- plain big-integer references ---------------------------------------------------------------------------------------

def fold_ref(w):
    """The reference's 512 -> 256 fold (IntMod.cpp / GPUMath.h): -> (result, whether the last carry was dropped)."""
    r1 = (w & M256) + (w >> 256) * C
    s = (r1 & M256) + (r1 >> 256) * C
    return s & M256, s > M256


def sub_ref(a, b):
    """a - b mod 2^256, plus p (mod 2^256) when the subtraction borrowed."""
    return (a - b + (P if a < b else 0)) & M256


# Each 32-bit limb from this palette (None = random): carries then run through long stretches of full or empty limbs, which
# uniform random operands almost never produce.
PALETTE = [0, 1, 2, 0x3D0, 0x3D1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF, None]


def palette_values(n, seed):
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        v = 0
        for k in range(8):
            limb = rng.choice(PALETTE)
            v |= (rng.getrandbits(32) if limb is None else limb) << (32 * k)
        out.append(v)
    return out


# Operands whose fold drops its last carry (the result is then NOT congruent to the product): (2^256 - m)^2 for small m, and
# (2^256 - 1) * b with b the least value for which the first fold's high part is t and its low part lands within t*c of 2^256.
SQR_DROPPED = [2**256 - m for m in list(range(1, 65)) + [0x3D0, 0x3D1, 2**16, 2**31, C - 2**17]]
MUL_DROPPED = [(M256, -(-(t * 2**256 - t * C + C) // (C - 1))) for t in (1, 2, 3, 0x3D1, 2**16, 2**31, 2**32, C - 3)]


def check_fold(x, y, g):
    want, dropped = fold_ref(x * y)
    assert g == want, (hex(x), hex(y))
    if not dropped:
        assert g % P == x * y % P, (hex(x), hex(y))
    return dropped


@pytest.mark.parametrize("op", ["MUL", "MUL_INPLACE"])
def test_mul_limb_palette_and_dropped_carry(oracle, op):
    a, b = palette_values(100000, 11), palette_values(100000, 12)
    a += [x for x, _ in MUL_DROPPED] + SQR_DROPPED
    b += [y for _, y in MUL_DROPPED] + SQR_DROPPED
    got = run(op, a, b)
    dropped = [check_fold(x, y, g) for x, y, g in zip(a, b, got)]
    assert sum(dropped[-len(MUL_DROPPED) - len(SQR_DROPPED):]) == len(MUL_DROPPED) + len(SQR_DROPPED)
    for x, y, g in zip(a, b, got):
        assert g == oracle.mod_mul(x, y), (hex(x), hex(y))


@pytest.mark.parametrize("op", ["SQR", "SQR_INPLACE"])
def test_sqr_limb_palette_and_dropped_carry(oracle, op):
    a = palette_values(100000, 13) + SQR_DROPPED
    got = run(op, a, a)
    dropped = [check_fold(x, x, g) for x, g in zip(a, got)]
    assert sum(dropped[-len(SQR_DROPPED):]) == len(SQR_DROPPED)
    for x, g in zip(a, got):
        assert g == oracle.mod_sqr(x), hex(x)


@pytest.mark.parametrize("op", ["SUB", "SUB_INPLACE"])
def test_sub_limb_palette(oracle, op):
    a, b = palette_values(100000, 14) + EDGE * len(EDGE), palette_values(100000, 15) + [y for y in EDGE for _ in EDGE]
    got = run(op, a, b)
    for x, y, g in zip(a, b, got):
        assert g == sub_ref(x, y) == oracle.mod_sub(x, y), (hex(x), hex(y))


def test_inv_of_values_above_p():
    """Products of fe_mul live in [0, 2^256): an input in (p, 2^256) must give the inverse of its residue.  (p itself is
    documented to give 1 and cannot come from the jump, herd or import paths.)"""
    rng = random.Random(17)
    a = [P + k for k in range(1, 6)] + [2**256 - k for k in range(1, 6)] + [P + 0x3D1, P + 2**32] + \
        [rng.randrange(P + 1, 2**256) for _ in range(4000)]
    got = run("INV", a, a)
    for x, g in zip(a, got):
        assert g == pow(x - P, -1, P), hex(x)


def around(*centres):
    return sorted({(c + k) & M256 for c in centres for k in range(-3, 4)})


# every value within 3 of the branch points, (p-1)/2 off by one in each 32-bit word, and p with each word forced to 0 / all
# ones / off by one
BOUNDARY = sorted(set(around(HALF, P, 0, 2**256)) | {HALF + s * (1 << (32 * w)) for w in range(8) for s in (-1, 1)}
                  | {(P & ~(ALL << (32 * w))) | (v << (32 * w)) for w in range(8) for v in (0, 1, ALL, ALL - 1, (P >> (32 * w)) & ALL ^ 1)})


def test_gt_half_mask_at_boundaries():
    vals = BOUNDARY + palette_values(20000, 19)
    got = run("GT_HALF", vals, vals)
    for v, g in zip(vals, got):
        assert g == (ALL if v > HALF else 0), hex(v)
    assert HALF in vals and HALF + 1 in vals


def test_cneg_at_boundaries():
    vals = BOUNDARY + palette_values(20000, 21)
    for mask in (0, ALL):
        got = run("CNEG", vals, [mask] * len(vals))
        for v, g in zip(vals, got):
            assert g == ((P - v) & M256 if mask else v), (hex(v), mask)


def test_is_zero_modp_at_boundaries():
    vals = BOUNDARY + palette_values(20000, 23) + [1 << k for k in range(256)] + [P ^ (1 << k) for k in range(256)]
    got = run("IS_ZERO", vals, vals)
    for v, g in zip(vals, got):
        assert g == (1 if v % P == 0 else 0), hex(v)
    assert 0 in vals and P in vals


def test_neg_and_dbl():
    vals = BOUNDARY + EDGE + palette_values(50000, 25)
    got_neg = run("NEG", vals, vals)
    got_dbl = run("DBL", vals, vals)
    for v, n, d in zip(vals, got_neg, got_dbl):
        assert n == sub_ref(0, v), hex(v)
        assert d == sub_ref(v, sub_ref(0, v)), hex(v)
        if v < P:
            assert n % P == -v % P and d % P == 2 * v % P, hex(v)


D128_EDGE = [0, 1, 2, M128, M128 - 1, 2**127, 2**127 - 1, 2**127 + 1, 2**126, 2**64 - 1, 2**64, 2**96 - 1, 2**128 - 2**64]


def test_d128_add_and_cneg():
    rng = random.Random(27)
    extra = [rng.getrandbits(128) for _ in range(2000)]
    a = [x for x in D128_EDGE for _ in D128_EDGE] + extra
    b = [y for _ in D128_EDGE for y in D128_EDGE] + extra[::-1]
    got = run("D128_ADD", a, b)
    for x, y, g in zip(a, b, got):
        assert g == (x + y) & M128, (hex(x), hex(y))
    for mask in (0, ALL):
        got = run("D128_CNEG", a, [mask] * len(a))
        for x, g in zip(a, got):
            assert g == ((-x) & M128 if mask else x), (hex(x), mask)


LASTJUMP, SYMCLASS = 1, 2


def jump_index_ref(x0, aux, rule):
    if rule == SYMCLASS:
        return (x0 & 15) | ((aux & 1) << 4)
    j0 = x0 & 31
    return (aux + 1) & 31 if j0 == aux else j0


def test_jump_index_both_rules():
    rng = random.Random(29)
    cases = []
    for rule in (LASTJUMP, SYMCLASS):
        for aux in (0, 30, 31, 32):                                  # 32 = no previous jump
            for low in {aux % 32, (aux + 1) % 32, (aux - 1) % 32}:
                for high in (0, 0x7FFFFFF, 0x7FFFFFF & rng.getrandbits(27)):
                    cases.append(((high << 5) | low, aux, rule))
        cases += [(rng.getrandbits(32) & ~31 | low, aux, rule) for aux in range(33) for low in range(32)]
    got = run("JUMP_INDEX", [x for x, _, _ in cases], [aux | (rule << 32) for _, aux, rule in cases])
    for (x, aux, rule), g in zip(cases, got):
        assert g & ALL == jump_index_ref(x, aux, rule), (hex(x), aux, rule)
        assert g >> 32 == x & 31, (hex(x), aux, rule)


def test_sym_next_aux_both_rules():
    cases = [(j, neg, aux, rule) for rule in (LASTJUMP, SYMCLASS) for aux in (0, 1, 30, 31, 32) for j in range(32) for neg in (0, ALL)]
    got = run("SYM_NEXT_AUX", [j | (neg << 32) for j, neg, _, _ in cases], [aux | (rule << 32) for _, _, aux, rule in cases])
    for (j, neg, aux, rule), g in zip(cases, got):
        assert g == (j if rule == LASTJUMP else (aux & 1) ^ (neg & 1)), (j, neg, aux, rule)


def test_unknown_op_is_rejected():
    lib = kangaroo_b200.load_library()
    a = np.zeros((1, 4), dtype=np.uint64)
    assert lib.kgx_test_field(0, max(OP.values()) + 1, 1, a.ctypes.data_as(_u64p), a.ctypes.data_as(_u64p), a.ctypes.data_as(_u64p)) != 0


# ---- device HashTable::Convert (dp_convert_kernel) ----------------------------------------------------------------------

def dp_convert(recs, wild_offset, signed, count=None, max_found=None):
    """recs: list of (x, biased d, kIdx) -> (count word, list of (kIdx32, h, x128, raw 128-bit tagged d)) over max_found slots."""
    lib = kangaroo_b200.load_library()
    count = len(recs) if count is None else count
    max_found = len(recs) if max_found is None else max_found
    arr = np.zeros((max(len(recs), 1), 7), dtype=np.uint64)
    for i, (x, d, k) in enumerate(recs):
        arr[i, 0:4] = kgo.to_limbs(x); arr[i, 4:6] = kgo.to_limbs(d, 2); arr[i, 6] = k
    wo = kgo.to_limbs(wild_offset, 2)
    out = np.zeros(4 + max_found * 40, dtype=np.uint8)
    rc = lib.kgx_test_dp_convert(0, count, max_found, arr.ctypes.data_as(ctypes.c_void_p), wo.ctypes.data_as(_u64p), int(signed),
                                 out.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0, lib.kgx_last_error(None)
    b = out.tobytes()
    rows = []
    for o in range(4, len(b), 40):
        rows.append((int.from_bytes(b[o:o + 4], "little"), int.from_bytes(b[o + 4:o + 8], "little"),
                     int.from_bytes(b[o + 8:o + 24], "little"), int.from_bytes(b[o + 24:o + 40], "little")))
    return int.from_bytes(b[:4], "little"), rows


def convert_ref(oracle, x, d, kidx, wild_offset, signed):
    """HashTable::Convert of the distance GPUEngine.cu:672 forms: (biased - wild offset) mod n for wild kangaroos; in signed
    mode the record holds a two's complement 128-bit distance and no offset."""
    ktype = kidx & 1
    if signed:
        dist = (d - 2**128) % N if d >> 127 else d
    else:
        dist = (d - wild_offset) % N if ktype else d
    h, X, D = oracle.hash_convert(x, dist, ktype)
    return kidx & ALL, h, X, D


WILD_OFFSETS = [(2**79 - 1), (1 << 64) + 5, (0x1234 << 64) | 0xFFFFFFFFFFFFFFF0, (1 << 124) + 0xDEADBEEF, 2**127 - 1]
KIDX = [1, 2, 2**32 - 1, 2**32, 2**32 + 1, 2**33 + 6, 2**63 + 3, 2**64 - 2]


def crafted_unsigned(wo, rng):
    wo0, wo1 = wo & (2**64 - 1), wo >> 64
    ds = [wo, wo + 1, wo - 1, wo + 2**64, wo - 2**64,
          (wo1 << 64) | 0, (wo1 << 64) | (2**64 - 1), (wo1 << 64) | max(wo0 - 1, 0), (wo1 << 64) | min(wo0 + 1, 2**64 - 1),
          ((wo1 + 1) << 64) | 0, ((wo1 + 1) << 64) | max(wo0 - 1, 0), (((wo1 - 1) % 2**64) << 64) | (2**64 - 1),
          0, 1, M128, 2**127, 2**127 - 1, 2**126, 2**126 - 1, 3 << 126, M128 - 2**126]
    return [(rng.getrandbits(256), d & M128, k) for d in ds for k in KIDX]


@pytest.mark.parametrize("wo", WILD_OFFSETS, ids=[hex(w) for w in WILD_OFFSETS])
def test_dp_convert_unsigned_at_offset_boundaries(oracle, wo):
    rng = random.Random(wo & 0xFFFF)
    recs = crafted_unsigned(wo, rng)
    cnt, got = dp_convert(recs, wo, False)
    assert cnt == len(recs)
    for (x, d, k), g in zip(recs, got):
        assert g == convert_ref(oracle, x, d, k, wo, False), (hex(x), hex(d), k)
    # the wild record whose distance equals the offset is +0: no sign bit
    assert any(d == wo and k & 1 and g[3] == 1 << 126 for (x, d, k), g in zip(recs, got))


def test_dp_convert_signed_mode(oracle):
    rng = random.Random(31)
    ds = [0, 1, M128, 2**127, 2**127 - 1, 2**127 + 1, 2**126, M128 - 2**126 + 1, 2**64, M128 - 2**64 + 1]
    recs = [(rng.getrandbits(256), d, k) for d in ds for k in KIDX]
    for wo in (0, 2**79 - 1):                     # the offset must be ignored in signed mode
        cnt, got = dp_convert(recs, wo, True)
        assert cnt == len(recs)
        for (x, d, k), g in zip(recs, got):
            assert g == convert_ref(oracle, x, d, k, wo, True), (hex(x), hex(d), k)


def test_dp_convert_count_and_bulk(oracle):
    """More records than the 64 x 256 threads of the launch (grid-stride loop), a count above max_found (capped) and one below
    it (slots past the count untouched)."""
    rng = random.Random(37)
    wo = 2**79 - 1
    recs = [(rng.getrandbits(256), rng.getrandbits(128), rng.getrandbits(64)) for _ in range(20000)]
    cnt, got = dp_convert(recs, wo, False, count=len(recs) + 777)
    assert cnt == len(recs)
    for (x, d, k), g in zip(recs, got):
        assert g == convert_ref(oracle, x, d, k, wo, False), (hex(x), hex(d), k)
    cnt, got = dp_convert(recs[:100], wo, False, max_found=128)
    assert cnt == 100
    assert all(g == convert_ref(oracle, x, d, k, wo, False) for (x, d, k), g in zip(recs, got[:100]))
    assert all(g == (ALL, ALL, M128, M128) for g in got[100:])
