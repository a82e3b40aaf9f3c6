"""Crafted inputs for the group-law edge tests (tests/test_group_law_edges_cpu.py, tests/test_gpu_group_law_edges.py) and a
big-integer model of the work-file check.

Every key here has a known scalar: the key to search K = pub - start*G = k*G, so a crafted entry or kangaroo can sit exactly
on K, on -K, on 2K or on the x of another key.  Expected values come from kangaroo_b200.ecmath alone, never from the engine.

The check model (kgx_work_check, kgx_work_check_records): a table entry {x lo 128, tagged d} of bucket h passes when
S = +-|d|*G (bit 127 the sign, bit 126 the herd, |d| the low 126 bits) plus K -- for a wild entry, K of some key of the file;
S itself when that K is the point at infinity -- follows the group law (a doubling is fine) to a point whose x has bits
128..145 equal to h and low 128 bits equal to x.  The point at infinity passes nothing.  A kangaroo record {x, y, d} is tame
OK when (x, y) = d*G, else wild OK when (x, y) = K_target + d*G, wrong when neither holds or d >= n or min(d, n - d) >= 2^128."""
import random
import struct
from collections import namedtuple

from kangaroo_b200 import ecmath as ec

N = ec.N
M64 = (1 << 64) - 1
M128 = (1 << 128) - 1
MAG = (1 << 126) - 1
WILD_BIT, NEG_BIT = 1 << 126, 1 << 127
KB = 8                                   # keys per batched inverse in wt_check_entries_multi_kernel
START = 0x9E3779B97F4A7C15
END = START + (1 << 56) - 1
INF_KEY = 2                              # key index whose pub is start*G (K at infinity) when n_keys > 2


# ---- keys -----------------------------------------------------------------------------------------------------------------
def key_scalars(n_keys, seed=1):
    """k of every key: 100-bit values, every fourth one negated (so that S = +K needs the sign bit); with 3 keys or more key 2
    is at infinity; with 7 or more keys 6 repeats key 3; key 4 has its negative at 12 (17 keys) or 5 (7 to 12 keys)"""
    rnd = random.Random(seed * 1000 + n_keys)
    kk = [rnd.getrandbits(100) | (1 << 99) for _ in range(n_keys)]
    for i in range(1, n_keys, 4):
        kk[i] = N - kk[i]
    if n_keys > INF_KEY:
        kk[INF_KEY] = 0
    if n_keys >= 7:
        kk[6] = kk[3]
        kk[12 if n_keys > 12 else 5] = N - kk[4]
    return kk


def key_point(k):
    """K = k*G, None for the point at infinity"""
    return ec.mul(k)


def pub_of(k):
    """the public key whose K is k*G"""
    return ec.mul((k + START) % N)


def key_pairs(n_keys):
    """(same, opposite): index pairs of keys that are the same point and that are each other's negative"""
    if n_keys < 7:
        return [], []
    return [(3, 6)], [(4, 12 if n_keys > 12 else 5)]


# ---- table entries --------------------------------------------------------------------------------------------------------
Entry = namedtuple("Entry", "cls key other h x d")     # key: the key it is built on (or None); other: the key it shares x with


def tagged(mag, wild, neg):
    assert 0 <= mag <= MAG
    return mag | (WILD_BIT if wild else 0) | (NEG_BIT if neg else 0)


def signed_mag(k):
    """(|d|, sign) with +-|d| = k mod n, |d| < 2^126"""
    if k < (1 << 126):
        return k, False
    assert N - k < (1 << 126)
    return N - k, True


def s_point(d):
    """S = +-|d|*G of a tagged distance"""
    s = ec.mul(d & MAG)
    return ec.neg(s) if d & NEG_BIT else s


def hx(pt):
    """(bucket, stored x) of a point"""
    return (pt[0] >> 128) & 0x3FFFF, pt[0] & M128


def entry_ok(h, x, d, keys):
    """the check model for one table entry; keys: the K of every key of the file (None = infinity)"""
    s = s_point(d)
    cands = [ec.add(s, K) for K in keys] if d & WILD_BIT else [s]
    return any(p is not None and hx(p) == (h, x) for p in cands)


def match_indices(n_keys):
    """keys at the edges of the batches of 8 that a wild entry is made to match"""
    return sorted({0, 7, 8, 9, 15, 16, n_keys - 1} & set(range(n_keys)) - {INF_KEY})


def shared_pairs(n_keys, kk):
    """(j, j') in one batch of 8, both keys finite: an entry whose S is +-K_j and which matches K_j' (both orders)"""
    out = []
    for b0 in range(0, n_keys, KB):
        fin = [j for j in range(b0, min(b0 + KB, n_keys)) if kk[j]]
        if len(fin) >= 2:
            out += [(fin[0], fin[-1]), (fin[-1], fin[0])]
    return out


def batch_entries(kk, seed=5):
    """the crafted entries of a batch file of keys kk: a list of Entry, every class tame and wild where it makes sense, with
    the sign bit both ways"""
    rnd = random.Random(seed)
    n = len(kk)
    K = [key_point(k) for k in kk]
    out = []

    def add(cls, key, pt, d, other=None):
        h, x = hx(pt) if pt is not None else (rnd.getrandbits(18), rnd.getrandbits(128))
        out.append(Entry(cls, key, other, h, x, d))

    for neg in (False, True):
        for j in match_indices(n):                                     # a match at the edges of the batches
            m = rnd.getrandbits(100)
            add("match", j, ec.add(s_point(tagged(m, True, neg)), K[j]), tagged(m, True, neg))
        for m in (rnd.getrandbits(100), MAG):                          # tame, and the largest magnitude
            add("tame", None, s_point(tagged(m, False, neg)), tagged(m, False, neg))
        j = match_indices(n)[-1]
        add("max", j, ec.add(s_point(tagged(MAG, True, neg)), K[j]), tagged(MAG, True, neg))
        for j in sorted({0, n - 1} - {INF_KEY}):                        # magnitude 0: the point is K itself
            add("zero", j, K[j], tagged(0, True, neg))
        add("zero_tame", None, None, tagged(0, False, neg))            # the point at infinity: wrong
        if n > INF_KEY:                                                # S itself, through the key at infinity
            m = rnd.getrandbits(100)
            add("inf_key", INF_KEY, s_point(tagged(m, True, neg)), tagged(m, True, neg))
    for j in range(n):
        if not kk[j]:
            continue
        m, neg = signed_mag(kk[j])
        add("dbl", j, ec.add(K[j], K[j]), tagged(m, True, neg))        # S = +K: a doubling
        m, neg = signed_mag(N - kk[j])
        add("opp", j, None, tagged(m, True, neg))                      # S = -K: infinity, no match with j
    for j, j2 in shared_pairs(n, kk):
        for sign in (1, -1):                                           # S = +-K_j, matching K_j'
            m, neg = signed_mag(kk[j] if sign == 1 else N - kk[j])
            d = tagged(m, True, neg)
            add("shared", j2, ec.add(s_point(d), K[j2]), d, other=j)
    # one wrong x bit and a bucket one off, on entries that are right otherwise
    good = [e for e in out if e.cls in ("match", "tame", "dbl")]
    for i, e in enumerate(good[::3]):
        out.append(e._replace(cls="bad_x", x=e.x ^ (1 << (17 * i % 128))))
        out.append(e._replace(cls="bad_h", h=(e.h + (1 if i % 2 else -1)) % (1 << 18)))
    return out


# ---- kangaroo records -----------------------------------------------------------------------------------------------------
Walk = namedtuple("Walk", "cls x y d target")


def walk_kind(x, y, d, K):
    """the check model for one kangaroo record against its target's K (None = infinity): 1 tame OK, 2 wild OK, 0 wrong"""
    if d >= N or min(d, N - d) >= (1 << 128):
        return 0
    p = ec.mul(d)
    if p is not None and p == (x, y):
        return 1
    q = ec.add(p, K)
    return 2 if q is not None and q == (x, y) else 0


def batch_walks(kk, seed=7):
    """crafted kangaroo records of a batch file of keys kk (n_keys >= 7): tame and wild ones, a wild of the last key, wilds
    whose target is the key at infinity, wilds at distance 0, right points under a wrong target (a key equal to the right
    one, its negative, another key), d >= n, magnitudes >= 2^128 and a flipped y"""
    rnd = random.Random(seed)
    n = len(kk)
    K = [key_point(k) for k in kk]
    out = []

    def wild(j, d, target=None, cls="wild"):
        p = ec.add(K[j], ec.mul(d))
        out.append(Walk(cls, p[0], p[1], d, j if target is None else target))

    for i in range(4):
        d = rnd.getrandbits(90) if i % 2 else N - rnd.getrandbits(80)
        p = ec.mul(d)
        out.append(Walk("tame", p[0], p[1], d, rnd.randrange(n)))
        wild(rnd.choice([j for j in range(n) if kk[j]]), d)
    wild(n - 1, rnd.getrandbits(90), cls="last")
    d = rnd.getrandbits(90)
    p = ec.mul(d)
    out.append(Walk("inf_target", p[0], p[1], d, INF_KEY))                # K at infinity: the point is d*G (tame OK)
    out.append(Walk("inf_target_zero", 0, 0, 0, INF_KEY))                 # K + 0*G at infinity: wrong
    for j in (0, n - 1):
        wild(j, 0, cls="zero")
    (a, a2), = key_pairs(n)[0]
    (b, b2), = key_pairs(n)[1]
    wild(a, rnd.getrandbits(90), a2, "same_key_target")                    # K_a2 == K_a: OK
    wild(b, rnd.getrandbits(90), b2, "neg_key_target")                     # K_b2 == -K_b: wrong
    wild(0, rnd.getrandbits(90), n - 1, "wrong_target")
    p = ec.mul(5)
    out.append(Walk("d_ge_n", p[0], p[1], N + 5, 0))
    p = ec.mul(1 << 130)
    out.append(Walk("mag_2_128", p[0], p[1], 1 << 130, 0))
    p = ec.mul(N - 1)
    out.append(Walk("n_minus_1", p[0], p[1], N - 1, 0))                    # magnitude 1, negative: -G
    d = rnd.getrandbits(90)
    p = ec.add(K[n - 1], ec.mul(d))
    out.append(Walk("bad_y", p[0], p[1] ^ 1, d, n - 1))
    return out


def walk_bytes(walks):
    """the kangaroo block of a HEADW file: the count, then {x, y, d} as 4 u64 limbs each"""
    return struct.pack("<Q", len(walks)) + b"".join(struct.pack("<12Q", *[(v >> (64 * k)) & M64 for v in (w.x, w.y, w.d) for k in range(4)])
                                                    for w in walks)


def work_of(entries, key):
    """a HEADW file (tests.worktool_util.Work) of the entries, public key `key` in the header, no kangaroos"""
    from tests.worktool_util import Work
    w = Work(14, START, END, key, 1000, 1.5)
    for e in entries:
        w.add(e.x, e.d, e.h)
    return w


def file_bytes(w, kk, walks=(), block=True):
    """w's bytes with the kangaroo records `walks`, followed by the batch block of keys kk (all unsolved) and the walks'
    targets when `block`"""
    from kangaroo_b200.worktool import BatchBlock, batch_block
    w.walks = walk_bytes(walks)
    plain = w.to_bytes()
    if not block:
        return plain
    b = BatchBlock([pub_of(k) for k in kk], [False] * len(kk), [None] * len(kk), [v.target for v in walks])
    return plain + batch_block(b, len(plain)).tobytes()


def wrong_positions(w, keys):
    """the model's wrong entries of w as (bucket, index in bucket), file order; keys: the K of every key (None = infinity)"""
    return [(h, i) for h in range(len(w.table)) for i, (x, d) in enumerate(w.table[h]) if not entry_ok(h, x, d, keys)]


# ---- retargeting ----------------------------------------------------------------------------------------------------------
RETARGET_NTO = 7


def retarget_case(n, seed=3):
    """A multi-key herd of n kangaroos whose retarget from key 0 meets every degenerate branch.  -> dict:
    ks: key scalars (keys = ks*G); special: {kIdx: (kind, d, b)} wilds of key 0 with chosen scalars d moved to key b; to: the
    destination list (spread rule to[(kIdx >> 1) % len(to)]).
      p_eq_delta  keys[b] = 2*keys[0] + d*G: the point K_0 + d*G equals delta = K_b - K_0, a doubling, giving 2P = K_b + d*G;
      p_neg_delta keys[b] = -d*G: the point is -delta, the result is infinity, stored as (0, 0);
      key 1 = -key 0: the delta itself is a doubling (-2 K_0).
    Two of the specials are kIdx n - 1 and n - 3, in the padded last tile."""
    rnd = random.Random(seed)
    k0 = rnd.getrandbits(62) | (1 << 62)
    ks = [k0, N - k0]
    special, to = {}, [None] * RETARGET_NTO
    for s, kind in ((1, "p_eq_delta"), (3, "p_neg_delta"), (n - 1, "p_neg_delta"), (n - 3, "p_eq_delta")):
        d = rnd.getrandbits(60) | 1
        ks.append((2 * k0 + d) % N if kind == "p_eq_delta" else N - d)
        j = (s >> 1) % RETARGET_NTO
        assert to[j] is None
        to[j] = len(ks) - 1
        special[s] = (kind, d, len(ks) - 1)
    ks.append(rnd.getrandbits(62) | (1 << 61))                              # an ordinary destination
    free = [j for j in range(RETARGET_NTO) if to[j] is None]
    for i, j in enumerate(free):
        to[j] = 1 if i % 2 == 0 else len(ks) - 1
    return dict(ks=ks, special=special, to=to)


# ---- the checkpoint conversion --------------------------------------------------------------------------------------------
WILD_OFFSETS = (0, 1, 1 << 127, (1 << 128) - 1)


def import_distances(wo, wild):
    """record distances at the edges of herd_import_kernel's reductions"""
    ds = [0, 1, N - 1, N, N + 1, M128, 1 << 128, N + M128, (1 << 256) - 1]
    if wild:
        ds += [N - wo, N - wo - 1, N - wo + M128, N - wo + (1 << 128)]
    assert all(0 <= d < (1 << 256) for d in ds)
    return ds


def biased(d, wo, wild):
    """the engine's distance of record distance d: ((d mod n) + wo) mod n for a wild kangaroo, d mod n for a tame one"""
    return ((d % N) + (wo if wild else 0)) % N


def export_biased(wo):
    """biased distances at the edges of herd_export_kernel's borrow"""
    return sorted({b for b in (0, wo - 1, wo, wo + 1, M128) if 0 <= b <= M128})


def exported(b, wo, wild):
    return (b - wo) % N if wild else b
