"""-m gpu: every compiled kernel variant stays bit-exact.  VARIANTS names each instantiation kgx_engine.cu compiles, SYM_VARIANTS
each symmetric-mode one (a CPU test, tests/test_abi_cpu.py, fails when one is added without an entry here).  Each variant runs
the smoke check (1024 kangaroos x 64 jumps vs the oracle, state and DP multiset) in a subprocess, and an in-process shape test on
a herd that pads the last tile of every geometry, loops over tiles, and runs 1 or 63 jumps per launch; each symmetric variant
runs the shape test under both jump rules.  kgx_create reads the KGX_* environment at every create."""
import ctypes
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# KGX_MODE=resident without KGX_CFG is the default geometry, 128,7.  Stream variants without KGX_STREAM_G take the adaptive
# group size: 2 for the smoke herd, 30 (2 CTAs/SM) or 20 (3 CTAs/SM) for the shape herd on 132 SMs.
VARIANTS = [
    {"KGX_MODE": "stream"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "64"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "256"},
    {"KGX_MODE": "resident"},
    {"KGX_MODE": "resident", "KGX_CFG": "64,5"},
    {"KGX_MODE": "resident", "KGX_CFG": "256,3"},
    {"KGX_MODE": "resident", "KGX_CFG": "32,12"},
    {"KGX_MODE": "tmem"},
    # the other resident geometries; 96,6 is the only tile with an odd warp count (3) in tile_inverse
    {"KGX_MODE": "resident", "KGX_CFG": "128,4"},
    {"KGX_MODE": "resident", "KGX_CFG": "128,5"},
    {"KGX_MODE": "resident", "KGX_CFG": "64,7"},
    {"KGX_MODE": "resident", "KGX_CFG": "64,6"},
    {"KGX_MODE": "resident", "KGX_CFG": "64,4"},
    {"KGX_MODE": "resident", "KGX_CFG": "96,6"},
    {"KGX_MODE": "resident", "KGX_CFG": "32,8"},
    # stream_kernel<128, CTAS, WARPINV>: both launch bounds x both group inverses
    {"KGX_MODE": "stream", "KGX_STREAM_CTAS": "2", "KGX_STREAM_INV": "warp"},
    {"KGX_MODE": "stream", "KGX_STREAM_CTAS": "2", "KGX_STREAM_INV": "thread"},
    {"KGX_MODE": "stream", "KGX_STREAM_CTAS": "3", "KGX_STREAM_INV": "warp"},
    {"KGX_MODE": "stream", "KGX_STREAM_CTAS": "3", "KGX_STREAM_INV": "thread"},
    # group sizes: the smallest, one that is not a power of two, the reference's 128, one above it
    {"KGX_MODE": "stream", "KGX_STREAM_G": "2"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "128"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "130"},
    # L2 prefetch distance: off, 1, one where the guard i + pf + 1 < G stops it inside the group, and pf = G (never issued)
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6", "KGX_STREAM_PF": "0"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6", "KGX_STREAM_PF": "1"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6", "KGX_STREAM_PF": "3"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6", "KGX_STREAM_PF": "6"},
]
KGX_VARS = ("KGX_MODE", "KGX_CFG", "KGX_STREAM_G", "KGX_STREAM_CTAS", "KGX_STREAM_INV", "KGX_STREAM_PF")
_SHORT = {"KGX_STREAM_CTAS": "ctas", "KGX_STREAM_INV": "inv", "KGX_STREAM_PF": "pf"}


def variant_id(env):
    return "-".join(_SHORT.get(k, "") + v for k, v in env.items())


VARIANT_IDS = [variant_id(v) for v in VARIANTS]

# Symmetric engine mode (kgx_set_symmetry): kgx_engine.cu compiles one symmetric stream kernel, stream_kernel<128, 2, true, true>,
# and one symmetric tile geometry, 128,7 (KGX_CFG_ENTRY_SYM).  The symmetric engine refuses KGX_STREAM_CTAS=3 and every other
# geometry (tests/test_gpu_errors.py) and ignores KGX_STREAM_INV: it always runs the warp inverse.  The adaptive group size is
# 30 on the shape herd with 132 SMs.
SYM_VARIANTS = [
    {"KGX_MODE": "stream"},
    # group sizes: the smallest, one that is not a power of two, 64, the reference's 128, one above it
    {"KGX_MODE": "stream", "KGX_STREAM_G": "2"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "64"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "128"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "130"},
    # L2 prefetch distance: off, 1, one the guard stops inside the group, pf = G
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6", "KGX_STREAM_PF": "0"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6", "KGX_STREAM_PF": "1"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6", "KGX_STREAM_PF": "3"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "6", "KGX_STREAM_PF": "6"},
    {"KGX_MODE": "stream", "KGX_STREAM_INV": "thread"},      # runs the warp-inverse kernel all the same
    {"KGX_MODE": "resident"},
]
SYM_VARIANT_IDS = [variant_id(v) for v in SYM_VARIANTS]
SYM_RULES = [("lastjump", 32), ("symclass", 0)]             # rule, state byte after SetKangaroos / SetKangaroo


@pytest.mark.parametrize("env", VARIANTS, ids=VARIANT_IDS)
def test_variant_bit_exact(env):
    e = {k: v for k, v in os.environ.items() if k not in KGX_VARS}; e.update(env)
    p = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], cwd=ROOT, env=e,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "smoke ok" in p.stdout, (p.stdout + p.stderr)[-2000:]


SHAPE_GRID = (61, 127)            # 61 x 127 x 128 = 991,616 kangaroos: a multiple of no compiled tile
SAMPLE = 2048


def shape_sample(n, size=SAMPLE):
    """A strided sample plus the last 128 kangaroos, which sit in the padded last tile of every geometry."""
    import numpy as np
    return np.unique(np.concatenate([np.arange(0, n, n // size), np.arange(n - 128, n)]))


@pytest.fixture(scope="module")
def shape_herd():
    import numpy as np
    from kangaroo_b200 import random_herd_arrays
    from tests.golden_util import load_cases
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    n = SHAPE_GRID[0] * SHAPE_GRID[1] * 128
    sc, d128 = random_herd_arrays(n, 80, case["width_div2"], np.random.Generator(np.random.PCG64(4242)))
    return case, sc, d128, shape_sample(n)


@pytest.mark.parametrize("n_run", [1, 63])
@pytest.mark.parametrize("env", VARIANTS, ids=VARIANT_IDS)
def test_variant_shapes_match_oracle(env, n_run, shape_herd, oracle, monkeypatch):
    """991,616 kangaroos made on the device, two launches of n_run jumps.  Walks are independent, so replaying a sample
    through the oracle is exact: the sample's end state (x, y, biased d) and, launch by launch, the DPs of its kangaroos must
    equal the replay; no DP may come from a padding slot."""
    import numpy as np
    from kangaroo_b200 import GPUEngine
    for k in KGX_VARS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    case, sc, d128, idx = shape_herd
    n = sc.shape[0]
    mask = oracle.dp_mask(4 if n_run == 1 else 10)        # about 62 k DPs per launch either way
    max_found = 1 << 17
    eng = GPUEngine(*SHAPE_GRID, 0, max_found)
    assert eng.kernel == env["KGX_MODE"]
    eng.set_jumps_per_launch(n_run)
    eng.SetParams(mask, *case["table"])
    eng.SetWildOffset(case["width_div2"])
    eng.CreateHerdRaw(sc, d128, case["key"])
    ax, ay, ad = eng.GetKangaroosRaw()
    px, py, pd = ax[idx].copy(), ay[idx].copy(), ad[idx].copy()
    eng.callKernel()
    launches = [eng.Launch()]
    assert eng.lastFound <= max_found
    launches.append(eng.Launch(relaunch=False))
    assert eng.lastFound <= max_found
    ax, ay, ad = eng.GetKangaroosRaw()
    eng.close()

    want = oracle.jump_gpu_conv(px, py, pd, case["table"], 2 * n_run, mask)
    assert np.array_equal(ax[idx], px) and np.array_equal(ay[idx], py) and np.array_equal(ad[idx], pd)
    in_sample = set(idx.tolist())
    for launch, found in enumerate(launches):
        assert len(found) > 1000 and max(it.kIdx for it in found) < n
        got = sorted((it.x, it.d, it.kIdx) for it in found if it.kIdx in in_sample)
        exp = sorted((x, eng._unbias(d, int(idx[k])), int(idx[k])) for x, d, k, j in want if (j - 1) // n_run == launch)
        assert got == exp and len(exp) > 50, launch


SYM_RP = 80                       # symmetric table (distances: multiples of two primes near 2^20) and herd (tame d < 2^79)
SYM_WDIV4 = ((1 << SYM_RP) - 1) >> 2
M128 = (1 << 128) - 1
# Kangaroos per tile of the symmetric variants whose CTAs must loop over tiles of the shape herd.  Both symmetric kernels run
# 2 CTAs per SM: the stream kernel is the 2-CTA instantiation, and a 128,7 tile keeps 105 KB of shared memory per CTA.
SYM_LOOPING = {"resident": 128 * 7, "stream-2": 128 * 2}


def sym_herd_arrays(n, rng):
    """kgo_create_herd_sym's draws, vectorised: d uniform in [0, 2^(SYM_RP-1)), minus width/4 for wild kangaroos (odd kIdx).
    -> (scalars (n,4) = d mod the group order, d128 (n,2) = d as signed 128-bit): what CreateHerdRaw takes in symmetric mode,
    where the device flips y into the lower half and negates d with it."""
    import numpy as np
    from kangaroo_b200 import random_herd_arrays
    sc, d128 = random_herd_arrays(n, SYM_RP - 1, SYM_WDIV4, rng)      # wild scalars already shifted; d128 = the plain draw
    w0, w1 = np.uint64(SYM_WDIV4 & (2**64 - 1)), np.uint64(SYM_WDIV4 >> 64)
    lo, hi = d128[:, 0].copy(), d128[:, 1].copy()
    wild = np.arange(n) % 2 == 1
    d128[:, 0] = np.where(wild, lo - w0, lo)
    d128[:, 1] = np.where(wild, hi - w1 - (lo < w0).astype(np.uint64), hi)
    return sc, d128


def s128_mod_n(a):
    """(m,2) signed 128-bit distances -> (m,4) limbs of d mod the group order (the oracle's form)."""
    from oracle import kgo
    return kgo.ints_to_array([(v - (1 << 128)) % kgo.N if v >> 127 else v for v in kgo.array_to_ints(a)])


def snapshot_raw(eng):
    """SnapshotRead into limb arrays, distances as the device stores them."""
    import numpy as np
    n = eng.nbKangaroo
    ax, ay, ad = np.empty((n, 4), dtype=np.uint64), np.empty((n, 4), dtype=np.uint64), np.empty((n, 2), dtype=np.uint64)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))
    assert eng._lib.kgx_snapshot_read(eng._h, p(ax), p(ay), p(ad)) == 0, eng._lib.kgx_last_error(eng._h)
    return ax, ay, ad


def device_sms():
    import kangaroo_b200
    buf = ctypes.create_string_buffer(256)
    assert kangaroo_b200.load_library().kgx_device_info(0, buf, 256) == 0
    return int(buf.value.split(b"|")[1])


@pytest.fixture(scope="module")
def sym_shape_herd(oracle):
    """The symmetric shape herd and, for its sample, the start state the device must make: the class representative of d*G
    (tame) or key + d*G (wild), with d negated wherever y was flipped."""
    import numpy as np
    from oracle import kgo
    from tests.golden_util import load_cases
    key = [c for c in load_cases() if c["range_power"] == 80][0]["key"]
    n = SHAPE_GRID[0] * SHAPE_GRID[1] * 128
    sc, d128 = sym_herd_arrays(n, np.random.Generator(np.random.PCG64(4343)))
    idx = shape_sample(n)
    for i in idx.tolist():
        d = kgo.from_limbs(d128[i])
        assert ((d - (1 << 128)) if d >> 127 else d) % kgo.N == kgo.from_limbs(sc[i])
    x, y, d, flipped = herd_start_state(oracle, key, sc, d128, idx, symmetric=True)
    assert 0 < flipped < len(idx)
    return dict(n=n, sc=sc, d128=d128, key=key, idx=idx, table=oracle.create_jump_table_sym(SYM_RP), x=x, y=y, d=d)


def herd_start_state(oracle, key, sc, d128, idx, symmetric=False):
    """The start state CreateHerdRaw(sc, d128, key) must give the sample idx: d*G (tame, even kIdx) or key + d*G (wild) with
    the distance d128 as stored; in symmetric mode the class representative, with d negated wherever y was flipped.
    -> x, y (m,4) and d (m,2) limb arrays, and how many kangaroos were flipped."""
    from oracle import kgo
    xs, ys, ds, flipped = [], [], [], 0
    for i in idx.tolist():
        pt = oracle.ec_mul_g(kgo.from_limbs(sc[i]))
        if i % 2:
            pt = oracle.ec_add(key, pt)
        d = kgo.from_limbs(d128[i])
        flip = symmetric and pt[1] > (kgo.P - 1) // 2
        xs.append(pt[0]); ys.append(kgo.P - pt[1] if flip else pt[1]); ds.append(-d & M128 if flip else d)
        flipped += flip
    return kgo.ints_to_array(xs), kgo.ints_to_array(ys), kgo.ints_to_array(ds, 2), flipped


def fresh_sym_kangaroo(oracle, key, kidx, stale, init, rule):
    """A new symmetric kangaroo for slot kidx, chosen where the rule allows it so that its first jump depends on SetKangaroo
    resetting the slot's state byte from `stale` to `init`.  lastjump bumps x mod 32 when it equals the previous jump, so the
    kangaroo has x = stale mod 32 (after a launch a lastjump byte is never 32); symclass takes the table half from the byte
    alone, so only a stale 1 can show."""
    from oracle import kgo
    from tests.test_gpu_field import LASTJUMP, SYMCLASS, jump_index_ref
    r = LASTJUMP if rule == "lastjump" else SYMCLASS
    for seed in range(1, 1024):
        oracle.rseed(seed)
        x, y, d = (kgo.from_limbs(a[0]) for a in oracle.create_herd_sym(1, SYM_RP, SYM_WDIV4, key, kidx % 2))
        if rule == "symclass" or jump_index_ref(x & 31, stale, r) != jump_index_ref(x & 31, init, r):
            return x, y, d
    raise AssertionError("no kangaroo with x = %d mod 32 in 1023 draws" % stale)


@pytest.mark.parametrize("n_run", [1, 63])
@pytest.mark.parametrize("rule,init", SYM_RULES, ids=[r for r, _ in SYM_RULES])
@pytest.mark.parametrize("env", SYM_VARIANTS, ids=SYM_VARIANT_IDS)
def test_symmetric_variant_shapes_match_oracle(env, rule, init, n_run, sym_shape_herd, oracle, monkeypatch):
    """The symmetric engine on 991,616 kangaroos made on the device: launch 1, a snapshot ordered after it, SetKangaroo of the
    last kangaroo (in the padded last tile of every geometry), launch 2, of n_run jumps each.  The per-kangaroo state byte only
    chooses the jump, so a wrongly indexed byte still makes a valid walk; the sample's oracle replay catches it.  Snapshot and end
    state (x, y, d mod n) and, launch by launch, the sample's DPs must equal the replay; no DP may come from a padding slot."""
    import numpy as np
    from kangaroo_b200 import GPUEngine
    from oracle import kgo
    for k in KGX_VARS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    h = sym_shape_herd
    n, idx, table = h["n"], h["idx"], h["table"]
    vid = variant_id(env)
    if vid in SYM_LOOPING:            # the tile loop this test exists for must still happen on this part
        assert -(-n // SYM_LOOPING[vid]) > 2 * device_sms(), vid
    mask = oracle.dp_mask(4 if n_run == 1 else 10)        # about 62 k DPs per launch either way
    max_found = 1 << 17
    eng = GPUEngine(*SHAPE_GRID, 0, max_found)
    assert eng.kernel == env["KGX_MODE"]
    eng.SetSymmetry(rule)
    eng.set_jumps_per_launch(n_run)
    eng.SetParams(mask, *table)
    eng.CreateHerdRaw(h["sc"], h["d128"], h["key"])
    ax, ay, ad = eng.GetKangaroosRaw()
    assert np.array_equal(ax[idx], h["x"]) and np.array_equal(ay[idx], h["y"]) and np.array_equal(ad[idx], h["d"])
    eng.callKernel()
    eng.SnapshotBegin()                                   # stream-ordered after launch 1
    launches = [eng.Launch(relaunch=False)]
    assert eng.lastFound <= max_found
    snap = snapshot_raw(eng)
    px, py, pd = h["x"].copy(), h["y"].copy(), s128_mod_n(h["d"])
    state = np.full(len(idx), init, dtype=np.uint8)
    want = [oracle.jump_sym(px, py, pd, state, table, n_run, mask, rule=rule)]
    assert np.array_equal(snap[0][idx], px) and np.array_equal(snap[1][idx], py) and np.array_equal(s128_mod_n(snap[2][idx]), pd)
    assert idx[-1] == n - 1
    nx, ny, nd = fresh_sym_kangaroo(oracle, h["key"], n - 1, int(state[-1]), init, rule)
    eng.SetKangaroo(n - 1, nx, ny, nd)
    px[-1], py[-1], pd[-1], state[-1] = kgo.to_limbs(nx), kgo.to_limbs(ny), kgo.to_limbs(nd), init
    eng.callKernel()
    launches.append(eng.Launch(relaunch=False))
    assert eng.lastFound <= max_found
    want.append(oracle.jump_sym(px, py, pd, state, table, n_run, mask, rule=rule))
    if vid in ("stream", "resident") and n_run == 63:     # device HashTable::Convert, once per kernel family and rule
        import torch
        from kangaroo_b200.dist import SlabView, decode_dp40
        raw = torch.as_tensor(SlabView(eng.convert_dps_device_ptr(), 4 + max_found * 40), device="cuda").cpu()
        cnt = int.from_bytes(bytes(raw[:4].numpy().tobytes()), "little")
        assert cnt == len(launches[1])
        ref = {}
        for it in launches[1]:
            hh, X, D = oracle.hash_convert(it.x, it.d, it.kIdx % 2)
            ref[(it.kIdx, X)] = (hh, D)
        for kidx, hh, x, dist, ktype in decode_dp40(raw[4:4 + cnt * 40]):
            assert ktype == kidx % 2
            D = (abs(dist) & ((1 << 126) - 1)) | ((1 << 127) if dist < 0 else 0) | (ktype << 126)
            assert (hh, D) == ref[(kidx, x)]
    ax, ay, ad = eng.GetKangaroosRaw()
    eng.close()

    assert np.array_equal(ax[idx], px) and np.array_equal(ay[idx], py) and np.array_equal(s128_mod_n(ad[idx]), pd)
    assert max(kgo.array_to_ints(ay[idx])) <= (kgo.P - 1) // 2
    negative = int((ad[idx, 1] >> np.uint64(63)).sum())
    assert 0 < negative < len(idx)
    in_sample = set(idx.tolist())
    for launch, (found, exp_dps) in enumerate(zip(launches, want)):
        assert len(found) > 1000 and max(it.kIdx for it in found) < n
        got = sorted((it.x, it.d, it.kIdx) for it in found if it.kIdx in in_sample)
        exp = sorted((x, d, int(idx[k])) for x, d, k, j in exp_dps)
        assert got == exp and len(exp) > 50, launch


LONG_WALK = (64,) * 100
# The same 6400 jumps for the stream kernel in launches that end its jump-log windows at every kind of place: after one run,
# one short of and exactly at a full window, one run past it, around two windows, and 5823 = 90 x 64 + 63 (91 folds).
LONG_WALK_IRREGULAR = (1, 63, 64, 65, 127, 128, 129, 5823)


def long_walks_agree(monkeypatch, rule=None, sym_table=None, stream_runs=LONG_WALK):
    """1,048,576 kangaroos x 6400 jumps on every kernel that runs `rule` (None: the non-symmetric engine; else the symmetric
    engine with that jump rule and sym_table): bit-identical end states and DP multisets.  The stream kernel takes its jumps
    in launches of stream_runs jumps, the tile kernels in LONG_WALK's 100 launches of 64."""
    import numpy as np
    from kangaroo_b200 import GPUEngine, random_herd_arrays
    from tests.golden_util import load_cases
    assert sum(stream_runs) == sum(LONG_WALK)
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    rng = np.random.Generator(np.random.PCG64(2024))
    if rule is None:
        sc, d128 = random_herd_arrays(64 * 128 * 128, 80, case["width_div2"], rng)
        table, modes = case["table"], ("stream", "resident", "tmem")
    else:
        sc, d128 = sym_herd_arrays(64 * 128 * 128, rng)
        table, modes = sym_table, ("stream", "resident")     # the cluster kernel has no symmetric instantiation
    results = {}
    for mode in modes:
        monkeypatch.setenv("KGX_MODE", mode)
        eng = GPUEngine(64, 128, 0, 1 << 17)
        if rule is not None:
            eng.SetSymmetry(rule)
        eng.SetParams(0xFFFFF00000000000, *table)          # dp = 20
        eng.SetWildOffset(case["width_div2"])               # not applied in symmetric mode
        eng.CreateHerdRaw(sc, d128, case["key"])
        runs = stream_runs if mode == "stream" else LONG_WALK
        dps = []
        eng.set_jumps_per_launch(runs[0])
        eng.callKernel()
        for nxt in runs[1:] + (None,):
            if nxt:
                eng.set_jumps_per_launch(nxt)               # read when Launch() starts the next launch
            dps += [(it.x, it.d, it.kIdx) for it in eng.Launch(relaunch=nxt is not None)]
        ax, ay, ad = eng.GetKangaroosRaw()
        results[mode] = (ax, ay, ad, sorted(dps))
        eng.close()
    a = results["stream"]
    for other in modes[1:]:
        b = results[other]
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), other
        assert a[3] == b[3] and len(a[3]) > 3000, other


def test_stream_and_resident_agree_over_a_long_walk(monkeypatch):
    """Cross-validation at a scale the CPU oracle cannot reach: 1,048,576 kangaroos x 100 launches (6400 jumps each) on the
    three kernels (different memory layout, different batch-inverse topology; the tile kernels loop over several tiles per
    CTA here) must end in bit-identical states and produce the same DP multiset.  The per-kangaroo jump is one function
    shared by all three, so the independent check of the arithmetic is the CPU oracle, which every variant is compared
    against at smaller sizes."""
    long_walks_agree(monkeypatch)


@pytest.mark.parametrize("rule", ["lastjump", "symclass"])
def test_stream_and_resident_agree_over_a_long_symmetric_walk(rule, oracle, monkeypatch):
    """The same cross-validation in symmetric mode, stream against resident kernel: their per-kangaroo state bytes carry the
    jump rule across all 100 launches, and the resident CTAs loop over tiles."""
    long_walks_agree(monkeypatch, rule, oracle.create_jump_table_sym(SYM_RP))


def test_stream_walk_in_irregular_launches_agrees_with_the_tile_kernels(monkeypatch):
    """The long walk with the stream kernel's 6400 jumps in launches of 1 to 5823 jumps: a fold after a short window, several
    folds inside one launch and DPs rebuilt after them must leave the same states and DPs as the tile kernels, which keep no
    jump log."""
    long_walks_agree(monkeypatch, stream_runs=LONG_WALK_IRREGULAR)


@pytest.mark.parametrize("rule", ["lastjump", "symclass"])
def test_stream_symmetric_walk_in_irregular_launches_agrees_with_the_resident_kernel(rule, oracle, monkeypatch):
    """The same in symmetric mode, where the folds inside a launch also replay the class switches logged in bit 5."""
    long_walks_agree(monkeypatch, rule, oracle.create_jump_table_sym(SYM_RP), LONG_WALK_IRREGULAR)


def test_cluster_kernel_odd_jump_count_over_several_tiles_per_cluster(monkeypatch):
    """The cluster tile kernel alternates its exchange slot on every tile inverse.  With an odd number of jumps per launch and
    more tiles than clusters (262,144 kangaroos = 147 tiles of 1792 on at most one cluster per SM pair), consecutive tiles of a
    cluster meet at an odd/even slot boundary; the result must still equal the stream kernel's bit for bit."""
    import numpy as np
    from kangaroo_b200 import GPUEngine, random_herd_arrays
    from tests.golden_util import load_cases
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    sc, d128 = random_herd_arrays(16 * 128 * 128, 80, case["width_div2"], np.random.Generator(np.random.PCG64(7)))
    results = {}
    for mode in ("stream", "tmem"):
        monkeypatch.setenv("KGX_MODE", mode)
        eng = GPUEngine(16, 128, 0, 1 << 17)
        eng.set_jumps_per_launch(63)
        eng.SetParams(0xFFF0000000000000, *case["table"])          # dp = 12
        eng.SetWildOffset(case["width_div2"])
        eng.CreateHerdRaw(sc, d128, case["key"])
        dps = []
        eng.callKernel()
        for _ in range(2):
            dps += [(it.x, it.d, it.kIdx) for it in eng.Launch()]
        dps += [(it.x, it.d, it.kIdx) for it in eng.Launch(relaunch=False)]
        results[mode] = eng.GetKangaroosRaw() + (sorted(dps),)
        eng.close()
    a, b = results["stream"], results["tmem"]
    assert all(np.array_equal(u, v) for u, v in zip(a[:3], b[:3]))
    assert a[3] == b[3] and len(a[3]) > 1000
