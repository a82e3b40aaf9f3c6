"""-m gpu: every compiled kernel variant stays bit-exact.  VARIANTS names each instantiation kgx_engine.cu compiles (a CPU test,
tests/test_abi_cpu.py, fails when one is added without an entry here).  Each variant runs the smoke check (1024 kangaroos x 64
jumps vs the oracle, state and DP multiset) in a subprocess, and an in-process shape test on a herd that pads the last tile of
every geometry, loops over tiles, and runs 1 or 63 jumps per launch; kgx_create reads the KGX_* environment at every create."""
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


@pytest.mark.parametrize("env", VARIANTS, ids=VARIANT_IDS)
def test_variant_bit_exact(env):
    e = {k: v for k, v in os.environ.items() if k not in KGX_VARS}; e.update(env)
    p = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], cwd=ROOT, env=e,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "smoke ok" in p.stdout, (p.stdout + p.stderr)[-2000:]


SHAPE_GRID = (61, 127)            # 61 x 127 x 128 = 991,616 kangaroos: a multiple of no compiled tile
SAMPLE = 2048


@pytest.fixture(scope="module")
def shape_herd():
    import numpy as np
    from kangaroo_b200 import random_herd_arrays
    from tests.golden_util import load_cases
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    n = SHAPE_GRID[0] * SHAPE_GRID[1] * 128
    sc, d128 = random_herd_arrays(n, 80, case["width_div2"], np.random.Generator(np.random.PCG64(4242)))
    # a strided sample plus the last 128 kangaroos, which sit in the padded last tile of every geometry
    idx = np.unique(np.concatenate([np.arange(0, n, n // SAMPLE), np.arange(n - 128, n)]))
    return case, sc, d128, idx


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


def test_stream_and_resident_agree_over_a_long_walk(monkeypatch):
    """Cross-validation at a scale the CPU oracle cannot reach: 1,048,576 kangaroos x 100 launches (6400 jumps each) on the
    three independent kernel implementations (different memory layout, different batch-inverse topology; the tile kernels loop
    over several tiles per CTA here) must end in bit-identical states and produce the same DP multiset."""
    import numpy as np
    from kangaroo_b200 import GPUEngine, random_herd_arrays
    from tests.golden_util import load_cases
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    sc, d128 = random_herd_arrays(64 * 128 * 128, 80, case["width_div2"], np.random.Generator(np.random.PCG64(2024)))
    results = {}
    for mode in ("stream", "resident", "tmem"):
        monkeypatch.setenv("KGX_MODE", mode)
        eng = GPUEngine(64, 128, 0, 1 << 17)
        eng.SetParams(0xFFFFF00000000000, *case["table"])          # dp = 20
        eng.SetWildOffset(case["width_div2"])
        eng.CreateHerdRaw(sc, d128, case["key"])
        dps = []
        eng.callKernel()
        for _ in range(99):
            dps += [(it.x, it.d, it.kIdx) for it in eng.Launch()]
        dps += [(it.x, it.d, it.kIdx) for it in eng.Launch(relaunch=False)]
        ax, ay, ad = eng.GetKangaroosRaw()
        results[mode] = (ax, ay, ad, sorted(dps))
        eng.close()
    a = results["stream"]
    for other in ("resident", "tmem"):
        b = results[other]
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), other
        assert a[3] == b[3] and len(a[3]) > 3000, other


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
