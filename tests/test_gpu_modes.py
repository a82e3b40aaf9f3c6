"""-m gpu: every compiled kernel variant stays bit-exact: the smoke check (1024 kangaroos x 64 jumps vs the oracle, state and
DP multiset) is run in a subprocess per KGX_MODE / geometry, because the variant is fixed at kgx_create from the environment."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

VARIANTS = [
    {"KGX_MODE": "stream"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "64"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "256"},
    {"KGX_MODE": "resident"},
    {"KGX_MODE": "resident", "KGX_CFG": "64,5"},
    {"KGX_MODE": "resident", "KGX_CFG": "256,3"},
    {"KGX_MODE": "resident", "KGX_CFG": "32,12"},
    {"KGX_MODE": "tmem"},
]


@pytest.mark.parametrize("env", VARIANTS, ids=["-".join(v.values()) for v in VARIANTS])
def test_variant_bit_exact(env):
    e = dict(os.environ); e.update(env)
    p = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], cwd=ROOT, env=e,
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "smoke ok" in p.stdout, (p.stdout + p.stderr)[-2000:]


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
