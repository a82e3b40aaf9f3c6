"""Raw device microbenchmarks (BASELINE config 5 inputs): IMAD.WIDE issue rate, fe_mul / fe_sqr / inverse
throughput, and jump-kernel launch time on a synthetic herd.  Writes results/microbench.json."""
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kangaroo_b200  # noqa: E402
from kangaroo_b200 import GPUEngine, NB_RUN  # noqa: E402


def raw(kind, iters):
    lib = kangaroo_b200.load_library()
    ms, ops = ctypes.c_float(0), ctypes.c_double(0)
    assert lib.kgx_bench_raw(0, kind, iters, ctypes.byref(ms), ctypes.byref(ops)) == 0
    return ms.value, ops.value


def main():
    out = {}
    for name, kind, iters in (("imad_wide", 0, 20000), ("fe_mul", 1, 2000), ("fe_sqr", 2, 2000), ("fe_inv", 3, 20)):
        best = None
        for _ in range(3):
            ms, ops = raw(kind, iters)
            r = ops / (ms * 1e-3)
            best = r if best is None or r > best else best
        out[name + "_per_s"] = best
        print(name, "%.3e /s" % best, flush=True)
    # jump kernel on a synthetic herd built on the device (kgx_create_herd); jump table from the reference-generated fixture
    from kangaroo_b200 import random_herd_arrays
    from tests.golden_util import load_cases
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    for grid in ((264, 128), (66, 128), (16, 128)):
        n = grid[0] * grid[1] * 128
        eng = GPUEngine(grid[0], grid[1], 0, 1 << 20)
        eng.SetParams(0xFFFF000000000000, *case["table"])
        eng.SetWildOffset(case["width_div2"])
        sc, d128 = random_herd_arrays(n, 80, case["width_div2"], np.random.Generator(np.random.PCG64(5)))
        eng.CreateHerdRaw(sc, d128, case["key"])
        eng.callKernel()
        times = []
        for i in range(6):
            eng.Launch()
            times.append(eng.last_launch_ms())
        eng.sync()
        ms = min(times[1:])
        out["jump_%dx%d" % grid] = {"kangaroos": n, "ms_per_launch": ms, "mjump_s": n * NB_RUN / ms / 1e3, "all_ms": times}
        print(grid, out["jump_%dx%d" % grid], flush=True)
        eng.close()
    os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "results", "microbench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
