"""BASELINE config 5: batch-inverse microbench -- 2^20 kangaroos x 1024 jumps (16 launches of NB_RUN=64), dpMask = all ones
(never fires), Montgomery group sizes 32 / 64 / 128 per thread (stream kernel: one inverse per thread, or one
warp-wide shuffle-butterfly inverse per 32 x G kangaroos), the tile-wide groups of the resident kernel and of the cluster tile kernel.  Reports MJump/s, ModMult/s (= 6 x MJump/s, SURVEY 8d) and the fraction of the measured wide-IMAD
roofline (416 IMAD.WIDE per jump)."""
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kangaroo_b200  # noqa: E402
from kangaroo_b200 import GPUEngine, NB_RUN, random_herd_arrays  # noqa: E402
from tests.golden_util import load_cases  # noqa: E402


def main():
    lib = kangaroo_b200.load_library()
    peak = 0.0
    for kind, iters, scale in ((0, 20000, 1.0), (1, 2000, 73.0)):          # accumulate probe; 73 x the fe_mul-chain rate (as bench.py)
        for _ in range(2):
            ms, ops = ctypes.c_float(0), ctypes.c_double(0)
            lib.kgx_bench_raw(0, kind, iters, ctypes.byref(ms), ctypes.byref(ops))
            peak = max(peak, scale * ops.value / (ms.value * 1e-3))
    case = [c for c in load_cases() if c["range_power"] == 64][0]
    n = 1 << 20
    sc, d128 = random_herd_arrays(n, 64, case["width_div2"], np.random.Generator(np.random.PCG64(1)))
    variants = []
    for inv in ("thread", "warp"):
        for g in (32, 64, 128):
            grp = g if inv == "thread" else 32 * g
            variants.append(("stream G=%d, %s inverse (group %d)" % (g, inv, grp), {"KGX_MODE": "stream", "KGX_STREAM_G": str(g), "KGX_STREAM_INV": inv}))
    variants += [("stream auto (G=28, thread inverse)", {"KGX_MODE": "stream"}),
                 ("resident tile 128x7=896", {"KGX_MODE": "resident", "KGX_CFG": "128,7"}),
                 ("resident tile 64x7=448", {"KGX_MODE": "resident", "KGX_CFG": "64,7"}),
                 ("cluster tile 2x(128x7)=1792", {"KGX_MODE": "tmem"})]
    lines = ["batch-inverse microbench (BASELINE config 5): 2^20 kangaroos x 1024 jumps, rangePower 64 table, dp = 64 (never fires)",
             "measured wide-IMAD peak %.3e /s ; roofline = 416 IMAD.WIDE per jump" % peak, "",
             "%-44s %10s %12s %14s %9s" % ("variant (Montgomery group)", "ms/1024j", "MJump/s", "ModMult/s", "roofline")]
    for name, env in variants:
        for k in ("KGX_MODE", "KGX_STREAM_G", "KGX_CFG", "KGX_STREAM_INV"):
            os.environ.pop(k, None)
        os.environ.update(env)
        eng = GPUEngine(64, 128, 0, 1 << 16)
        eng.SetParams(0xFFFFFFFFFFFFFFFF, *case["table"])
        eng.SetWildOffset(case["width_div2"])
        eng.CreateHerdRaw(sc, d128, case["key"])
        eng.callKernel()
        eng.Launch()                                   # warm-up launch
        tot = 0.0
        for _ in range(16):
            eng.Launch()
            tot += eng.last_launch_ms()
        eng.sync(); eng.close()
        mj = n * 1024 / tot / 1e3
        lines.append("%-44s %10.2f %12.1f %14.3e %8.1f%%" % (name, tot, mj, mj * 6e6, 100 * mj * 1e6 * 416 / peak))
        print(lines[-1], flush=True)
    os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
    open(os.path.join(ROOT, "results", "batchinv_microbench.txt"), "w").write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
