"""Sweep the compiled tile geometries (KGX_CFG=T,K) at the BASELINE grid and report MJump/s per launch."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kangaroo_b200 import GPUEngine, NB_RUN  # noqa: E402
from tests.golden_util import load_cases, arrays  # noqa: E402


def main():
    cfgs = sys.argv[1:] or ["128,7", "128,5", "128,4", "96,6", "64,7", "64,6", "64,5", "64,4", "256,3", "32,8", "32,12"]
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    sx, sy, sd = arrays(case["start"])
    gx, gy = (int(v) for v in os.environ.get('KGX_SWEEP_GRID', '264,128').split(','))
    n = gx * gy * 128
    idx = np.arange(n) % sx.shape[0]
    ax, ay = sx[idx], sy[idx]
    ad = np.ascontiguousarray(sd[idx, :2])
    out = {}
    for cfg in cfgs:
        os.environ["KGX_CFG"] = cfg
        eng = GPUEngine(gx, gy, 0, 1 << 17)
        eng.SetParams(0xFFFF000000000000, *case["table"])
        eng.SetKangaroosRaw(ax, ay, ad)
        eng.callKernel()
        times = []
        for i in range(5):
            eng.Launch()
            times.append(eng.last_launch_ms())
        eng.sync()
        ms = min(times[1:])
        out[cfg] = dict(ms=ms, mjump_s=n * NB_RUN / ms / 1e3)
        extra = ""
        if os.environ.get("KGX_PROF"):
            import ctypes
            pr = (ctypes.c_uint64 * 4)()
            if eng._lib.kgx_debug_prof(eng._h, pr) == 0 and pr[3]:
                extra = "  per tile-step cycles: serial %.0f (modinv %.0f) parallel %.0f" % (pr[0] / pr[3], pr[1] / pr[3], pr[2] / pr[3])
                out[cfg]["prof"] = [int(v) for v in pr]
        print("KGX_CFG=%-7s %8.3f ms/launch  %8.1f MJump/s%s" % (cfg, ms, out[cfg]["mjump_s"], extra), flush=True)
        eng.close()
    os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "results", "sweep.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
