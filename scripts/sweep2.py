"""Sweep: MJump/s of engine variants selected through the environment, several herd sizes in one process.
  python scripts/sweep2.py "label|ENV=VAL,ENV=VAL|gx,gy" ...      -> results/sweep2.json + one line per variant
Herd = replicated rows of the reference-generated in80 fixture (valid curve points; throughput does not depend on values)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kangaroo_b200 import GPUEngine, NB_RUN  # noqa: E402
from tests.golden_util import load_cases, arrays  # noqa: E402

KEYS = ("KGX_MODE", "KGX_CFG", "KGX_STREAM_G", "KGX_STREAM_CTAS", "KGX_STREAM_INV", "KGX_STREAM_PF")


def main():
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    sx, sy, sd = arrays(case["start"])
    out = {}
    for spec in sys.argv[1:]:
        label, envs, grid = spec.split("|")
        for k in KEYS:
            os.environ.pop(k, None)
        sym = None
        for kv in filter(None, envs.split(",")):
            k, v = kv.split("=")
            if k == "SYM":                       # symmetric engine mode: SYM=symclass | SYM=lastjump
                sym = v
                continue
            os.environ[k] = v.replace(";", ",")
        gx, gy = (int(v) for v in grid.split(","))
        n = gx * gy * 128
        idx = np.arange(n) % sx.shape[0]
        try:
            eng = GPUEngine(gx, gy, 0, 1 << 17)
        except RuntimeError as e:
            print("%-44s FAILED %s" % (label, e), flush=True)
            continue
        if sym:
            eng.SetSymmetry(sym)
        eng.SetParams(0xFFFF000000000000, *case["table"])
        eng.SetKangaroosRaw(sx[idx], sy[idx], np.ascontiguousarray(sd[idx, :2]))
        eng.callKernel()
        times = []
        for i in range(6):
            eng.Launch()
            times.append(eng.last_launch_ms())
        eng.sync()
        ms = min(times[1:])
        out[label] = dict(ms=ms, mjump_s=n * NB_RUN / ms / 1e3, kangaroos=n, kernel=eng.kernel, env=envs)
        print("%-44s %9d kangaroos  %-8s %8.3f ms/launch  %8.1f MJump/s" % (label, n, eng.kernel, ms, out[label]["mjump_s"]), flush=True)
        eng.close()
    os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "results", "sweep2.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
