"""-m gpu: the stand-alone driver (kangaroo_b200/solver.py) end to end on one GPU: device herd creation, jump engine,
DP table, collision -> private key.  Known answers: in56 (README.md:146-147) and a 2^56 window around puzzle #110
(puzzle32.txt:6-9), the BASELINE config-4 key."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the solver's rank-0 table is the reference's HashTable (build/libkgx_ingest.so, built only with the reference sources)
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "build", "libkgx_ingest.so")),
                                                  reason="build/libkgx_ingest.so not built (needs the reference sources at build time)")]


def solve(cfg, extra):
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.solver", os.path.join(ROOT, "tests", "golden", cfg)] + extra,
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    return p.stdout + p.stderr


def test_solver_in56():
    out = solve("in56.txt", ["--dp", "8", "--grid", "32,128", "--seed", "7"])
    assert "Priv: 0x3447F65ABC9F46F736A95F87B044829C8A0129D56782D635CD612C0F05F3DA03" in out, out[-2000:]


def test_solver_puzzle110_window():
    out = solve("puzzle110_window56.txt", ["--dp", "8", "--grid", "32,128", "--seed", "11"])
    assert "Priv: 0x35C0D7234DF7DEB0F20CF7062444" in out, out[-2000:]
