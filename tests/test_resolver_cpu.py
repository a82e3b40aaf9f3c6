"""CPU checks of the solver without build/libkgx_ingest.so: importing it and parsing a --dp-table device or sharded command
line load no reference code, and --dp-table host without the library is refused with a message that names the device
tables.  KGX_INGEST_LIB points at a path that does not exist, as in a checkout built without the reference sources."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IN56 = os.path.join(ROOT, "tests", "golden", "in56.txt")
MISSING = os.path.join(ROOT, "build", "no_such_libkgx_ingest.so")

PROBE = r"""
import sys
from kangaroo_b200 import ingest, solver
a = solver.parse_args(sys.argv[1:])[0]
maps = open("/proc/self/maps").read()
print("table=%s ingest_loaded=%s mapped=%s" % (a.dp_table, ingest._lib is not None, "libkgx_ingest" in maps))
"""


def probe(args, missing=True):
    env = dict(os.environ)
    if missing:
        env["KGX_INGEST_LIB"] = MISSING
    return subprocess.run([sys.executable, "-c", PROBE] + args, capture_output=True, text=True, cwd=ROOT, env=env, timeout=300)


def test_device_tables_load_no_ingest_library():
    for table in ("device", "sharded"):
        for missing in (True, False):                            # with the library present it is not loaded either
            p = probe([IN56, "--dp-table", table], missing)
            assert p.returncode == 0, p.stderr
            assert "table=%s ingest_loaded=False mapped=False" % table in p.stdout, p.stdout + p.stderr


def test_host_table_without_the_library_is_a_usage_error():
    p = probe([IN56, "--dp-table", "host"])
    assert p.returncode == 2, p.stdout + p.stderr
    assert MISSING in p.stderr and "--dp-table device" in p.stderr and "--dp-table sharded" in p.stderr, p.stderr
    p = probe([IN56])                                            # host is the default table
    assert p.returncode == 2 and "--dp-table device" in p.stderr, p.stderr


def test_an_unloadable_library_is_reported_like_a_missing_one(tmp_path):
    bad = tmp_path / "libkgx_ingest.so"
    bad.write_bytes(b"not a shared object")
    env = dict(os.environ, KGX_INGEST_LIB=str(bad))
    p = subprocess.run([sys.executable, "-c", PROBE, IN56, "--dp-table", "host"], capture_output=True, text=True, cwd=ROOT, env=env,
                       timeout=300)
    assert p.returncode == 2 and "cannot be loaded" in p.stderr and "--dp-table sharded" in p.stderr, p.stderr
