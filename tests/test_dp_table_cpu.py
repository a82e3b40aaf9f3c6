"""CPU: the device DP table's boundary -- its entry points are exported and typed, it fails loudly without a GPU (no host
fallback), and the solver refuses --dp-table-capacity without --dp-table device or with a non-positive capacity."""
import os

import pytest

import kangaroo_b200
from kangaroo_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DPTABLE_SYMBOLS = ["kgx_dptable_create", "kgx_dptable_destroy", "kgx_dptable_last_error", "kgx_dptable_count", "kgx_dptable_capacity",
                   "kgx_dptable_memory_bytes", "kgx_dptable_bytes_for", "kgx_dptable_reserve", "kgx_dptable_add", "kgx_dptable_save_work",
                   "kgx_dptable_load_work"]


def test_the_table_entry_points_are_declared_exported_and_typed():
    hdr = open(os.path.join(ROOT, "include", "kgx.h")).read()
    lib = kangaroo_b200.load_library()
    for name in DPTABLE_SYMBOLS:
        assert name + "(" in hdr, name
        assert name in _lib.EXPORTED_SYMBOLS, name
        assert getattr(lib, name).argtypes is not None or name == "kgx_dptable_create", name


def test_bytes_for_is_48_per_entry_plus_fixed_scratch():
    lib = kangaroo_b200.load_library()
    a, b = lib.kgx_dptable_bytes_for(1 << 26), lib.kgx_dptable_bytes_for(1 << 27)
    assert b - a == 48 * (1 << 26)
    assert a < 48 * (1 << 26) + (256 << 20)


@pytest.mark.skipif(_lib.load_library().kgx_device_count() > 0, reason="a CUDA device is present")
def test_create_fails_loudly_without_a_device():
    from kangaroo_b200.ingest import DeviceDPTable
    lib = kangaroo_b200.load_library()
    assert not lib.kgx_dptable_create(0, 1000)
    assert b"no CUDA device" in lib.kgx_dptable_last_error(None)
    with pytest.raises(RuntimeError, match="no CUDA device"):
        DeviceDPTable(1000)


@pytest.mark.parametrize("args, msg", [
    (["--dp-table-capacity", "1000"], "--dp-table-capacity needs --dp-table device"),
    (["--dp-table", "host", "--dp-table-capacity", "1000"], "--dp-table-capacity needs --dp-table device"),
    (["--dp-table", "device", "--dp-table-capacity", "0"], "--dp-table-capacity must be 1 .. 2^32-2 entries"),
    (["--dp-table", "device", "--dp-table-capacity", "-5"], "--dp-table-capacity must be 1 .. 2^32-2 entries"),
    (["--dp-table", "device", "--dp-table-capacity", str(1 << 32)], "--dp-table-capacity must be 1 .. 2^32-2 entries"),
    (["--dp-table", "disk"], "invalid choice"),
])
def test_solver_refuses_bad_table_arguments(args, msg, capsys):
    from kangaroo_b200 import solver
    with pytest.raises(SystemExit) as e:
        solver.main([os.path.join(ROOT, "tests", "golden", "in56.txt")] + args)
    assert e.value.code == 2
    assert msg in capsys.readouterr().err


def test_default_capacity_fits_the_free_memory_less_the_margin():
    from kangaroo_b200 import solver
    from kangaroo_b200.ingest import DeviceDPTable
    free = 70 << 30
    cap = solver.default_table_capacity(free)
    assert DeviceDPTable.bytes_for(cap) <= free - solver.DP_TABLE_MARGIN
    assert DeviceDPTable.bytes_for(cap * 65 // 64) > free - solver.DP_TABLE_MARGIN
    assert solver.default_table_capacity(solver.DP_TABLE_MARGIN) == 0
