"""CPU: --dp-table-entries host -- its options and refusals in the solver and the server, the default-capacity rule at chosen
free-memory, MemAvailable and local-rank values, and the new table calls declared, exported and typed."""
import os
import re

import pytest

import kangaroo_b200
from kangaroo_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "tests", "golden", "in56.txt")
GiB = 1 << 30


def test_the_new_calls_are_declared_exported_and_typed():
    hdr = open(os.path.join(ROOT, "include", "kgx.h")).read()
    lib = kangaroo_b200.load_library()
    assert re.search(r"#define KGX_DPT_HOST_ENTRIES\s+1\b", hdr)
    for name in ("kgx_dptable_create_ex", "kgx_dptable_bytes_for_ex", "kgx_dptable_host_bytes"):
        assert name + "(" in hdr and name in _lib.EXPORTED_SYMBOLS, name
        assert getattr(lib, name).argtypes is not None, name


def test_bytes_for_ex_moves_the_entries_to_the_host():
    import ctypes
    lib = kangaroo_b200.load_library()
    for cap in (1000, 1 << 21, 1 << 26, (1 << 32) - 2):
        host = ctypes.c_uint64(7)
        dev = lib.kgx_dptable_bytes_for_ex(cap, 1, ctypes.byref(host))
        assert host.value == 32 * cap and dev == lib.kgx_dptable_bytes_for(cap) - 32 * cap
        assert lib.kgx_dptable_bytes_for_ex(cap, 0, ctypes.byref(host)) == lib.kgx_dptable_bytes_for(cap) and host.value == 0
    a, b = lib.kgx_dptable_bytes_for_ex(1 << 26, 1, None), lib.kgx_dptable_bytes_for_ex(1 << 27, 1, None)
    assert b - a == 16 * (1 << 26)


@pytest.mark.skipif(_lib.load_library().kgx_device_count() > 0, reason="a CUDA device is present")
def test_create_ex_fails_loudly_without_a_device():
    lib = kangaroo_b200.load_library()
    assert not lib.kgx_dptable_create_ex(0, 1000, 0, 1 << 18, 1)
    assert b"no CUDA device" in lib.kgx_dptable_last_error(None)
    assert not lib.kgx_dptable_create_ex(0, 1000, 0, 1 << 18, 2)
    assert b"unknown flags" in lib.kgx_dptable_last_error(None)


def test_the_host_limit_rule():
    from kangaroo_b200 import solver as S
    assert S.host_entries_limit(S.HOST_ENTRIES_MARGIN + 32 * 1000, 1) == 1000
    assert S.host_entries_limit(S.HOST_ENTRIES_MARGIN + 32 * 1000, 4) == 250
    assert S.host_entries_limit(S.HOST_ENTRIES_MARGIN - 1, 1) == 0
    assert S.host_entries_limit(1000 * GiB, 8) == (1000 * GiB - S.HOST_ENTRIES_MARGIN) // 8 // 32


@pytest.mark.parametrize("free, avail, tables, bound", [
    (80 * GiB, 2048 * GiB, 1, "2^32-2"),      # a large host: the slot format's limit
    (20 * GiB, 2048 * GiB, 1, "device"),      # a small GPU: the device rule at 16 bytes per entry
    (80 * GiB, 64 * GiB, 1, "host"),          # little host RAM
    (80 * GiB, 512 * GiB, 8, "host"),         # eight ranks share it
])
def test_the_default_capacity_is_the_smallest_of_three_limits(free, avail, tables, bound):
    from kangaroo_b200 import solver as S
    from kangaroo_b200.ingest import DeviceDPTable
    limit = S.host_entries_limit(avail, tables)
    cap = S.default_table_capacity(free, entries="host", host_limit=limit)
    dev_rule = S.default_table_capacity(free, entries="host")
    assert cap == min(dev_rule, (1 << 32) - 2, limit)
    assert DeviceDPTable.bytes_for(cap, "host") <= free - S.DP_TABLE_MARGIN and 32 * cap <= avail - S.HOST_ENTRIES_MARGIN
    want = {"2^32-2": (1 << 32) - 2, "device": dev_rule, "host": limit}[bound]
    assert cap == want
    if bound == "device":
        assert DeviceDPTable.bytes_for(cap * 65 // 64, "host") > free - S.DP_TABLE_MARGIN
        assert cap > 2.5 * S.default_table_capacity(free)   # the same GPU holds about 3x the entries of the device layout
    assert S.default_table_capacity(free) == S.default_table_capacity(free, entries="device", host_limit=1)   # unchanged


def test_tables_on_the_node(monkeypatch):
    from kangaroo_b200 import solver as S
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "4")
    assert S.tables_on_node("sharded") == 4 and S.tables_on_node("device") == 1
    monkeypatch.delenv("LOCAL_WORLD_SIZE")
    assert S.tables_on_node("sharded") == 1


@pytest.mark.parametrize("args, msg", [
    (["--dp-table-entries", "host"], "--dp-table-entries needs --dp-table device or sharded"),
    (["--dp-table", "host", "--dp-table-entries", "device"], "--dp-table-entries needs --dp-table device or sharded"),
    (["--dp-table", "device", "--dp-table-entries", "disk"], "invalid choice"),
    (["--dp-table", "device", "--dp-table-entries", "host", "--dp-table-capacity", str((1 << 32) - 2)], "more than the host limit"),
])
def test_solver_refusals(args, msg, capsys, monkeypatch):
    from kangaroo_b200 import solver as S
    monkeypatch.setattr(S, "mem_available", lambda: 64 * GiB)
    with pytest.raises(SystemExit) as e:
        S.main([CFG] + args)
    assert e.value.code == 2
    assert msg in capsys.readouterr().err


def test_solver_refusal_names_both_numbers(capsys, monkeypatch):
    from kangaroo_b200 import solver as S
    monkeypatch.setattr(S, "mem_available", lambda: 40 * GiB)
    monkeypatch.setenv("WORLD_SIZE", "1")
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "2")
    limit = S.host_entries_limit(40 * GiB, 2)
    with pytest.raises(SystemExit):
        S.parse_args([CFG, "--dp-table", "sharded", "--dp-table-entries", "host", "--dp-table-capacity", str(limit + 1)])
    err = capsys.readouterr().err
    assert str(limit + 1) in err and str(limit) in err and "shared by 2 table(s)" in err
    a = S.parse_args([CFG, "--dp-table", "sharded", "--dp-table-entries", "host", "--dp-table-capacity", str(limit)])[0]
    assert a.dp_table_entries == "host"
    assert S.parse_args([CFG, "--dp-table", "device"])[0].dp_table_entries == "device"


def test_server_options(capsys, monkeypatch):
    from kangaroo_b200 import server
    from kangaroo_b200 import solver as S
    monkeypatch.setattr(S, "mem_available", lambda: 40 * GiB)
    assert server.parse_args([CFG, "--dp", "8"])[0].dp_table_entries == "device"
    assert server.parse_args([CFG, "--dp", "8", "--dp-table-entries", "host"])[0].dp_table_entries == "host"
    one, three = S.host_entries_limit(40 * GiB, 1), S.host_entries_limit(40 * GiB, 3)
    server.parse_args([CFG, "--dp", "8", "--dp-table-entries", "host", "--dp-table-capacity", str(one)])
    for extra, cap in (([], one + 1), (["--devices", "0,0,0"], three + 1)):
        with pytest.raises(SystemExit) as e:
            server.parse_args([CFG, "--dp", "8", "--dp-table-entries", "host", "--dp-table-capacity", str(cap)] + extra)
        assert e.value.code == 2
        err = capsys.readouterr().err
        assert "more than the host limit of %d entries" % (cap - 1) in err
    server.parse_args([CFG, "--dp", "8", "--dp-table-entries", "device", "--dp-table-capacity", str(one + 1)])
    with pytest.raises(SystemExit):
        server.parse_args([CFG, "--dp", "8", "--dp-table-entries", "pinned"])
