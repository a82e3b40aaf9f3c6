"""-m gpu: error behaviour of the C ABI (include/kgx.h): return codes + kgx_last_error, never a crash, never a fallback."""
import ctypes

import numpy as np
import pytest

import kangaroo_b200
from kangaroo_b200 import GPUEngine
from kangaroo_b200._lib import Item

pytestmark = pytest.mark.gpu


def test_bad_create_arguments():
    lib = kangaroo_b200.load_library()
    assert not lib.kgx_create(0, 0, 128, 1024) and b"bad arguments" in lib.kgx_last_error(None)
    assert not lib.kgx_create(0, 2, 32, 0)
    assert not lib.kgx_create(99, 2, 32, 1024) and lib.kgx_last_error(None) != b""


def test_launch_requires_params_and_single_flight():
    lib = kangaroo_b200.load_library()
    eng = GPUEngine(1, 1, 0, 64)
    assert lib.kgx_launch_async(eng._h) != 0 and b"kgx_set_params" in lib.kgx_last_error(eng._h)
    z2, z4 = np.ones((32, 2), dtype=np.uint64), np.ones((32, 4), dtype=np.uint64)
    eng.SetParams(0xFFFFFFFFFFFFFFFF, z2, z4, z4)
    # a herd of copies of G with an all-ones "table" is arithmetically meaningless but must not fault
    G = (0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798, 0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8)
    eng.SetKangaroos([G[0]] * 128, [G[1]] * 128, [5] * 128)
    assert eng.callKernel()
    assert lib.kgx_launch_async(eng._h) != 0 and b"not collected" in lib.kgx_last_error(eng._h)
    eng.Launch(relaunch=False)
    eng.close()


def test_patch_out_of_range_and_collect_without_launch():
    lib = kangaroo_b200.load_library()
    eng = GPUEngine(1, 1, 0, 64)
    one = np.ones((1, 4), dtype=np.uint64)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))
    assert lib.kgx_patch(eng._h, 128, p(one), p(one), p(one)) != 0 and b"out of range" in lib.kgx_last_error(eng._h)
    n, f = ctypes.c_uint32(7), ctypes.c_uint32(7)
    items = (Item * 64)()
    assert lib.kgx_collect(eng._h, items, 64, ctypes.byref(n), ctypes.byref(f), 0, 0) == 0      # Check.cpp:526: Launch before any kernel
    assert n.value == 0 and f.value == 0
    eng.close()


SYM_REFUSALS = [
    ({"KGX_MODE": "stream", "KGX_STREAM_CTAS": "3"}, 2, b"2-CTA"),
    ({"KGX_MODE": "resident", "KGX_CFG": "64,5"}, 2, b"64,5 has no symmetric"),
    ({"KGX_MODE": "tmem"}, 2, b"cluster tile kernel"),
    ({"KGX_MODE": "stream"}, 3, b"mode must be"),
]


@pytest.mark.parametrize("env,mode,msg", SYM_REFUSALS, ids=["stream-ctas3", "resident-64,5", "tmem", "mode3"])
def test_symmetry_refused_where_no_symmetric_kernel_runs(env, mode, msg, monkeypatch):
    """kgx_set_symmetry on an engine with no symmetric instantiation, or with an unknown rule, fails and leaves the engine
    non-symmetric."""
    from tests.test_gpu_modes import KGX_VARS
    lib = kangaroo_b200.load_library()
    for k in KGX_VARS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng = GPUEngine(1, 1, 0, 64)
    assert eng.kernel == env["KGX_MODE"]
    assert lib.kgx_set_symmetry(eng._h, mode) != 0 and msg in lib.kgx_last_error(eng._h)
    assert lib.kgx_get_symmetry(eng._h) == 0
    eng.close()


def test_symmetry_refused_while_a_launch_is_in_flight(monkeypatch):
    monkeypatch.delenv("KGX_CFG", raising=False)
    lib = kangaroo_b200.load_library()
    eng = GPUEngine(1, 1, 0, 64, kernel="resident")
    z2, z4 = np.ones((32, 2), dtype=np.uint64), np.ones((32, 4), dtype=np.uint64)
    eng.SetParams(0xFFFFFFFFFFFFFFFF, z2, z4, z4)
    G = (0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798, 0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8)
    eng.SetKangaroos([G[0]] * 128, [G[1]] * 128, [5] * 128)
    assert eng.callKernel()
    assert lib.kgx_set_symmetry(eng._h, 2) != 0 and b"in flight" in lib.kgx_last_error(eng._h)
    assert lib.kgx_get_symmetry(eng._h) == 0
    eng.Launch(relaunch=False)
    assert lib.kgx_set_symmetry(eng._h, 2) == 0 and lib.kgx_get_symmetry(eng._h) == 2      # refused only for the launch
    eng.close()


def test_unknown_kernel_mode_is_rejected(monkeypatch):
    lib = kangaroo_b200.load_library()
    monkeypatch.setenv("KGX_MODE", "cpu")
    assert not lib.kgx_create(0, 1, 1, 64) and b"KGX_MODE" in lib.kgx_last_error(None)
