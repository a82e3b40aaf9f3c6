"""ctypes bindings for the parity oracle (TEST INFRASTRUCTURE ONLY).

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference legs) may import this
module.  The product package `kangaroo_b200` never does.

Two back ends with the same function set:
  * Oracle()    -> oracle/libkgx_oracle.so  : the C restatement (kgx_oracle.c), prefix kgo_
  * Reference() -> oracle/_ref/libkref.so   : the reference's own SECPK1 code behind ref_harness.cpp, prefix ref_
Field elements / scalars cross the boundary as Python ints; arrays as numpy uint64 of shape (n, limbs).
"""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
P = 2**256 - 0x1000003D1
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
GX = 0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798
GY = 0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8
NB_JUMP = 32

_u64p = ctypes.POINTER(ctypes.c_uint64)


class DP(ctypes.Structure):
    _fields_ = [("x", ctypes.c_uint64 * 4), ("d", ctypes.c_uint64 * 4), ("kidx", ctypes.c_uint64),
                ("jump", ctypes.c_uint32), ("pad", ctypes.c_uint32)]


def to_limbs(v, limbs=4):
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(limbs)], dtype=np.uint64)


def from_limbs(a):
    a = np.asarray(a, dtype=np.uint64).reshape(-1)
    return sum(int(a[i]) << (64 * i) for i in range(a.shape[0]))


def ints_to_array(vals, limbs=4):
    out = np.zeros((len(vals), limbs), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(limbs):
            out[i, k] = (v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF
    return out


def array_to_ints(a):
    a = np.asarray(a, dtype=np.uint64)
    return [from_limbs(a[i]) for i in range(a.shape[0])]


def _ptr(a):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(_u64p)


def build(ref=True):
    """Build the oracle (and, where KANGAROO_REF names the reference sources, the reference harness)."""
    subprocess.check_call(["make", "-s", "-C", HERE, "oracle"] + (["ref"] if ref else []))


class _Backend:
    prefix = None
    path = None

    def __init__(self):
        if not os.path.exists(self.path):
            build(ref=(self.prefix == "ref_"))
        self.lib = ctypes.CDLL(self.path)
        L, p = self.lib, self.prefix
        self._f = lambda name: getattr(L, p + name)
        self._f("jump_cpu").restype = ctypes.c_uint64
        self._f("create_jump_table").restype = ctypes.c_int
        self._f("rndl").restype = ctypes.c_uint32
        if p == "ref_":
            L.ref_init()
            L.ref_bench_cpu.restype = ctypes.c_uint64
        else:
            L.kgo_jump_gpu_conv.restype = ctypes.c_uint64
            L.kgo_dp_mask.restype = ctypes.c_uint64
            L.kgo_bench_cpu.restype = ctypes.c_uint64
            L.kgo_ec_mul_g.restype = ctypes.c_int
            L.kgo_ec_on_curve.restype = ctypes.c_int

    # --- scalar helpers -------------------------------------------------------------------------
    def _bin(self, name, a, b):
        r = np.zeros(4, dtype=np.uint64)
        self._f(name)(_ptr(r), _ptr(to_limbs(a)), _ptr(to_limbs(b)))
        return from_limbs(r)

    def mod_mul(self, a, b): return self._bin("mod_mul", a, b)
    def mod_sub(self, a, b): return self._bin("mod_sub", a, b)
    def order_add(self, a, b): return self._bin("order_add", a, b)
    def order_sub(self, a, b): return self._bin("order_sub", a, b)

    def mod_sqr(self, a):
        r = np.zeros(4, dtype=np.uint64)
        self._f("mod_sqr")(_ptr(r), _ptr(to_limbs(a)))
        return from_limbs(r)

    def mod_inv(self, a):
        r = np.zeros(4, dtype=np.uint64)
        self._f("mod_inv")(_ptr(r), _ptr(to_limbs(a)))
        return from_limbs(r)

    def ec_mul_g(self, k):
        rx = np.zeros(4, dtype=np.uint64); ry = np.zeros(4, dtype=np.uint64)
        self._f("ec_mul_g")(_ptr(rx), _ptr(ry), _ptr(to_limbs(k)))
        return from_limbs(rx), from_limbs(ry)

    def ec_add(self, a, b):
        rx = np.zeros(4, dtype=np.uint64); ry = np.zeros(4, dtype=np.uint64)
        self._f("ec_add")(_ptr(rx), _ptr(ry), _ptr(to_limbs(a[0])), _ptr(to_limbs(a[1])),
                          _ptr(to_limbs(b[0])), _ptr(to_limbs(b[1])))
        return from_limbs(rx), from_limbs(ry)

    def rseed(self, s): self._f("rseed")(ctypes.c_uint32(s & 0xFFFFFFFF))
    def rndl(self): return int(self._f("rndl")())

    def rand_bits(self, nbit):
        r = np.zeros(4, dtype=np.uint64)
        self._f("rand_bits")(_ptr(r), ctypes.c_int(nbit))
        return from_limbs(r)

    # --- search set-up ---------------------------------------------------------------------------
    def create_jump_table(self, range_power):
        """-> (jd (32,2), jpx (32,4), jpy (32,4)) uint64 arrays. Kangaroo.cpp:742-832."""
        jd = np.zeros((NB_JUMP, 2), dtype=np.uint64)
        jpx = np.zeros((NB_JUMP, 4), dtype=np.uint64)
        jpy = np.zeros((NB_JUMP, 4), dtype=np.uint64)
        self.last_draws = self._f("create_jump_table")(ctypes.c_int(range_power), _ptr(jd), _ptr(jpx), _ptr(jpy))
        return jd, jpx, jpy

    def create_herd(self, n, range_power, width_div2, key, first_type=0):
        """Kangaroo.cpp:670-738; uses the current MT state. -> px,py,d arrays (n,4); d is mod n."""
        px = np.zeros((n, 4), dtype=np.uint64); py = np.zeros((n, 4), dtype=np.uint64)
        d = np.zeros((n, 4), dtype=np.uint64)
        self._f("create_herd")(ctypes.c_int(n), ctypes.c_int(range_power), _ptr(to_limbs(width_div2)),
                               _ptr(to_limbs(key[0])), _ptr(to_limbs(key[1])), ctypes.c_int(first_type),
                               _ptr(px), _ptr(py), _ptr(d))
        return px, py, d

    # --- jump loop -------------------------------------------------------------------------------
    def jump_cpu(self, px, py, d, table, njumps, dp_mask, grp=1024, max_dp=1 << 20):
        """SolveKeyCPU inner loop (Kangaroo.cpp:375-433), CPU convention (d 256-bit mod n). In place.
        -> list of (x, d, kidx, jump) DPs."""
        jd, jpx, jpy = table
        n = px.shape[0]
        dps = (DP * max_dp)()
        cnt = self._f("jump_cpu")(ctypes.c_int(n), ctypes.c_int(njumps), ctypes.c_int(grp), _ptr(px), _ptr(py), _ptr(d),
                                  _ptr(jd), _ptr(jpx), _ptr(jpy), ctypes.c_uint64(dp_mask), dps,
                                  ctypes.c_uint64(max_dp))
        assert cnt <= max_dp, "DP buffer too small"
        return [(from_limbs(dps[i].x), from_limbs(dps[i].d), int(dps[i].kidx), int(dps[i].jump)) for i in range(cnt)]

    # --- USE_SYMMETRY paths (Constants.h:25) ------------------------------------------------------
    def create_jump_table_sym(self, range_power):
        """Kangaroo.cpp:742-832, USE_SYMMETRY branch -> (jd, jpx, jpy); self.last_uv = the two primes."""
        jd = np.zeros((NB_JUMP, 2), dtype=np.uint64)
        jpx = np.zeros((NB_JUMP, 4), dtype=np.uint64)
        jpy = np.zeros((NB_JUMP, 4), dtype=np.uint64)
        uv = np.zeros(2, dtype=np.uint64)
        f = self._f("create_jump_table_sym"); f.restype = ctypes.c_int
        self.last_draws = f(ctypes.c_int(range_power), _ptr(jd), _ptr(jpx), _ptr(jpy), _ptr(uv))
        assert self.last_draws > 0
        self.last_uv = (int(uv[0]), int(uv[1]))
        return jd, jpx, jpy

    def create_herd_sym(self, n, range_power, width_div4, key, first_type=0):
        """Kangaroo.cpp:670-738, USE_SYMMETRY branch -> px, py, d (n,4); y already in the lower half, d sign-switched with it."""
        px = np.zeros((n, 4), dtype=np.uint64); py = np.zeros((n, 4), dtype=np.uint64)
        d = np.zeros((n, 4), dtype=np.uint64)
        self._f("create_herd_sym")(ctypes.c_int(n), ctypes.c_int(range_power), _ptr(to_limbs(width_div4)),
                                   _ptr(to_limbs(key[0])), _ptr(to_limbs(key[1])), ctypes.c_int(first_type),
                                   _ptr(px), _ptr(py), _ptr(d))
        return px, py, d

    def jump_sym(self, px, py, d, state, table, njumps, dp_mask, grp=1024, max_dp=1 << 20, rule="lastjump"):
        """The symmetric walk, in place.  rule "lastjump": Check.cpp:534-556 / GPUCompute.h:53-58 (state = last jump index, uint8,
        initially 32); rule "symclass": SolveKeyCPU, Kangaroo.cpp:381-384, 422-428 (state = symClass, initially 0).
        -> list of (x, d mod n, kidx, jump) DPs."""
        jd, jpx, jpy = table
        n = px.shape[0]
        dps = (DP * max_dp)()
        st = state.ctypes.data_as(ctypes.c_void_p)
        if self.prefix == "ref_":
            if rule == "lastjump":
                f = self._f("jump_sym"); f.restype = ctypes.c_uint64
                cnt = f(ctypes.c_int(n), ctypes.c_int(njumps), _ptr(px), _ptr(py), _ptr(d), st, _ptr(jd), _ptr(jpx), _ptr(jpy),
                        ctypes.c_uint64(dp_mask), dps, ctypes.c_uint64(max_dp))
            else:
                f = self._f("jump_symclass"); f.restype = ctypes.c_uint64
                cnt = f(ctypes.c_int(n), ctypes.c_int(njumps), ctypes.c_int(grp), _ptr(px), _ptr(py), _ptr(d), st, _ptr(jd), _ptr(jpx),
                        _ptr(jpy), ctypes.c_uint64(dp_mask), dps, ctypes.c_uint64(max_dp))
        else:
            f = self._f("jump_sym"); f.restype = ctypes.c_uint64
            cnt = f(ctypes.c_int(n), ctypes.c_int(njumps), ctypes.c_int(grp), _ptr(px), _ptr(py), _ptr(d), st, _ptr(jd), _ptr(jpx),
                    _ptr(jpy), ctypes.c_uint64(dp_mask), dps, ctypes.c_uint64(max_dp), ctypes.c_int(2 if rule == "symclass" else 1))
        assert cnt <= max_dp, "DP buffer too small"
        return [(from_limbs(dps[i].x), from_limbs(dps[i].d), int(dps[i].kidx), int(dps[i].jump)) for i in range(cnt)]

    def jump_single(self, x, y, d, table):
        """Check.cpp:534-549 formulation (one AddDirect per jump). -> (x, y, d)."""
        jd, jpx, jpy = table
        ax, ay, ad = to_limbs(x), to_limbs(y), to_limbs(d)
        self._f("jump_single")(_ptr(ax), _ptr(ay), _ptr(ad), _ptr(jd), _ptr(jpx), _ptr(jpy))
        return from_limbs(ax), from_limbs(ay), from_limbs(ad)

    def hash_convert(self, x, d, ktype):
        h = ctypes.c_uint64(0)
        X = np.zeros(2, dtype=np.uint64); D = np.zeros(2, dtype=np.uint64)
        self._f("hash_convert")(_ptr(to_limbs(x)), _ptr(to_limbs(d)), ctypes.c_uint32(ktype), ctypes.byref(h),
                                _ptr(X), _ptr(D))
        return int(h.value), from_limbs(X), from_limbs(D)

    def bench_cpu(self, threads, jumps_per_kangaroo, range_power=64):
        """-> (total_jumps, seconds): the SolveKeyCPU inner loop on `threads` pthreads x 1024 kangaroos."""
        sec = ctypes.c_double(0)
        tot = self._f("bench_cpu")(ctypes.c_int(threads), ctypes.c_int(jumps_per_kangaroo), ctypes.c_int(range_power),
                                   ctypes.byref(sec))
        return int(tot), float(sec.value)


class Oracle(_Backend):
    prefix = "kgo_"
    path = os.path.join(HERE, "libkgx_oracle.so")

    def jump_gpu_conv(self, px, py, d128, table, njumps, dp_mask, grp=1024, max_dp=1 << 20):
        """Device convention (GPUCompute.h:45-109): d is (n,2) uint64, 128-bit wrap, already biased."""
        jd, jpx, jpy = table
        n = px.shape[0]
        dps = (DP * max_dp)()
        cnt = self.lib.kgo_jump_gpu_conv(ctypes.c_int(n), ctypes.c_int(njumps), ctypes.c_int(grp), _ptr(px), _ptr(py),
                                         _ptr(d128), _ptr(jd), _ptr(jpx), _ptr(jpy), ctypes.c_uint64(dp_mask), dps,
                                         ctypes.c_uint64(max_dp))
        assert cnt <= max_dp, "DP buffer too small"
        return [(from_limbs(dps[i].x), from_limbs(dps[i].d), int(dps[i].kidx), int(dps[i].jump)) for i in range(cnt)]

    def dp_mask(self, bits): return int(self.lib.kgo_dp_mask(ctypes.c_int(bits)))

    def on_curve(self, x, y): return bool(self.lib.kgo_ec_on_curve(_ptr(to_limbs(x)), _ptr(to_limbs(y))))


class Reference(_Backend):
    prefix = "ref_"
    path = os.path.join(HERE, "_ref", "libkref.so")
