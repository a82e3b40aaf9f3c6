"""CPU-side checks of the boundary: the C-ABI library loads and exports every symbol include/kgx.h declares,
the product fails loudly without a GPU (no CPU fallback), and the host-portable safegcd inverse is correct."""
import ctypes
import os
import random
import re

import pytest

import kangaroo_b200
from kangaroo_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_are_exported():
    hdr = open(os.path.join(ROOT, "include", "kgx.h")).read()
    declared = set(re.findall(r"\b(kgx_[a-z_0-9]+)\s*\(", hdr))
    lib = kangaroo_b200.load_library()
    for name in sorted(declared):
        assert hasattr(lib, name), name
    assert declared == set(_lib.EXPORTED_SYMBOLS)


def kernel_table(src, sym):
    """The entries of kgx_engine.cu's g_kernels table for the non-symmetric (sym = "false") or symmetric ("true") engine:
    ("resident", "T,K") per KGX_RESIDENT (in table order; the first is the default geometry), ("stream", CTAS, inverse) per
    KGX_STREAM and ("tmem",) for the cluster kernel's entry."""
    table = re.search(r"g_kernels\[\]\s*=\s*\{(.*?)\n\};", src, re.S).group(1)
    kernels = [("resident", "%s,%s" % (t, k)) for t, k in re.findall(
        r"KGX_RESIDENT\(\s*(\d+)\s*,\s*(\d+)\s*,\s*%s\s*\)" % sym, table)]
    for ctas, warp in re.findall(r"KGX_STREAM\(\s*(\d+)\s*,\s*(true|false)\s*,\s*%s\s*\)" % sym, table):
        kernels.append(("stream", ctas, "warp" if warp == "true" else "thread"))
    if re.search(r"\b%s\s*,\s*jump_kernel_cluster\b" % sym, table):      # the entry's sym field precedes its function
        kernels.append(("tmem",))
    return kernels


def compiled_jump_kernels(src):
    """The jump-kernel instantiations kgx_engine.cu launches in the non-symmetric engine, and its default tile geometry."""
    kernels = kernel_table(src, "false")
    return set(kernels), kernels[0][1]


def variant_kernel(env, default_geometry):
    """The instantiation a tests/test_gpu_modes.py variant selects, or None where that depends on the herd size."""
    mode = env["KGX_MODE"]
    if mode == "resident":
        return ("resident", env.get("KGX_CFG", default_geometry))
    if mode == "tmem":
        return ("tmem",)
    inv = env.get("KGX_STREAM_INV") or ("warp" if int(env.get("KGX_STREAM_G", "0")) >= 64 else None)
    return ("stream", env.get("KGX_STREAM_CTAS", "2"), inv) if inv else None


def compiled_symmetric_jump_kernels(src):
    """The instantiations the symmetric engine (kgx_set_symmetry) launches."""
    return set(kernel_table(src, "true"))


def symmetric_variant_kernel(env, default_geometry):
    """The instantiation a SYM_VARIANTS entry selects.  The symmetric engine ignores KGX_STREAM_INV: its stream kernel always
    takes the warp inverse."""
    mode = env["KGX_MODE"]
    if mode == "resident":
        return ("resident", env.get("KGX_CFG", default_geometry))
    if mode == "tmem":
        return ("tmem",)
    return ("stream", env.get("KGX_STREAM_CTAS", "2"), "warp")


def check_variants_cover(src, variants, sym_variants):
    kernels, default_geometry = compiled_jump_kernels(src)
    selected = {variant_kernel(v, default_geometry) for v in variants} - {None}
    assert kernels - selected == set(), "compiled jump kernels that no entry of VARIANTS runs"
    assert selected - kernels == set(), "VARIANTS entries that select no compiled jump kernel"
    kernels = compiled_symmetric_jump_kernels(src)
    selected = {symmetric_variant_kernel(v, default_geometry) for v in sym_variants}
    assert kernels - selected == set(), "compiled symmetric jump kernels that no entry of SYM_VARIANTS runs"
    assert selected - kernels == set(), "SYM_VARIANTS entries that select no compiled symmetric jump kernel"


def test_every_compiled_jump_kernel_has_a_gpu_test():
    """tests/test_gpu_modes.py runs every entry of VARIANTS and SYM_VARIANTS; a geometry or stream instantiation added to
    kgx_engine.cu without an entry there fails here, on a machine without a GPU."""
    from tests.test_gpu_modes import SYM_VARIANTS, VARIANTS
    src = open(os.path.join(ROOT, "kangaroo_b200", "csrc", "kgx_engine.cu")).read()
    kernels, _ = compiled_jump_kernels(src)
    assert {("resident", "128,7"), ("resident", "96,6"), ("stream", "3", "thread"), ("tmem",)} <= kernels   # the parser finds them
    assert compiled_symmetric_jump_kernels(src) == {("resident", "128,7"), ("stream", "2", "warp")}
    check_variants_cover(src, VARIANTS, SYM_VARIANTS)
    # the guard itself: one more geometry, one more symmetric geometry, or one variant fewer, must fail it
    extra = src.replace("KGX_RESIDENT(32, 12, false),", "KGX_RESIDENT(32, 12, false), KGX_RESIDENT(160, 3, false),")
    extra_sym = src.replace("KGX_RESIDENT(64, 7, false),", "KGX_RESIDENT(64, 7, false), KGX_RESIDENT(64, 7, true),")
    assert extra != src and extra_sym != src
    for bad_src in (extra, extra_sym):
        with pytest.raises(AssertionError):
            check_variants_cover(bad_src, VARIANTS, SYM_VARIANTS)
    with pytest.raises(AssertionError):
        check_variants_cover(src, [v for v in VARIANTS if v.get("KGX_CFG") != "96,6"], SYM_VARIANTS)
    with pytest.raises(AssertionError):
        check_variants_cover(src, VARIANTS, [v for v in SYM_VARIANTS if v["KGX_MODE"] != "resident"])


def adaptive_group_bounds(src):
    """The (smallest, largest) stream group size kgx_create_ex picks from the herd size; the largest is the benchmarked one."""
    lo, hi = (int(re.search(r"if \(g %s (\d+)\) g = \1;" % op, src).group(1)) for op in "<>")
    return lo, hi


def check_log_variants_cover(src, log_variants, sym_log_variants):
    """tests/test_gpu_jumplog.py's matrices, in each engine mode: every stream instantiation at the adaptive group size, the
    stream kernel at the smallest group size (CTAs loop over tiles) and one step above the largest (the longest log run
    stride), in the non-symmetric engine also at the largest (the benchmarked kernel), and as controls without a log the
    default tile and the cluster kernel where the mode compiles them."""
    kernels, default_geometry = compiled_jump_kernels(src)
    lo, hi = adaptive_group_bounds(src)
    for name, variants, compiled, select, sizes in (
            ("LOG_VARIANTS", log_variants, kernels, variant_kernel, {lo, hi, hi + 2}),
            ("SYM_LOG_VARIANTS", sym_log_variants, compiled_symmetric_jump_kernels(src), symmetric_variant_kernel, {lo, hi + 2})):
        streams = {k for k in compiled if k[0] == "stream"}
        adaptive = {select(v, default_geometry) for v in variants if v["KGX_MODE"] == "stream" and "KGX_STREAM_G" not in v}
        assert streams - adaptive == set(), "stream instantiations that no entry of %s runs at the adaptive group size" % name
        explicit = {int(v["KGX_STREAM_G"]) for v in variants if "KGX_STREAM_G" in v}
        assert sizes - explicit == set(), "stream group sizes that no entry of %s runs" % name
        selected = {select(v, default_geometry) for v in variants} - {None}
        controls = {("resident", default_geometry), ("tmem",)} & compiled
        assert controls - selected == set(), "kernels without a log that %s does not run as controls" % name
        assert selected - compiled == set(), "%s entries that select no compiled kernel" % name


def test_every_stream_instantiation_runs_multi_window_launches():
    """tests/test_gpu_jumplog.py runs LOG_VARIANTS and SYM_LOG_VARIANTS over several jump-log windows per launch; a stream
    instantiation added to kgx_engine.cu without an entry there, or an entry dropped, fails here."""
    from tests.test_gpu_jumplog import LOG_VARIANTS, SYM_LOG_VARIANTS
    src = open(os.path.join(ROOT, "kangaroo_b200", "csrc", "kgx_engine.cu")).read()
    assert adaptive_group_bounds(src) == (2, 128)
    check_log_variants_cover(src, LOG_VARIANTS, SYM_LOG_VARIANTS)
    # the guard itself: a 3-CTA symmetric stream kernel, or any one entry fewer in either list, must fail it
    sym3 = src.replace("KGX_STREAM(2, true, true)", "KGX_STREAM(3, true, true)")
    assert sym3 != src
    with pytest.raises(AssertionError):
        check_log_variants_cover(sym3, LOG_VARIANTS, SYM_LOG_VARIANTS)
    for i in range(len(LOG_VARIANTS)):
        with pytest.raises(AssertionError):
            check_log_variants_cover(src, LOG_VARIANTS[:i] + LOG_VARIANTS[i + 1:], SYM_LOG_VARIANTS)
    for i in range(len(SYM_LOG_VARIANTS)):
        with pytest.raises(AssertionError):
            check_log_variants_cover(src, LOG_VARIANTS, SYM_LOG_VARIANTS[:i] + SYM_LOG_VARIANTS[i + 1:])


def test_no_oracle_in_product():
    # the product package must never import / link the oracle
    for dirpath, _, files in os.walk(os.path.join(ROOT, "kangaroo_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src and "kgx_oracle" not in src and "libkref" not in src, f


def test_engine_fails_loudly_without_gpu():
    lib = kangaroo_b200.load_library()
    if lib.kgx_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError, match="no CUDA device"):
        kangaroo_b200.GPUEngine(2, 32)


def test_host_modinv_safegcd():
    L = ctypes.CDLL(_lib.HOSTTEST_PATH)
    P = 2**256 - 0x1000003D1

    def inv(a):
        i = (ctypes.c_uint64 * 4)(*[(a >> (64 * k)) & (2**64 - 1) for k in range(4)])
        o = (ctypes.c_uint64 * 4)()
        L.kgx_host_modinv(o, i)
        return sum(o[k] << (64 * k) for k in range(4))

    rng = random.Random(1)
    vals = [1, 2, 3, P - 1, P - 2, 2**255, (P + 1) // 2] + [2**k for k in range(256)] + [P - 2**k for k in range(255)]
    vals += [rng.randrange(1, P) for _ in range(5000)]
    for a in vals:
        assert inv(a) == pow(a, -1, P)
    assert inv(0) == 0      # GPUMath.h:785-793


def test_host_fp64_multiplier_is_exact():
    """kgx_field_fp64.cuh (the DFMA-pipe 256x256 -> 512 multiplier, 52-bit limbs, round-toward-zero FMA splitting): the host
    twin must reproduce big-integer products exactly, incl. all-ones and limb-boundary operands."""
    import ctypes
    import random
    from kangaroo_b200 import _lib
    L = ctypes.CDLL(_lib.HOSTTEST_PATH)
    A, O = ctypes.c_uint64 * 4, ctypes.c_uint64 * 8
    M = 2**64 - 1

    def mul(a, b, sq=0):
        o = O()
        L.kgx_host_mul512_fp64(o, A(*[(a >> (64 * i)) & M for i in range(4)]), A(*[(b >> (64 * i)) & M for i in range(4)]), sq)
        return sum(int(o[i]) << (64 * i) for i in range(8))
    random.seed(5)
    edge = [0, 1, 2**256 - 1, 2**255, 2**52 - 1, 2**52, 2**104 - 1, 2**104, 2**208 - 1, (1 << 256) - (1 << 52), 2**256 - 0x1000003D1]
    vals = edge + [random.getrandbits(256) for _ in range(1500)]
    for i, a in enumerate(vals):
        b = vals[(i * 7 + 3) % len(vals)]
        assert mul(a, b) == a * b
        assert mul(a, a, 1) == a * a
    for a in edge:
        for b in edge:
            assert mul(a, b) == a * b
