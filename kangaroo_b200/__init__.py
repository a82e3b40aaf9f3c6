"""kangaroo_b200 -- H100-native (sm_90a) Pollard's-kangaroo jump engine for secp256k1.

One hot path of JeanLucPons/Kangaroo rebuilt from scratch: the GPU jump engine behind `class GPUEngine`
(reference GPU/GPUEngine.h:40-84).  The product is the CUDA library `csrc/libkgx.so` (C ABI: include/kgx.h);
this package is the thin host-side mirror of the reference interface used by the tests, bench.py and the
multi-GPU rank driver.  There is no CPU fallback: importing works anywhere, creating an engine needs a GPU.
"""
from .engine import GPUEngine, ITEM, NB_JUMP, NB_RUN, GPU_GRP_SIZE, TAME, WILD, random_herd_arrays  # noqa: F401
from ._lib import load_library, build_library, LIB_PATH  # noqa: F401
