import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")
    config.addinivalue_line("markers", "slow: takes more than a few seconds on CPU")


@pytest.fixture(scope="session")
def oracle():
    from oracle import kgo
    return kgo.Oracle()


# Every oracle / reference-fixture parity test runs on BOTH jump kernels (kgx_create_ex): "stream128" is the benchmarked
# configuration (stream kernel, 128 kangaroos per thread, what the default 264x128 grid of an H100 resolves to), "stream" the
# adaptive group size small grids get, "resident" the shared-memory tile kernel.
KERNEL_VARIANTS = {"stream128": dict(kernel="stream", stream_g=128), "stream": dict(kernel="stream"), "resident": dict(kernel="resident"),
                   "tmem": dict(kernel="tmem")}      # cluster tile kernel: one 1792-kangaroo tile over the shared memory of 2 CTAs


@pytest.fixture(params=sorted(KERNEL_VARIANTS))
def kernel(request):
    return KERNEL_VARIANTS[request.param]
