import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    import oracle as O
    from oracle import build as oracle_build
    oracle_build.build_oracle()
    oracle_build.build_ref(sim=False)   # no-op without a reference checkout
    O.lib()
    return O


@pytest.fixture(scope="session")
def mm():
    """The product binding.  If the C-ABI library has not been built in this checkout yet (it is
    git-ignored), build it first — the test harness may do that, the product itself never falls
    back to anything when the library is missing."""
    import gemm_hls_b200 as G
    if not os.path.exists(G.LIB_PATH):
        from gemm_hls_b200 import build as product_build
        product_build.build()
    G.lib()
    return G
