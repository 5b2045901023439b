import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def b200():
    """The product library bound to cuda:0 (fails loudly when there is no sm_90 device)."""
    import svt_av1_psy_b200 as pkg
    pkg.init(0)
    yield pkg.dsp
    pkg.shutdown()


@pytest.fixture(scope="session")
def oracle():
    import oracle as o
    return o


@pytest.fixture(scope="session")
def refc(oracle, request):
    """ctypes handle on the unmodified reference objects.  For a GPU test a missing oracle is an ERROR -- the parity
    tests must not silently skip; the CPU pins may run on a clone where the reference sources are not available."""
    if oracle.ref is None:
        if request.node.get_closest_marker("gpu") is not None:
            pytest.fail("oracle/_ref/libsvtav1_ref.so is missing: build it with `python __graft_entry__.py --oracle` where "
                        "the reference sources are available")
        pytest.skip("oracle/_ref/libsvtav1_ref.so not built (no /root/reference)")
    return oracle.ref
