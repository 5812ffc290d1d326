import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
SCENES = os.path.join(ROOT, "tests", "scenes")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def pb():
    import pbrt_v3_b200
    pbrt_v3_b200.lib()  # fails loudly if the extension has not been built
    return pbrt_v3_b200


@pytest.fixture(scope="session")
def port():
    from oracle import pyoracle
    o = pyoracle.port()
    if o is None:
        pytest.fail("oracle/lib/libpb2_oracle.so is missing: run __graft_entry__.build()")
    return o


@pytest.fixture(scope="session")
def checker(port):
    """The strongest CPU checker available: the compiled reference if present, else the port."""
    from oracle import pyoracle
    return pyoracle.reference() or port
