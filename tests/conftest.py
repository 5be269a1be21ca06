import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the product library and the oracle once per session (both compile without a GPU)."""
    from xflow_b200 import build as xbuild
    from oracle import oracle as O
    if not os.path.exists(xbuild.LIB):
        xbuild.build()
    O.build()
    yield


@pytest.fixture(scope="session")
def syn_data(tmp_path_factory):
    """The synthetic multi-block text shards of tests/golden/cases.py (regenerated from the seed)."""
    from common import materialise_syn
    return materialise_syn(str(tmp_path_factory.mktemp("syn")))
