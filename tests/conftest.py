import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def built_lib():
    import __graft_entry__ as g
    g.build()
    from videoseal_b200 import _lib
    return _lib.lib()
