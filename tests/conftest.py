import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built_lib():
    from ipopt_b200.capi import lib_path
    if not os.path.exists(lib_path()):
        import __graft_entry__
        __graft_entry__.build()
    return lib_path()
