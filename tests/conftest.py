import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """the C-ABI library must exist for every test (CPU tests exercise its host-side entry points)"""
    lib = os.path.join(ROOT, "madnlp.jl_b200", "csrc", "libb200kkt.so")
    if not os.path.exists(lib):
        sys.path.insert(0, ROOT)
        import __graft_entry__ as g
        g.build()
    yield
