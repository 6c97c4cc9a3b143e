import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "ma-lio_b200"), os.path.join(ROOT, "oracle"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure the checkers and the product library exist (cheap no-op when already built)."""
    import __graft_entry__ as g
    g.build(quiet=True)
