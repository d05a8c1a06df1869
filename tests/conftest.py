import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def ctx():
    from tinygp_b200 import _cabi

    return _cabi.get_context()


@pytest.fixture(autouse=True)
def _library_defaults(request):
    """GPU tests share one process-global context: every test starts from, and leaves behind, the LIBRARY defaults
    (b200gp_set_option "reset"), so a test that changes an option -- or fails half-way -- cannot leak it into later
    tests (round 1: restores to a literal 8 digit planes made the full-size golden test run a non-default path)."""
    if request.node.get_closest_marker("gpu") is None:
        yield
        return
    from tinygp_b200 import _cabi

    c = _cabi.get_context()
    c.reset_options()
    yield
    c.reset_options()
