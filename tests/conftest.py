import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    if not config.pluginmanager.hasplugin("timeout"):
        # pytest-timeout absent: the marker is registered so that it is not an unknown-mark warning, and the emulated
        # kernel tests (which rely on it against deadlocked barriers) install their own watchdog (see below)
        config.addinivalue_line("markers", "timeout(seconds): per-test time limit (pytest-timeout)")


@pytest.fixture(autouse=True)
def _watchdog_without_pytest_timeout(request):
    """Without the pytest-timeout plugin a `timeout` marker would be a silent no-op: arm a faulthandler watchdog that
    dumps all stacks and exits instead, so a deadlocked emulated barrier cannot hang the suite."""
    mark = request.node.get_closest_marker("timeout")
    if mark is None or request.config.pluginmanager.hasplugin("timeout"):
        yield
        return
    import faulthandler
    faulthandler.dump_traceback_later(float(mark.args[0]) if mark.args else 900.0, exit=True)
    try:
        yield
    finally:
        faulthandler.cancel_dump_traceback_later()


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))


def lib_from_fixture(d, prefix="lib_"):
    from irbpp_b200 import shapes
    res = d[prefix + "res"]
    return shapes.ShapeLibrary.from_flat(d[prefix + "dims"], d[prefix + "ext"], d[prefix + "vol"],
                                         d[prefix + "maps"], d[prefix + "offsets"], float(res[0]), float(res[1]))


@pytest.fixture(scope="session")
def golden():
    return load_golden
