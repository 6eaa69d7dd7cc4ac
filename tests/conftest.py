import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")

DEFAULT_ARGS = dict(use_bias=False, tanh=True, append_smoothers=True, resnet_blocks=7,
                    filters=[32, 64, 128, 128, 128, 64], input_channels=6)
VARIANT_ARGS = dict(use_bias=True, tanh=False, append_smoothers=False, resnet_blocks=2,
                    filters=[64, 64, 128, 128, 64, 32], input_channels=5)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (H100, sm_90) device; run with -m gpu on a GPU machine")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def built_lib():
    """The in-tree shared library (built by __graft_entry__.build())."""
    import __graft_entry__ as g
    if not os.path.exists(g.LIB):
        g.build()
    return g.LIB
