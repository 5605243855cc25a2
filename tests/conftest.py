import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def engine_lib():
    """Build (if needed) and load the CUDA engine library; never falls back to anything else."""
    from whisper_medusa_b200 import _lib, build

    if not os.path.isfile(_lib.LIB_PATH):
        build.build()
    return _lib.load()
