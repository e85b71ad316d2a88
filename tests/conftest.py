import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from lookoncetohear_b200.configs import EMBED_PARAMS as EMBED, TSH_PARAMS as TSH  # noqa: E402


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def tsh_params():
    return dict(TSH)


@pytest.fixture(scope="session")
def embed_params():
    return dict(EMBED)
