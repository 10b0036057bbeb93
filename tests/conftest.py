import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _exact_engine_unless_parametrised(request):
    """GPU tests that do not ask for the ``engine`` fixture were written against the exact fp32 engine; the library
    default is the product engine (tf32x3), so select fp32 for them explicitly and restore the default afterwards."""
    if "gpu" not in request.keywords:
        yield
        return
    import ta3n_b200
    ta3n_b200.set_gemm_engine("fp32")
    yield
    ta3n_b200.set_gemm_engine("tf32x3")
