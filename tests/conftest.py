import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_sessionstart(session):
    """A clean checkout has no built artefacts (they are git-ignored): build the CUDA library (nvcc cross-compiles
    without a GPU) and the oracle before collection, exactly what ``__graft_entry__.build()`` does.  The product
    package itself never builds implicitly."""
    from taichi_3d_gaussian_splatting_b200 import build as _build
    if not os.path.exists(_build.LIB):
        _build.build()
    from oracle import build_oracle
    build_oracle()


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import lib
    return lib()


@pytest.fixture(scope="session")
def golden():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "reference_vectors.json")) as f:
        return json.load(f)
