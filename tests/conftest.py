import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# GPU tests written after the round's GPU budget was spent have never executed on an H100.  They are recorded as non-strict
# xfail so that an unvalidated TEST cannot turn a validated suite red: "xpassed" in a GPU run means the test ran and held,
# "xfailed" means the new test (or what it checks) needs attention.  The mark is removed once a GPU run has shown XPASS.
not_yet_run_on_gpu = pytest.mark.xfail(reason="added after the round's GPU budget was spent: never executed on an H100 "
                                              "(XPASS = validated)", strict=False)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU; run with -m gpu")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def lib():
    from visiondk_b200 import build, _lib
    build.build()
    return _lib.load()
