import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the oracle is the checker; build it if the .so is not there yet (gcc only, seconds)
    if not os.path.exists(os.path.join(ROOT, "oracle", "liboracle.so")):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])


def _has_gpu():
    # a library that does not load is an error, never a reason to skip the GPU tests
    import lurk_beta_b200 as L
    return L._capi.lib().lurk_device_count() > 0


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def L():
    import lurk_beta_b200
    return lurk_beta_b200


@pytest.fixture(scope="session")
def oracle():
    from oracle import capi
    return capi


@pytest.fixture(scope="session")
def spec():
    from oracle import spec as s
    return s
