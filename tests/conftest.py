import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# tests/golden/ holds fixtures -- among them unmodified copies of the reference's own unit-test
# modules, which tests/test_reference_unit_tests.py runs in a subprocess with the drop-in aliased as
# `tritonclient`; pytest must not collect them itself
collect_ignore_glob = ["golden/*"]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def _has_gpu():
    try:
        import ctypes

        from client_b200 import _native

        n = ctypes.c_int(0)
        rc = _native.load().tb200_device_count(ctypes.byref(n))
        return rc == 0 and n.value > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def gpu_ops():
    """DeviceOps on cuda:0; the library must be there -- no fallback."""
    from client_b200 import _native
    from client_b200.device import DeviceOps

    assert _has_gpu(), "gpu-marked test but no usable CUDA device / libtb200.so"
    return DeviceOps(_native.default_context(0))
