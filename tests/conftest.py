import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


def _usable_devices():
    """mb2_device_count() of the product library, 0 when the library is missing (no compute call is made)."""
    try:
        from momentum_b200 import solver as ms

        return int(ms.load_library().mb2_device_count())
    except Exception:  # noqa: BLE001 - library not built / not loadable
        # on a box WITH a GPU a missing extension must fail the gpu tests loudly, not skip them
        return 1 if os.path.exists("/dev/nvidiactl") else 0


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a box without an sm_90 device skips the gpu tests instead of failing them; `-m gpu` on a GPU
    box runs them (and fails loudly if the extension is missing there: the skip only applies when no device is usable)."""
    gpu_items = [it for it in items if it.get_closest_marker("gpu") is not None]
    if not gpu_items or _usable_devices() > 0:
        return
    skip = pytest.mark.skip(reason="no usable sm_90 CUDA device (momentum_b200 has no CPU fallback)")
    for it in gpu_items:
        it.add_marker(skip)
