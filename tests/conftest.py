import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _ensure_library():
    """Build libcpb200.so when it is missing or stale (nvcc cross-compiles without a GPU), so a fresh checkout can run
    the suite directly; __graft_entry__.build() does the same."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("cpb_build", os.path.join(ROOT, "crypto_primitives_b200", "_build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    if mod.needs_build():
        mod.build()


_ensure_library()


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a device)")


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a machine without an H100 skips the gpu-marked tests instead of failing with CPB_NO_DEVICE."""
    from crypto_primitives_b200 import _native as N
    if N.lib.cpb_device_count() > 0:
        return
    skip = pytest.mark.skip(reason="no sm_90 device visible (cpb_device_count() == 0)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
