import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


def pytest_collection_modifyitems(config, items):
    """gpu-marked tests are SKIPPED (not errored) on a machine without an H100; everything else runs everywhere."""
    try:
        from glim_b200 import capi

        have_gpu = capi.lib().gb_device_count() > 0
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs an H100 (no CUDA device visible)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def pytest_sessionstart(session):
    """The suites need the native artefacts (the library for the boundary tests even without a GPU, the oracle everywhere).
    They are git-ignored build products: build them if a fresh checkout has none (nvcc cross-compiles without a GPU)."""
    lib = os.path.join(ROOT, "glim_b200", "libglim_b200.so")
    orc = os.path.join(ROOT, "oracle", "libglim_oracle.so")
    if not (os.path.exists(lib) and os.path.exists(orc)):
        import __graft_entry__

        __graft_entry__.build()


@pytest.fixture(scope="session")
def ctx():
    """One gb_ctx for the whole GPU test session (fails loudly when libglim_b200.so or the GPU is missing)."""
    from glim_b200 import gpu

    c = gpu.Context(0)
    yield c
    c.synchronize()
