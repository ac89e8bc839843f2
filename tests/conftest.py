import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def _ensure_native_built():
    """The native libs are git-ignored build products.  Build them only when missing (on the GPU box the
    prebuilt files travel with the snapshot; mtimes are not reliable there, so no staleness check)."""
    import os

    import __graft_entry__ as entry

    _build = entry.load_build_module()   # by path: the package itself cannot be imported before the libraries exist
    libs = (_build.LIB / "libao_b200.so", _build.LIB / "ao_b200_torch.so")
    if not all(p.exists() for p in libs) or os.environ.get("AO_B200_FORCE_BUILD"):
        _build.build_all(force=True)
    from oracle import oracle as o

    if not (o._DIR / "_build" / "libao_oracle.so").exists():
        o.build()


_ensure_native_built()
