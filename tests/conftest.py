import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


try:  # property tests: same examples on every run, nothing written into the tree
    from hypothesis import settings as _hyp_settings
    _hyp_settings.register_profile("repo", derandomize=True, database=None)
    _hyp_settings.load_profile("repo")
except ImportError:  # hypothesis is optional: the fuzz files skip themselves without it
    pass


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA GPU (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "multigpu: test needs >= 2 GPUs")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _deterministic_global_rng(request):
    """Every test starts from a seed derived from its own name: statistical assertions (unbiasedness, sampled atom
    counts) see the same draws on every run and every machine instead of a fresh entropy seed per process."""
    import zlib

    import torch
    torch.manual_seed(zlib.crc32(request.node.nodeid.encode()) & 0x7FFFFFFF)
    yield
