"""Shared test plumbing: path setup, the ``gpu`` marker, golden-fixture loading."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "pytorch-wavenet_b200")
GOLDEN = os.path.join(ROOT, "tests", "golden")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not failed) when no device is visible, e.g. when someone runs the whole suite here."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """The arrays of tests/golden/<name> (fixtures over 900 KB are stored in shards, see golden_store.py)."""
    import golden_store
    return golden_store.load(os.path.join(GOLDEN, name))


@pytest.fixture(scope="session")
def golden():
    return load_golden
