import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")
    config.addinivalue_line("markers", "slow: long-running")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def load_golden(name):
    import gzip
    import json

    p = os.path.join(GOLDEN, name)
    if p.endswith(".gz"):
        with gzip.open(p, "rb") as f:
            return json.loads(f.read().decode())
    with open(p) as f:
        return json.load(f)
