import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'gptq-for-llama_b200')
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (pytest -m gpu)')


def pytest_collection_modifyitems(config, items):
    """GPU tests must never pass silently on a box without a GPU: they are skipped there, and on a GPU
    box the CUDA library has to be the thing that runs (ops raises if it is missing)."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden_cases():
    import glob
    import numpy as np
    out = {}
    for f in sorted(glob.glob(os.path.join(GOLDEN, 'pack_*.npz'))):
        out[os.path.basename(f)[5:-4]] = dict(np.load(f))
    assert len(out) >= 8
    return out
