import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# every engine buffer starts as 0xFF bytes in the test-suite: reads of never-written device memory become NaNs / wild indices
os.environ.setdefault('TDIFF_POISON', '1')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; select with -m gpu)')


def pytest_collection_modifyitems(config, items):
    # `-m gpu` tests must not silently skip on a GPU box; on a CPU box they are deselected by `-m "not gpu"`.
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if not has_gpu:
        skip = pytest.mark.skip(reason='no CUDA device')
        for it in items:
            if 'gpu' in it.keywords:
                it.add_marker(skip)
