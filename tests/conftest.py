import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not failed) on a box without CUDA."""
    reason = None
    try:
        import torch
        if not torch.cuda.is_available():
            reason = 'no CUDA device'
    except Exception as ex:   # noqa: BLE001
        reason = f'torch unavailable: {ex}'
    # (a missing libsevenn_b200.so on a CUDA box is NOT a reason to skip: those tests must fail loudly)
    if reason is None:
        return
    skip = pytest.mark.skip(reason=reason)
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def repo_root():
    return ROOT
