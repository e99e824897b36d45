import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests need a CUDA device AND the built library: without them they are skipped (not errors), so a
    CPU-only run tells real failures from a missing GPU."""
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    have_lib = os.path.exists(os.path.join(ROOT, 'vbx_b200', 'libvbx_b200.so'))
    if have_gpu and have_lib:
        for item in items:         # a hung kernel must cost one test, not the whole GPU session (needs pytest-timeout)
            if 'gpu' in item.keywords and item.get_closest_marker('timeout') is None:
                item.add_marker(pytest.mark.timeout(180))
        return
    why = 'no CUDA device' if not have_gpu else 'vbx_b200/libvbx_b200.so not built'
    skip = pytest.mark.skip(reason=f'gpu test: {why}')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


GOLDEN = os.path.join(ROOT, 'tests', 'golden')


@pytest.fixture(scope='session')
def golden_dir():
    return GOLDEN
