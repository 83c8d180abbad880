import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
for p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs an H100 (sm_90a) GPU; run with -m gpu on a GPU machine')


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device in this container')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden():
    import numpy as np
    gdir = os.path.join(ROOT, 'tests', 'golden')
    return {name: np.load(os.path.join(gdir, name + '.npz')) for name in ('corr_lookup', 'update_blocks', 'models')}
