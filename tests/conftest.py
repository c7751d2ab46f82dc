"""pytest configuration: registers the `gpu` marker and puts the repo root (for `oracle`) and the
product package directory `yolo2-pytorch_b200/` (for `b200`, `model`, `utils`, `detect`, `train`)
on sys.path.  The product directory mirrors the reference's import layout, so tests read
`import model.yolo2`, `import utils.postprocess` exactly like reference user code."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'yolo2-pytorch_b200')
for p in (PKG, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (select with -m gpu)')


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden_dir():
    return os.path.join(ROOT, 'tests', 'golden')
