import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
for _p in (str(ROOT), str(Path(__file__).resolve().parent)):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA GPU (an H100; run with -m gpu on a GPU machine)')


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests need a CUDA device and the in-tree library: on a box without them they are skipped (a plain
    `pytest` run there must not hard-fail), never silently passed."""
    import torch
    lib = ROOT / 'style-transfer-pytorch_b200' / 'libstb200.so'
    why = None
    if not torch.cuda.is_available():
        why = 'no CUDA device'
    elif not lib.exists():
        why = f'{lib.name} not built'
    if why:
        skip = pytest.mark.skip(reason=why)
        for item in items:
            if 'gpu' in item.keywords:
                item.add_marker(skip)


@pytest.fixture(scope='session')
def vgg_weights():
    from oracle import st_oracle as O
    return O.make_vgg_weights(1234)
