import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
if os.path.join(ROOT, 'tests') not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, 'tests'))

GOLDEN = os.path.join(ROOT, 'tests', 'golden')
# the parity tests load synthetic VGG weights AFTER construction; pretrained torchvision weights are not available offline
os.environ.setdefault('DASR_B200_ALLOW_RANDOM_VGG', '1')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden():
    import torch

    def load(name):
        # fixtures above 1 MB are stored as a skeleton NAME.pt plus NAME.partK.pt files, each {key path: tensor}
        obj = torch.load(os.path.join(GOLDEN, name), weights_only=False)
        k = 1
        while os.path.exists(os.path.join(GOLDEN, '%s.part%d.pt' % (name[:-3], k))):
            for path, t in torch.load(os.path.join(GOLDEN, '%s.part%d.pt' % (name[:-3], k)), weights_only=False).items():
                o = obj
                for key in path[:-1]:
                    o = o[key]
                o[path[-1]] = t
            k += 1
        return obj
    return load
