import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (H100); run with -m gpu on a GPU host')
    # The CPU oracle scales negatively past ~32 threads on the 128-core GPU hosts.
    import torch
    torch.set_num_threads(min(16, os.cpu_count() or 1))


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture
def flags():
    """Reference flag defaults, restored after the test."""
    from simclr_b200 import flags_def
    F = flags_def.FLAGS
    if not F.is_parsed():
        F(['test'])
    saved = {k: getattr(F, k) for k in flags_def.REFERENCE_FLAG_NAMES + ['b200_precision', 'b200_conv_engine']}
    yield flags_def
    for k, v in saved.items():
        setattr(F, k, v)
