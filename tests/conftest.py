import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')
    config.addinivalue_line('markers', 'refbin: needs the reference plant binaries under oracle/_ref')


def pytest_collection_modifyitems(config, items):
    """GPU tests go through the in-tree C-ABI library; build it (nvcc, sm_90a) if the tree arrived without it."""
    if any('gpu' in item.keywords for item in items):
        try:
            import torch
            from serl_b200 import _native, build
            if torch.cuda.is_available() and not os.path.exists(_native.LIB_PATH):
                build.build()
        except Exception as e:          # the tests themselves will fail loudly
            print('conftest: could not build libserl_b200.so:', e)
