import os
import os.path as osp
import sys

import pytest

ROOT = osp.dirname(osp.dirname(osp.abspath(__file__)))
for p in (ROOT, osp.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; select with -m gpu)')


@pytest.fixture(scope='session')
def golden():
    import numpy as np
    out = dict(np.load(osp.join(ROOT, 'tests', 'golden', 'reference_outputs.npz')))
    # bf16 / fp16 results are stored in their own 16-bit encoding (lossless, and small enough to keep each file < 1 MB)
    lowp = np.load(osp.join(ROOT, 'tests', 'golden', 'reference_outputs_lowp.npz'))
    for k in lowp.files:
        a = lowp[k]
        out[k] = (a.astype(np.uint32) << 16).view(np.float32) if a.dtype == np.uint16 else a.astype(np.float32)
    return out
