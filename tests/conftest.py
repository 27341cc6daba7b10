import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def load_golden(stem):
    """tests/golden/<stem>.<i>.npz merged: fixtures are stored in parts of under 1 MB each (tests/golden/make_golden*.py)."""
    import glob
    import numpy as np
    parts = sorted(glob.glob(os.path.join(REPO, 'tests', 'golden', f'{stem}.*.npz')))
    assert parts, f'no fixture parts for {stem}'
    return {k: v for p in parts for k, v in np.load(p).items()}


def save_golden(stem, arrays, part_bytes=900_000):
    """Write `arrays` as tests/golden/<stem>.<i>.npz parts of at most about part_bytes each (compressed)."""
    import glob
    import io
    import numpy as np
    for old in glob.glob(os.path.join(REPO, 'tests', 'golden', f'{stem}.*.npz')):
        os.remove(old)
    parts = [{}]
    for k, v in arrays.items():
        trial = dict(parts[-1], **{k: v})
        buf = io.BytesIO()
        np.savez_compressed(buf, **trial)
        if buf.tell() > part_bytes and parts[-1]:
            parts.append({k: v})
        else:
            parts[-1] = trial
    for i, part in enumerate(parts):
        np.savez_compressed(os.path.join(REPO, 'tests', 'golden', f'{stem}.{i}.npz'), **part)


@pytest.fixture(scope='session')
def golden():
    return load_golden('reference_outputs')


def rel_l2(a, b):
    import torch
    a = torch.as_tensor(a).double().flatten()
    b = torch.as_tensor(b).double().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()
