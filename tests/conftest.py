import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'vocal-remover_b200')
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a host without a GPU (or without the built library) skips the gpu-marked tests instead of
    failing them; on a GPU box nothing is skipped, so a missing library there is still a loud failure."""
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device visible (gpu-marked tests need an H100)')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """The arrays of fixture `name`, merged from its tests/golden/<name>.partN.npz files (oracle/make_golden.py)."""
    import glob
    import numpy as np
    paths = sorted(glob.glob(os.path.join(GOLDEN, name + '.part*.npz')))
    assert paths, 'missing golden fixture ' + name
    out = {}
    for path in paths:
        with np.load(path) as part:
            out.update({k: part[k] for k in part.files})
    return out


@pytest.fixture(scope='session')
def golden_default():
    return load_golden('ref_10s_default')


@pytest.fixture(scope='session')
def golden_small():
    return load_golden('ref_3s_small')


@pytest.fixture(scope='session')
def golden_direct():
    return load_golden('ref_direct')


def checksum(a):
    import numpy as np
    a = np.asarray(a)
    if np.iscomplexobj(a):
        return np.array([a.real.astype(np.float64).sum(), a.imag.astype(np.float64).sum(),
                         (np.abs(a).astype(np.float64) ** 2).sum(), np.abs(a).max()], dtype=np.float64)
    a64 = a.astype(np.float64)
    return np.array([a64.sum(), (a64 ** 2).sum(), a64.min(), a64.max()], dtype=np.float64)


_PARITY_PATH = os.environ.get('VR_PARITY_JSON')


def record_parity(name, value, tol=None):
    """Report a measured parity number (max-abs error of the CUDA path vs the oracle / golden fixture) so that the
    margin under the gate is on record, not only the pass/fail bit; also merged into the JSON file named by
    VR_PARITY_JSON when that is set."""
    import json
    if _PARITY_PATH:
        try:
            os.makedirs(os.path.dirname(os.path.abspath(_PARITY_PATH)), exist_ok=True)
            data = {}
            if os.path.exists(_PARITY_PATH):
                with open(_PARITY_PATH) as f:
                    data = json.load(f)
            data[name] = {'max_abs_err': float(value)} if tol is None else {'max_abs_err': float(value), 'gate': float(tol)}
            with open(_PARITY_PATH, 'w') as f:
                json.dump(data, f, indent=1, sort_keys=True)
        except OSError:
            pass
    print('PARITY %s = %.4g%s' % (name, float(value), '' if tol is None else ' (gate %.1g)' % tol))
