"""The dataset inspection scripts without a GPU: the numpy vocal-image oracle against the images the reference's own
lib/dataset.py writes (tests/golden/ref_vocal_image, oracle/dataset_image_oracle.py), the import of lib.dataset
without cv2, and the failure of both scripts, run as files and as modules, before they write anything."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import PKG, checksum, load_golden


@pytest.fixture(scope='module')
def golden_vocal():
    return load_golden('ref_vocal_image')


def test_vocal_cases_regenerate(golden_vocal):
    from oracle import dataset_image_oracle
    for name, X, y in dataset_image_oracle.vocal_cases():
        assert X.dtype == np.complex64 and y.dtype == np.complex64
        assert np.array_equal(checksum(X), golden_vocal[name + '_X_sum']), name
        assert np.array_equal(checksum(y), golden_vocal[name + '_y_sum']), name


def test_vocal_oracle_equals_reference(golden_vocal):
    from oracle import dataset_image_oracle
    for name, X, y in dataset_image_oracle.vocal_cases():
        img = dataset_image_oracle.vocal_image(X, y)
        assert img.dtype == np.uint8 and img.shape == (X.shape[1], X.shape[2], 3)
        assert np.array_equal(img, golden_vocal[name + '_vocal']), name


def test_vocal_oracle_constant_input_is_zero():
    from oracle import dataset_image_oracle
    X = np.zeros((2, 5, 7), np.complex64)
    assert not dataset_image_oracle.vocal_image(X, X).any()


def test_importing_lib_dataset_does_not_need_cv2():
    code = 'import sys; import lib.dataset, lib.spec_utils; assert "cv2" not in sys.modules'
    subprocess.run([sys.executable, '-c', code], cwd=PKG, check=True)


def test_vocal_image_rejects_bad_inputs():
    from lib import dataset
    X = np.ones((2, 5, 7), np.complex64)
    with pytest.raises(ValueError, match='shape'):
        dataset.vocal_image(X, X[:, :, :6])
    with pytest.raises(ValueError, match='shape'):
        dataset.vocal_image(X[0], X[0])
    with pytest.raises(ValueError, match='complex'):
        dataset.vocal_image(np.abs(X), X)


# (script, arguments) of both tools; every path is relative to the working directory
SCRIPTS = [('dataset', ['mix', 'inst', 'out']), ('spec_utils', ['mix.wav', 'inst.wav'])]


def _run(tmp_path, script, args, as_module):
    """Runs lib/<script>.py in the working directory tmp_path, as a file or as ``python -m lib.<script>``."""
    env = dict(os.environ)
    if as_module:
        cmd = [sys.executable, '-m', 'lib.' + script]
        env['PYTHONPATH'] = PKG + os.pathsep + env.get('PYTHONPATH', '')
    else:
        cmd = [sys.executable, os.path.join(PKG, 'lib', script + '.py')]
    return subprocess.run(cmd + args, capture_output=True, text=True, cwd=str(tmp_path), env=env)


def _dataset_dirs(tmp_path):
    for sub, name in (('mix', 'a.wav'), ('inst', 'a.wav')):
        os.makedirs(str(tmp_path / sub))
        open(str(tmp_path / sub / name), 'wb').close()


@pytest.mark.parametrize('as_module', [False, True])
@pytest.mark.parametrize('script,args', SCRIPTS)
def test_scripts_without_gpu_fail_on_cuda_and_write_nothing(tmp_path, script, args, as_module):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    pytest.importorskip('cv2')
    _dataset_dirs(tmp_path)
    before = sorted(os.walk(str(tmp_path)))
    r = _run(tmp_path, script, args, as_module)
    assert r.returncode != 0
    assert 'RuntimeError: no CUDA device' in r.stderr, r.stderr
    assert sorted(os.walk(str(tmp_path))) == before


@pytest.mark.parametrize('as_module', [False, True])
@pytest.mark.parametrize('script,args', SCRIPTS)
def test_scripts_with_a_wrong_argument_count_print_usage(tmp_path, script, args, as_module):
    _dataset_dirs(tmp_path)
    before = sorted(os.walk(str(tmp_path)))
    for wrong in (args[:-1], args + ['extra']):
        r = _run(tmp_path, script, wrong, as_module)
        assert r.returncode == 2, (wrong, r.stderr)
        assert r.stderr.startswith('usage:'), r.stderr
        assert 'Traceback' not in r.stderr
    assert sorted(os.walk(str(tmp_path))) == before
