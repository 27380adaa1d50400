"""--output_image without a GPU: the numpy image oracle against the reference's own images, the JPG helpers of
lib/utils.py, the unsupported spectrogram_to_image inputs and the CLI's failure order."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import PKG, checksum, load_golden


@pytest.fixture(scope='module')
def golden_image():
    return load_golden('ref_image')


def test_image_oracle_equals_reference(golden_image):
    from oracle import image_oracle, separator_oracle
    g = golden_image
    for name, X, m in image_oracle.image_cases():
        assert np.array_equal(checksum(X), g[name + '_X_sum']), name   # the seeded inputs regenerate bit for bit
        if m is None:
            assert np.array_equal(image_oracle.spectrogram_to_image(X), g[name + '_X']), name
            continue
        assert np.array_equal(checksum(m), g[name + '_mask_sum']), name
        y, v = separator_oracle.apply_mask(X, m)
        for stem, s in (('inst', y), ('voc', v)):
            img = image_oracle.spectrogram_to_image(s)
            assert img.dtype == np.uint8 and img.shape == (X.shape[1], X.shape[2], 3)
            assert np.array_equal(img, g[name + '_' + stem]), (name, stem)


def test_image_oracle_constant_input_is_zero():
    from oracle import image_oracle
    img = image_oracle.spectrogram_to_image(np.zeros((2, 5, 7), np.complex64))
    assert img.shape == (5, 7, 3) and not img.any()


def test_spectrogram_to_image_rejects_unsupported_inputs():
    from lib import spec_utils
    X = np.ones((2, 5, 7), np.complex64)
    with pytest.raises(NotImplementedError, match='magnitude'):
        spec_utils.spectrogram_to_image(X, mode='phase')
    with pytest.raises(NotImplementedError, match='complex'):
        spec_utils.spectrogram_to_image(np.abs(X))
    with pytest.raises(NotImplementedError, match='stereo'):
        spec_utils.spectrogram_to_image(X[0])


def test_importing_lib_does_not_need_cv2():
    code = 'import sys; from lib import utils, spec_utils; import inference; assert "cv2" not in sys.modules'
    subprocess.run([sys.executable, '-c', code], cwd=PKG, check=True)


def test_imwrite_imread(tmp_path):
    pytest.importorskip('cv2')
    from lib import utils
    img = np.random.default_rng(0).integers(0, 256, size=(40, 70, 3), dtype=np.uint8)
    path = str(tmp_path / 'a.jpg')
    assert utils.imwrite(path, img) is True
    back = utils.imread(path)
    assert back.shape == img.shape and back.dtype == np.uint8
    # failures are return values, never exceptions, and leave no file
    missing = str(tmp_path / 'no_such_dir' / 'a.jpg')
    assert utils.imwrite(missing, img) is False
    assert not os.path.exists(os.path.dirname(missing))
    wide = str(tmp_path / 'wide.jpg')
    assert utils.imwrite(wide, np.zeros((2, 65501, 3), np.uint8)) is False
    assert not os.path.exists(wide)
    assert utils.imread(str(tmp_path / 'absent.jpg')) is None


def test_cli_output_image_without_gpu_fails_on_cuda(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    pytest.importorskip('cv2')
    out = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-i', str(tmp_path / 'x.wav'), '-I'],
                         capture_output=True, text=True, cwd=PKG)
    assert out.returncode != 0
    assert 'RuntimeError: no CUDA device' in out.stderr and 'NotImplementedError' not in out.stderr
