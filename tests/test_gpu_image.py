"""--output_image on the GPU (run on an H100): vr_spec_image against the reference's own images
(tests/golden/ref_image, oracle/image_oracle.py), the images of Separator.separate_wave(images=True) against the oracle
image of the stems Separator.separate[_tta] returns, and the CLI's JPGs.

The GPU's |X| and the reference's |m |X| e^{j angle X}| differ in the last bit, so a pixel whose scaled level lies on
a truncation boundary may move by one level: every pixel must be within 1 level, at most 1e-4 of them may differ, and
channel 0 must be exactly the maximum of channels 1 and 2.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import PKG, load_golden, record_parity

pytestmark = pytest.mark.gpu

MAX_FRACTION = 1e-4


def _dev():
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    return torch.device('cuda:0')


def _diff(got, ref):
    """(pixels differing, max level difference, pixels) after checking shape, dtype and the max channel."""
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    assert got.dtype == np.uint8 and got.shape == ref.shape, (got.dtype, got.shape, ref.shape)
    assert np.array_equal(got[..., 0], got[..., 1:].max(axis=-1))
    d = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    return int((d > 0).sum()), int(d.max()), d.size


def _gate(name, results):
    n_diff = sum(r[0] for r in results)
    size = sum(r[2] for r in results)
    worst = max(r[1] for r in results)
    record_parity('image_%s_max_level_diff' % name, worst, 1)
    record_parity('image_%s_fraction_of_pixels_differing' % name, n_diff / size, MAX_FRACTION)
    assert worst <= 1 and n_diff <= MAX_FRACTION * size, (worst, n_diff, size)


@pytest.fixture(scope='module')
def golden_image():
    return load_golden('ref_image')


@pytest.fixture(scope='module')
def default_model():
    from lib import nets, synth
    m = nets.CascadedNet(2048, 1024, 32, 128)
    m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    m.to(_dev())
    return m


@pytest.fixture(scope='module')
def wave10():
    from lib import synth
    return synth.sine_mix(10.0)


def _spec_image(ctx, X, m):
    from lib import _native
    d_spec = torch.from_numpy(X).cuda()
    d_mask = torch.from_numpy(m).cuda()
    a = torch.empty((X.shape[1], X.shape[2], 3), dtype=torch.uint8, device='cuda')
    b = torch.empty_like(a)
    ctx.check(ctx.lib.vr_spec_image(ctx.handle, _native.ptr(d_spec), _native.ptr(d_mask), X.shape[2], _native.ptr(a),
                                    _native.ptr(b), _native.stream_ptr()), 'vr_spec_image')
    return a.cpu().numpy(), b.cpu().numpy()


def test_spec_image_matches_reference(golden_image):
    from lib import spec_utils
    from oracle import image_oracle, separator_oracle
    g = golden_image
    results = []
    for name, X, m in image_oracle.image_cases():
        if m is None:
            img = spec_utils.spectrogram_to_image(X)
            assert isinstance(img, np.ndarray)
            results.append(_diff(img, g[name + '_X']))
            d_img = spec_utils.spectrogram_to_image(torch.from_numpy(X).cuda())
            assert d_img.is_cuda and np.array_equal(d_img.cpu().numpy(), img)
            continue
        a, b = _spec_image(spec_utils._spectral_ctx(2 * (X.shape[1] - 1), X.shape[1] - 1), X, m)
        results += [_diff(a, g[name + '_inst']), _diff(b, g[name + '_voc'])]
        y, _ = separator_oracle.apply_mask(X, m)   # the reference's y_spec, through the public function
        results.append(_diff(spec_utils.spectrogram_to_image(y.astype(np.complex64)), g[name + '_inst']))
    _gate('fixture_vs_reference', results)


def test_spec_image_constant_and_repeatable(golden_image):
    from lib import spec_utils
    from oracle import image_oracle
    img = spec_utils.spectrogram_to_image(np.zeros((2, 1025, 50), np.complex64))
    assert img.shape == (1025, 50, 3) and not img.any()
    _, X, m = image_oracle.image_cases()[0]
    ctx = spec_utils._spectral_ctx(2048, 1024)
    first = _spec_image(ctx, X, m)
    second = _spec_image(ctx, X, m)
    assert all(np.array_equal(p, q) for p, q in zip(first, second))
    # the range scratch is reset per call: a constant spectrogram right after a non-constant one is still all zero
    a, b = _spec_image(ctx, np.zeros((2, 1025, 3), np.complex64), np.full((2, 1025, 3), 0.5, np.float32))
    assert not a.any() and not b.any()


@pytest.mark.parametrize('postprocess', [False, True])
@pytest.mark.parametrize('tta', [False, True])
def test_separate_wave_images(default_model, wave10, tta, postprocess):
    import inference
    from lib import spec_utils
    from oracle import image_oracle
    sp = inference.Separator(default_model, _dev(), 4, 256, postprocess)
    y, v = (sp.separate_tta if tta else sp.separate)(spec_utils.wave_to_spectrogram(wave10, 1024, 2048))
    ref_inst, ref_voc = image_oracle.spectrogram_to_image(y), image_oracle.spectrogram_to_image(v)
    results = []
    for wave in (wave10, torch.from_numpy(wave10).cuda()):
        inst, voc = sp.separate_wave(wave, tta=tta)
        out = sp.separate_wave(wave, tta=tta, images=True)
        assert len(out) == 4
        if torch.is_tensor(wave):
            assert all(t.is_cuda for t in out)
            inst, voc = inst.cpu().numpy(), voc.cpu().numpy()
            out = [t.cpu().numpy() for t in out]
        assert np.array_equal(out[0], inst) and np.array_equal(out[1], voc)
        results += [_diff(out[2], ref_inst), _diff(out[3], ref_voc)]
    _gate('separate_wave_tta%d_postprocess%d_vs_oracle' % (tta, postprocess), results)


def _cli(src, ckpt, out_dir, *extra):
    r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt, '-i', src,
                        '-o', out_dir] + list(extra), capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 0, r.stderr
    return sorted(os.listdir(out_dir)), r.stdout


def test_cli_writes_the_jpgs(default_model, wave10, tmp_path):
    import inference
    from lib import audio_io, synth
    src = str(tmp_path / 'mix.wav')
    audio_io.write(src, wave10.T, 44100)
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
    plain, with_images = str(tmp_path / 'plain'), str(tmp_path / 'images')
    assert _cli(src, ckpt, plain)[0] == ['mix_Instruments.wav', 'mix_Vocals.wav']
    cv2 = pytest.importorskip('cv2')
    assert _cli(src, ckpt, with_images, '-I')[0] == ['mix_Instruments.jpg', 'mix_Instruments.wav', 'mix_Vocals.jpg',
                                                     'mix_Vocals.wav']
    for stem in ('Instruments', 'Vocals'):
        with open(os.path.join(plain, 'mix_%s.wav' % stem), 'rb') as a, \
                open(os.path.join(with_images, 'mix_%s.wav' % stem), 'rb') as b:
            assert a.read() == b.read(), stem
    X, _ = audio_io.load(src, sr=44100, mono=False, dtype=np.float32, device=_dev())
    _, _, img_inst, img_voc = inference.Separator(default_model, _dev(), 4, 256, False).separate_wave(X, images=True)
    for stem, img in (('Instruments', img_inst), ('Vocals', img_voc)):
        got = cv2.imdecode(np.fromfile(os.path.join(with_images, 'mix_%s.jpg' % stem), np.uint8), cv2.IMREAD_COLOR)
        want = cv2.imdecode(cv2.imencode('.jpg', img)[1], cv2.IMREAD_COLOR)
        assert np.array_equal(got, want), stem


def test_cli_skips_jpgs_wider_than_jpeg_allows(tmp_path):
    """65501 frames (n_fft 512, hop 128 keep the track at 190 s): JPEG cannot encode the image, so, as with the
    reference, there is no JPG and the CLI still writes both stems and exits normally."""
    pytest.importorskip('cv2')
    from lib import audio_io, synth
    L = 65500 * 128
    src = str(tmp_path / 'long.wav')
    audio_io.write(src, synth.sine_mix(L / 44100.0 + 0.1)[:, :L].T, 44100)
    ckpt = str(tmp_path / 'synthetic512.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict(512, 32, 128)), ckpt)
    files, stdout = _cli(src, ckpt, str(tmp_path / 'out'), '-I', '-f', '512', '-H', '128')
    assert files == ['long_Instruments.wav', 'long_Vocals.wav']
    assert 'skipping long_Instruments.jpg and long_Vocals.jpg: 65501 frames' in stdout
