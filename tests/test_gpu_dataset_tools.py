"""The dataset inspection scripts on the GPU (run on an H100): vr_vocal_image against the images the reference's own
lib/dataset.py writes (tests/golden/ref_vocal_image, oracle/dataset_image_oracle.py), vr_spec_sub against numpy, and
both scripts end to end.

The GPU's |X| and numpy's may differ in the last bit, so a pixel whose scaled level lies on a truncation boundary may
move by one level: as for the --output_image images, every pixel must be within 1 level, at most 1e-4 of them may
differ, and channel 0 must be exactly the maximum of channels 1 and 2.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import PKG, load_golden, record_parity

pytestmark = pytest.mark.gpu

MAX_FRACTION = 1e-4
SR = 44100
CACHE = 'sr44100_hl1024_nf2048'


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


@pytest.fixture(scope='module')
def golden_vocal():
    return load_golden('ref_vocal_image')


def test_vocal_image_matches_reference(golden_vocal):
    from lib import dataset
    from oracle import dataset_image_oracle
    results = []
    for name, X, y in dataset_image_oracle.vocal_cases():
        img = dataset.vocal_image(X, y)
        assert isinstance(img, np.ndarray)
        results.append(_diff(img, golden_vocal[name + '_vocal']))
        d_img = dataset.vocal_image(torch.from_numpy(X).to(_dev()), torch.from_numpy(y).to(_dev()))
        assert d_img.is_cuda and np.array_equal(d_img.cpu().numpy(), img)
    n_diff = sum(r[0] for r in results)
    size = sum(r[2] for r in results)
    worst = max(r[1] for r in results)
    record_parity('vocal_image_fixture_max_level_diff', worst, 1)
    record_parity('vocal_image_fixture_fraction_of_pixels_differing', n_diff / size, MAX_FRACTION)
    assert worst <= 1 and n_diff <= MAX_FRACTION * size, (worst, n_diff, size)


def test_vocal_image_constant_and_repeatable():
    from lib import dataset, spec_utils
    from oracle import dataset_image_oracle
    silent = np.zeros((2, 1025, 50), np.complex64)
    img = dataset.vocal_image(silent, silent)
    assert img.shape == (1025, 50, 3) and not img.any()
    _, X, y = dataset_image_oracle.vocal_cases()[0]
    ctx = spec_utils._spectral_ctx(2048, 1024)
    before = ctx.launch_count()
    first = dataset.vocal_image(X, y)
    assert ctx.launch_count() - before == 2   # the range pass and the pixel pass
    assert np.array_equal(dataset.vocal_image(X, y), first)
    # the range scratch is reset per call: a constant pair right after a non-constant one is still all zero
    assert not dataset.vocal_image(X[:, :, :3], X[:, :, :3]).any()


def test_spectrogram_difference_is_numpys():
    from lib import spec_utils
    from oracle import dataset_image_oracle
    ctx = spec_utils._spectral_ctx(2048, 1024)
    for _, X, y in dataset_image_oracle.vocal_cases():
        want = (X - y).view(np.uint32)
        before = ctx.launch_count()
        got = spec_utils.spectrogram_difference(X, y)
        assert ctx.launch_count() - before == 1
        assert got.dtype == np.complex64 and np.array_equal(got.view(np.uint32), want)
        d_got = spec_utils.spectrogram_difference(torch.from_numpy(X).to(_dev()), torch.from_numpy(y).to(_dev()))
        assert d_got.is_cuda and np.array_equal(d_got.cpu().numpy().view(np.uint32), want)


def test_profile_dump_names_the_new_launches():
    from lib import dataset, spec_utils
    from oracle import dataset_image_oracle
    _, X, y = dataset_image_oracle.vocal_cases()[0]
    ctx = spec_utils._spectral_ctx(2048, 1024)
    ctx.check(ctx.lib.vr_profile_enable(ctx.handle, 1), 'vr_profile_enable')
    try:
        dataset.vocal_image(X, y)
        spec_utils.spectrogram_difference(X, y)
        need = ctypes.c_int64(0)
        ctx.check(ctx.lib.vr_profile_dump(ctx.handle, None, 0, ctypes.byref(need)), 'vr_profile_dump')
        buf = ctypes.create_string_buffer(need.value)
        ctx.check(ctx.lib.vr_profile_dump(ctx.handle, buf, need.value, None), 'vr_profile_dump')
    finally:
        ctx.check(ctx.lib.vr_profile_enable(ctx.handle, 0), 'vr_profile_enable')
    names = [ln.split()[0] for ln in buf.value.decode().splitlines()]
    assert names[-2:] == ['vocal_image', 'spec_sub'], names


def _write_pair(mix_path, inst_path, seed, delay):
    """A 6 s synthetic mixture and its instrumental: the mixture delayed by ``delay`` samples, with one second
    muted to 5%, so that the pair has a vocal residual there."""
    from lib import audio_io, synth
    mix = synth.sine_mix(6.0, seed=seed)
    inst = np.concatenate([np.zeros((2, delay), np.float32), mix], axis=1)
    inst[:, delay + 2 * SR:delay + 3 * SR] *= np.float32(0.05)
    audio_io.write(mix_path, mix.T, SR)
    audio_io.write(inst_path, inst.T, SR)


def _run(cwd, script, args, as_module=False, env=None):
    full_env = dict(os.environ, **(env or {}))
    if as_module:
        cmd = [sys.executable, '-m', 'lib.' + script]
        full_env['PYTHONPATH'] = PKG + os.pathsep + full_env.get('PYTHONPATH', '')
    else:
        cmd = [sys.executable, os.path.join(PKG, 'lib', script + '.py')]
    r = subprocess.run(cmd + list(args), capture_output=True, text=True, cwd=str(cwd), env=full_env)
    assert r.returncode == 0, r.stderr
    return r.stdout


def _read(path):
    with open(path, 'rb') as f:
        return f.read()


def _decoded(cv2, path_or_img):
    if isinstance(path_or_img, str):
        return cv2.imdecode(np.fromfile(path_or_img, np.uint8), cv2.IMREAD_COLOR)
    return cv2.imdecode(cv2.imencode('.jpg', path_or_img)[1], cv2.IMREAD_COLOR)


@pytest.fixture(scope='module')
def dataset_dirs(tmp_path_factory):
    root = tmp_path_factory.mktemp('pairs')
    for d in ('mix', 'inst'):
        os.makedirs(str(root / d))
    for k, (name, delay) in enumerate((('a', 1500), ('b', 300))):
        _write_pair(str(root / 'mix' / (name + '.wav')), str(root / 'inst' / (name + '.wav')), k, delay)
    return root


def test_vocal_jpg_tool(dataset_dirs, tmp_path):
    cv2 = pytest.importorskip('cv2')
    from lib import dataset, spec_utils
    root = dataset_dirs
    mix_dir, inst_dir = str(root / 'mix'), str(root / 'inst')
    out = str(tmp_path / 'out' / 'nested')
    assert not os.path.exists(os.path.join(mix_dir, CACHE))
    _run(tmp_path, 'dataset', [mix_dir, inst_dir, out])
    assert sorted(os.listdir(out)) == ['a_Vocal.jpg', 'b_Vocal.jpg']
    caches = [os.path.join(d, CACHE, n + '.npy') for d in (mix_dir, inst_dir) for n in ('a', 'b')]
    assert all(os.path.isfile(c) for c in caches)
    for d in (mix_dir, inst_dir):
        assert sorted(os.listdir(os.path.join(d, CACHE))) == ['a.npy', 'b.npy']
    mtimes = [os.stat(c).st_mtime_ns for c in caches]
    first = {n: _read(os.path.join(out, n)) for n in os.listdir(out)}

    # a second run hits the caches and writes the same bytes; so does the module form
    _run(tmp_path, 'dataset', [mix_dir, inst_dir, out])
    assert [os.stat(c).st_mtime_ns for c in caches] == mtimes
    assert {n: _read(os.path.join(out, n)) for n in os.listdir(out)} == first
    out_m = str(tmp_path / 'out_module')
    _run(PKG, 'dataset', [mix_dir, inst_dir, out_m], as_module=True)
    assert {n: _read(os.path.join(out_m, n)) for n in os.listdir(out_m)} == first

    for name in ('a', 'b'):
        X, y, _, _ = spec_utils.cache_or_load(os.path.join(mix_dir, name + '.wav'),
                                              os.path.join(inst_dir, name + '.wav'), SR, 1024, 2048)
        img = dataset.vocal_image(X, y)
        assert img.any()
        assert np.array_equal(_decoded(cv2, os.path.join(out, name + '_Vocal.jpg')), _decoded(cv2, img)), name


def test_vocal_jpg_tool_shards_over_ranks(dataset_dirs, tmp_path):
    pytest.importorskip('cv2')
    out = str(tmp_path / 'rank1')
    _run(tmp_path, 'dataset', [str(dataset_dirs / 'mix'), str(dataset_dirs / 'inst'), out],
         env={'WORLD_SIZE': '2', 'RANK': '1', 'LOCAL_RANK': '0'})
    assert os.listdir(out) == ['b_Vocal.jpg']


def test_vocal_jpg_tool_skips_pairs_wider_than_jpeg_allows(tmp_path):
    """65501 frames: JPEG cannot encode the image, so, as with the reference, there is no JPG.  The pair is given as
    its caches (3 bins keep them small), which the tool reads without decoding the placeholder WAVs."""
    pytest.importorskip('cv2')
    for d in ('mix', 'inst'):
        os.makedirs(str(tmp_path / d / CACHE))
        open(str(tmp_path / d / 'long.wav'), 'wb').close()
        np.save(str(tmp_path / d / CACHE / 'long.npy'), np.ones((65501, 2, 3), np.complex64))
    out = str(tmp_path / 'out')
    stdout = _run(tmp_path, 'dataset', [str(tmp_path / 'mix'), str(tmp_path / 'inst'), out])
    assert os.listdir(out) == []
    assert 'skipping {}/long_Vocal.jpg: 65501 frames'.format(out) in stdout


def test_pair_check(dataset_dirs, tmp_path):
    cv2 = pytest.importorskip('cv2')
    from lib import audio_io, spec_utils
    mix, inst = str(dataset_dirs / 'mix' / 'a.wav'), str(dataset_dirs / 'inst' / 'a.wav')
    run_dir = tmp_path / 'file'
    os.makedirs(str(run_dir))
    _run(run_dir, 'spec_utils', [mix, inst])
    names = ['test_%s.%s' % (s, e) for s in ('X', 'v', 'y') for e in ('jpg', 'wav')]
    assert sorted(os.listdir(str(run_dir))) == names
    module_dir = tmp_path / 'module'
    os.makedirs(str(module_dir))
    _run(module_dir, 'spec_utils', [mix, inst], as_module=True)
    for n in names:
        assert _read(str(run_dir / n)) == _read(str(module_dir / n)), n

    X, _ = audio_io.load(mix, sr=SR, mono=False, dtype=np.float32, device=0)
    y, _ = audio_io.load(inst, sr=SR, mono=False, dtype=np.float32, device=0)
    X, y = spec_utils.align_wave_head_and_tail(X, y, SR)
    X_spec = spec_utils.wave_to_spectrogram(X, 1024, 2048)
    y_spec = spec_utils.wave_to_spectrogram(y, 1024, 2048)
    specs = {'X': X_spec, 'y': y_spec, 'v': X_spec - y_spec}
    for s, spec in specs.items():
        want = str(tmp_path / ('want_%s.wav' % s))
        audio_io.write(want, spec_utils.spectrogram_to_wave(spec).T, SR)
        assert _read(str(run_dir / ('test_%s.wav' % s))) == _read(want), s
        assert np.array_equal(_decoded(cv2, str(run_dir / ('test_%s.jpg' % s))),
                              _decoded(cv2, spec_utils.spectrogram_to_image(spec))), s
