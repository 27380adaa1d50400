"""evaluate.py --oracle on the GPU (run on an H100): vr_oracle_mask bit for bit against the float64 restatement
(tests/oracle_masks.py), the oracle stems against a numpy chain, the oracle MWF against tests/wiener_oracle.py, closed
forms end to end, and the command line against direct calls, on a tree with no checkpoint.

Gates:
- the masks: bitwise equality, since the arithmetic is pinned;
- the mask oracles' stems against oracle STFT -> restated mask -> separator_oracle.apply_mask -> oracle inverse STFT:
  5e-6, the gate of the STFT and inverse STFT parity tests (tests/test_gpu_parity.py), on waves of peak below 1.  The
  binary mask may decide a bin the other way only where the oracle's spectrograms are within the STFT gate of a tie;
  such bins take the GPU's decision in the chain;
- the oracle MWF: 1e-5 of max|X|, the gate of the Wiener filter tests (tests/test_gpu_wiener.py).
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle_masks as om
import wiener_oracle as wo
from conftest import PKG, record_parity
from test_oracle_host import disjoint_pair

pytestmark = pytest.mark.gpu

SR = 44100
STFT_GATE = 5e-6
WIENER_GATE = 1e-5


def _dev():
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    return torch.device('cuda:0')


def _pair(seconds, seed):
    from lib import synth
    inst = 0.4 * synth.sine_mix(seconds, seed=seed)
    voc = 0.4 * synth.sine_mix(seconds / 2, sr=2 * SR, seed=seed + 10)[:, :inst.shape[1]]
    return (inst + voc).astype(np.float32), inst.astype(np.float32)


@pytest.fixture(scope='module')
def pair10():
    return _pair(10.0, 10)


@pytest.fixture(scope='module')
def specs10(pair10):
    from lib import spec_utils
    _dev()
    return tuple(spec_utils.wave_to_spectrogram(w, 1024, 2048) for w in pair10)


def _noise(shape, seed, gain=1.0):
    rng = np.random.default_rng(seed)
    return (gain * (rng.standard_normal(shape) + 1j * rng.standard_normal(shape))).astype(np.complex64)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def test_mask_is_bitwise_the_restatement(specs10):
    from lib import spec_utils
    cases = {'pair10': specs10}
    for T in (1, 2, 37, 1000):
        X = _noise((2, 1025, T), T, 20.0)
        Y = _noise((2, 1025, T), T + 1, 15.0)
        Y[:, :, :T // 3] = X[:, :, :T // 3]
        cases['noise_T%d' % T] = (X, Y)
    Z = np.zeros((2, 1025, 40), np.complex64)
    y = _noise((2, 1025, 40), 3)
    cases.update(silence=(Z, Z), equal=((2 * y).astype(np.complex64), y), instruments_silent=(y, Z),
                 opposite=(Z, y))
    for name, (X, Y) in cases.items():
        for kind in om.KINDS:
            got = spec_utils.oracle_mask(X, Y, kind)
            want = om.mask(X, Y, kind)
            assert got.dtype == np.float32 and got.shape == X.shape
            assert np.array_equal(_bits(got), _bits(want)), (name, kind, int((got != want).sum()))
            assert np.array_equal(_bits(spec_utils.oracle_mask(X, Y, kind)), _bits(got)), (name, kind)
    X, Y = cases['equal']
    for kind in ('iam', 'irm1', 'irm2'):
        assert np.all(spec_utils.oracle_mask(X, Y, kind) == 0.5)
    # CUDA tensors in, a CUDA tensor out; the inputs are untouched
    dX, dY = (torch.from_numpy(a).to(_dev()) for a in specs10)
    for kind in om.KINDS:
        m = spec_utils.oracle_mask(dX, dY, kind)
        assert m.is_cuda and np.array_equal(m.cpu().numpy(), om.mask(*specs10, kind))
    assert np.array_equal(dX.cpu().numpy(), specs10[0]) and np.array_equal(dY.cpu().numpy(), specs10[1])


def test_mask_errors():
    from lib import _native, spec_utils
    ctx = spec_utils._spectral_ctx(2048, 1024)
    d = torch.zeros((2, 1025, 4), dtype=torch.complex64, device=_dev())
    m = torch.empty((2, 1025, 4), dtype=torch.float32, device=_dev())
    p, q = _native.ptr(d), _native.ptr(m)
    for args in ((p, p, 4, 4, q), (p, p, 4, -1, q), (p, p, 0, 0, q), (None, p, 4, 0, q), (p, None, 4, 0, q),
                 (p, p, 4, 0, None)):
        rc = ctx.lib.vr_oracle_mask(ctx.handle, *args, _native.stream_ptr())
        assert rc != 0 and b'oracle_mask' in ctx.lib.vr_last_error(ctx.handle)


def _chain_stems(X, y, kind, gpu_specs):
    """Oracle STFT -> restated mask -> separator_oracle.apply_mask -> oracle inverse STFT.  For ibm, a bin whose
    decision differs from the GPU's must be within the STFT gate of a tie; it takes the GPU's decision."""
    from oracle import separator_oracle, stft_oracle
    Xo, Yo = (stft_oracle.wave_to_spectrogram(w, 1024, 2048) for w in (X, y))
    m = om.mask(Xo, Yo, kind)
    flips = 0
    if kind == 'ibm':
        m_gpu = om.mask(*gpu_specs, 'ibm')
        diff = m != m_gpu
        flips = int(diff.sum())
        margin = np.abs(np.abs(Yo) - np.abs(Xo - Yo))
        assert np.all(margin[diff] <= 2 * STFT_GATE * np.abs(Xo).max())
        m = np.where(diff, m_gpu, m)
    ys, vs = separator_oracle.apply_mask(Xo, m)
    return [stft_oracle.spectrogram_to_wave(s, 1024) for s in (ys, vs)], flips


@pytest.mark.parametrize('kind', om.KINDS)
def test_mask_oracle_stems_match_the_numpy_chain(pair10, specs10, kind):
    from lib import spec_utils
    X, y = pair10
    got = spec_utils.oracle_separate_wave(X, y, kind, 2048, 1024)
    want, flips = _chain_stems(X, y, kind, specs10)
    assert all(g.shape == w.shape == (2, 1024 * (X.shape[1] // 1024)) for g, w in zip(got, want))
    err = max(float(np.abs(g - w).max()) for g, w in zip(got, want))
    record_parity('oracle_%s_stems_10s_vs_numpy_chain' % kind, err, STFT_GATE)
    if kind == 'ibm':
        print('ibm: %d bins decided by the GPU within the STFT gate of a tie' % flips)
    assert err <= STFT_GATE
    # the device path gives the same stems
    d = [torch.from_numpy(w).to(_dev()) for w in (X, y)]
    on_dev = spec_utils.oracle_separate_wave(d[0], d[1], kind, 2048, 1024)
    assert all(t.is_cuda and np.array_equal(t.cpu().numpy(), g) for t, g in zip(on_dev, got))


def test_mwf_matches_the_wiener_oracle(pair10, specs10):
    from lib import spec_utils
    Xs, Ys = specs10
    Vs = spec_utils.spectrogram_difference(Xs, Ys)
    want = wo.wiener(Xs, Ys, Vs, 1, round32=True)
    got = spec_utils.oracle_spectrograms(Xs, Ys, 'mwf')
    err = max(float(np.abs(g.astype(np.complex128) - w).max()) for g, w in zip(got, want)) / float(np.abs(Xs).max())
    record_parity('oracle_mwf_10s_over_max_abs_X', err, WIENER_GATE)
    assert err <= WIENER_GATE
    # the stems are the inverse STFTs of those spectrograms
    stems = spec_utils.oracle_separate_wave(*pair10, 'mwf', 2048, 1024)
    for w, s in zip(stems, got):
        assert np.array_equal(w, spec_utils.spectrogram_to_wave(s, 1024))
    # and differ from the ratio mask's
    irm = spec_utils.oracle_separate_wave(*pair10, 'irm2', 2048, 1024)
    assert np.abs(stems[1] - irm[1]).max() > 1e-4


def test_closed_forms_end_to_end():
    from lib import spec_utils, synth
    # y = v: the GPU's spectrograms give X = 2Y exactly, so the masks are exactly 0.5 under iam, irm1 and irm2 and
    # both stems are istft(0.5 X); ibm gives everything to the instruments.  The masked inverse STFT transforms both
    # stems in one complex FFT (instruments real, vocals imaginary), so the two agree to its rounding, not bit for bit.
    y = (0.4 * synth.sine_mix(4.0, seed=30)).astype(np.float32)
    X = (2 * y).astype(np.float32)
    Xs, Ys = (spec_utils.wave_to_spectrogram(w, 1024, 2048) for w in (X, y))
    assert np.array_equal(Xs, 2 * Ys)
    half = spec_utils.spectrogram_to_wave((0.5 * Xs).astype(np.complex64), 1024)
    for kind in ('iam', 'irm1', 'irm2'):
        assert np.all(spec_utils.oracle_mask(Xs, Ys, kind) == 0.5), kind
        inst, voc = spec_utils.oracle_separate_wave(X, y, kind, 2048, 1024)
        err = max(float(np.abs(inst - half).max()), float(np.abs(voc - half).max()))
        record_parity('oracle_%s_equal_sources_vs_istft_half_X' % kind, err, STFT_GATE)
        assert err <= STFT_GATE
    assert np.all(spec_utils.oracle_mask(Xs, Ys, 'ibm') == 1.0)
    inst, voc = spec_utils.oracle_separate_wave(X, y, 'ibm', 2048, 1024)
    err = max(float(np.abs(inst - spec_utils.spectrogram_to_wave(Xs, 1024)).max()), float(np.abs(voc).max()))
    record_parity('oracle_ibm_equal_sources_vs_istft_X', err, STFT_GATE)
    assert err <= STFT_GATE

    # time-disjoint sources: every mask is 1 or 0 on the frames one source reaches, so the estimates are the references
    # up to the STFT round trip
    X, y, _, _ = disjoint_pair()
    v = X - y
    for kind in om.KINDS:
        inst, voc = spec_utils.oracle_separate_wave(X, y, kind, 2048, 1024)
        n = inst.shape[1]
        keep = slice(2048, n - 2048)
        err = max(float(np.abs(inst[:, keep] - y[:, keep]).max()), float(np.abs(voc[:, keep] - v[:, keep]).max()))
        record_parity('oracle_%s_disjoint_sources_vs_references' % kind, err, STFT_GATE)
        assert err <= STFT_GATE, kind


# ---- evaluate.py --oracle -----------------------------------------------------------------------------------------
def _write_pairs(root, count=2, seconds=5.0):
    from lib import audio_io
    pairs = []
    for k in range(count):
        X, y = _pair(seconds, 40 + k)
        pair = []
        for kind, w in (('mixtures', X), ('instruments', y)):
            d = os.path.join(root, kind)
            os.makedirs(d, exist_ok=True)
            path = os.path.join(d, 'track%d.wav' % k)
            audio_io.write(path, w.T, SR)
            pair.append(path)
        pairs.append(pair)
    return pairs


def _cli(cwd, *args):
    r = subprocess.run([sys.executable, os.path.join(PKG, 'evaluate.py'), '-g', '0'] + list(args),
                       capture_output=True, text=True, cwd=cwd)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    pairs = [l for l in lines if re.match(r'\d+ \S+\.wav \S+\.wav instruments SDR ', l)]
    assert lines[-1].startswith('median of %d pairs: ' % len(pairs)), r.stdout
    assert 'loading model' not in r.stdout
    return pairs, lines[-1]


def _expect(filelist, oracle, framewise=False, wiener_iterations=0):
    """The lines evaluate.py prints, formatted from direct calls of score_oracle_pair."""
    import evaluate
    import validate
    from lib import bsseval
    results = []
    for X_path, y_path in filelist:
        X, y = evaluate.pair_waves(X_path, y_path, SR, 0)
        results.append(evaluate.score_oracle_pair(oracle, X, y, 2048, 1024, SR, SR, 512, framewise, wiener_iterations))
    return (['{} {} {}'.format(i + 1, validate.pair_name(*pair), evaluate.format_values(bsseval.track_medians(r)))
             for i, (pair, r) in enumerate(zip(filelist, results))],
            'median of {} pairs: {}'.format(len(results), evaluate.format_values(evaluate.dataset_medians(results))))


def test_cli_without_a_checkpoint(tmp_path):
    from lib import spec_utils
    _dev()
    root = str(tmp_path / 'data')
    pairs = _write_pairs(root)
    assert not [f for _, _, files in os.walk(str(tmp_path)) for f in files if f.endswith('.pth')]
    cwd = str(tmp_path)
    seen = {}
    for kind in spec_utils.ORACLES:
        js = str(tmp_path / ('%s.json' % kind))
        got = _cli(cwd, '-d', root, '--all', '--oracle', kind, '--json', js)
        assert got == _expect(pairs, oracle=kind), kind
        with open(js) as f:
            doc = json.load(f)
        assert doc['oracle'] == kind and 'wiener_iterations' not in doc and 'framewise_filters' not in doc
        seen[kind] = got[1]
    assert len(set(seen.values())) == len(seen)   # five different separations
    print('\n'.join('%s: %s' % kv for kv in seen.items()))

    got = _cli(cwd, '-d', root, '--all', '--oracle', 'irm1', '--framewise_filters')
    assert got == _expect(pairs, oracle='irm1', framewise=True)
    assert got[1] != seen['irm1']

    js = str(tmp_path / 'iam_wiener.json')
    got = _cli(cwd, '-d', root, '--all', '--oracle', 'iam', '--wiener_iterations', '2', '--json', js)
    assert got == _expect(pairs, oracle='iam', wiener_iterations=2)
    with open(js) as f:
        doc = json.load(f)
    assert doc['oracle'] == 'iam' and doc['wiener_iterations'] == 2
    assert not [f for _, _, files in os.walk(str(tmp_path)) for f in files if f.endswith('.pth')]


def test_iam_with_wiener_is_the_filtered_masked_stems(pair10):
    """oracle iam + 2 Wiener iterations = spec_utils.wiener applied to the iam-masked spectrograms, then inverted."""
    from lib import spec_utils
    X, y = pair10
    Xs, Ys = (spec_utils.wave_to_spectrogram(w, 1024, 2048) for w in (X, y))
    y0, v0 = spec_utils.oracle_spectrograms(Xs, Ys, 'iam')
    m = spec_utils.oracle_mask(Xs, Ys, 'iam')
    assert np.abs(y0 - m * Xs).max() <= 1e-6 * np.abs(Xs).max()
    want = [spec_utils.spectrogram_to_wave(s, 1024) for s in spec_utils.wiener(Xs, y0, v0, 2)]
    got = spec_utils.oracle_separate_wave(X, y, 'iam', 2048, 1024, wiener_iterations=2)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    plain = spec_utils.oracle_separate_wave(X, y, 'iam', 2048, 1024)
    assert np.abs(plain[1] - got[1]).max() > 1e-4
