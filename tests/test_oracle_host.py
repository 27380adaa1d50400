"""evaluate.py --oracle without a GPU: the float64 restatement of the oracle masks (tests/oracle_masks.py) on closed
forms and on time-disjoint sources through the oracle STFT, and the command line's errors, which all come before any
GPU work."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_masks as om
from conftest import PKG

KINDS = om.KINDS


def _noise_spec(shape, seed, gain=1.0):
    rng = np.random.default_rng(seed)
    return (gain * (rng.standard_normal(shape) + 1j * rng.standard_normal(shape))).astype(np.complex64)


def test_equal_sources():
    """y = v, so X = 2y: iam, irm1 and irm2 are exactly 0.5 and ibm is 1 (the tie goes to the instruments)."""
    y = _noise_spec((2, 1025, 50), 1)
    X = (2 * y).astype(np.complex64)
    assert np.array_equal(X - y, y)
    for kind in ('iam', 'irm1', 'irm2'):
        assert np.all(om.mask(X, y, kind) == 0.5), kind
    assert np.all(om.mask(X, y, 'ibm') == 1.0)


def test_silent_instruments():
    X = _noise_spec((2, 1025, 50), 2)
    y = np.zeros_like(X)
    for kind in KINDS:
        assert np.all(om.mask(X, y, kind) == 0.0), kind


def test_opposite_sources():
    """y = -v, so X = 0 with |Y| = |V| > 0: iam is 1 (0/0 goes to the instruments), both irm masks 0.5, ibm 1."""
    y = _noise_spec((2, 1025, 50), 3)
    X = np.zeros_like(y)
    assert np.all(om.mask(X, y, 'iam') == 1.0)
    assert np.all(om.mask(X, y, 'irm1') == 0.5) and np.all(om.mask(X, y, 'irm2') == 0.5)
    assert np.all(om.mask(X, y, 'ibm') == 1.0)


def test_ranges_and_silence():
    X = _noise_spec((2, 1025, 80), 4, 10.0)
    y = _noise_spec((2, 1025, 80), 5, 7.0)
    y[:, :, :20] = X[:, :, :20]   # some instruments louder than the mixture, some equal to it
    y[:, :, 20:30] = 2 * X[:, :, 20:30]
    for kind in KINDS:
        m = om.mask(X, y, kind)
        assert m.dtype == np.float32 and m.shape == X.shape
        assert np.all((m >= 0) & (m <= 1)), kind
        assert np.all(m[:, :, :20] == 1.0), kind   # Y = X: V = 0
    assert set(np.unique(om.mask(X, y, 'ibm'))) == {0.0, 1.0}
    assert np.all(om.mask(X, y, 'iam')[:, :, 20:30] == 1.0)   # |Y| > |X|: clipped
    Z = np.zeros_like(X)
    assert np.all(om.mask(Z, Z, 'iam') == 1.0) and np.all(om.mask(Z, Z, 'ibm') == 1.0)
    assert np.all(om.mask(Z, Z, 'irm1') == 0.5) and np.all(om.mask(Z, Z, 'irm2') == 0.5)


def test_literal_definitions():
    """The vectorised restatement against a per-element loop in Python floats (IEEE doubles)."""
    import math
    X = _noise_spec((2, 7, 9), 6)
    y = _noise_spec((2, 7, 9), 7)
    y[0, 0, :3] = 0
    X[1, 1, :2] = y[1, 1, :2]
    X[1, 2, :2] = 0
    for kind in KINDS:
        got = om.mask(X, y, kind)
        for idx in np.ndindex(X.shape):
            x, t = complex(X[idx]), complex(y[idx])
            v = complex(float(np.float32(X[idx].real) - np.float32(y[idx].real)),
                        float(np.float32(X[idx].imag) - np.float32(y[idx].imag)))
            pX, pY, pV = (z.real * z.real + z.imag * z.imag for z in (x, t, v))
            if kind == 'iam':
                want = 1.0 if pY >= pX else math.sqrt(pY) / math.sqrt(pX)
            elif kind == 'ibm':
                want = 1.0 if pY >= pV else 0.0
            elif kind == 'irm1':
                s = math.sqrt(pY) + math.sqrt(pV)
                want = 0.5 if s == 0 else math.sqrt(pY) / s
            else:
                want = 0.5 if pY + pV == 0 else pY / (pY + pV)
            assert got[idx] == np.float32(want), (kind, idx)


def disjoint_pair(sr=44100, n_fft=2048, seed=8):
    """Instruments, then a gap longer than n_fft, then vocals: (X, y, inst_end, voc_start), float32 (2, L) waves."""
    from lib import synth
    n = sr * 2
    gap = n_fft + 3000
    inst = 0.4 * synth.sine_mix(2.0, seed=seed)
    voc = 0.4 * synth.sine_mix(1.0, sr=2 * sr, seed=seed + 1)[:, :n]
    y = np.zeros((2, 2 * n + gap), np.float32)
    v = np.zeros_like(y)
    y[:, :n] = inst
    v[:, n + gap:] = voc
    return (y + v).astype(np.float32), y, n, n + gap


def single_source_frames(T, hop, n_fft, inst_end, voc_start, L):
    """The frames whose whole window (centred STFT) lies in the instruments' span, and those in the vocals' span."""
    t = np.arange(T)
    lo, hi = t * hop - n_fft // 2, t * hop + n_fft // 2
    return t[hi <= inst_end], t[(lo >= voc_start) & (hi <= L)]


def test_time_disjoint_sources():
    from oracle import stft_oracle
    X, y, inst_end, voc_start = disjoint_pair()
    Xs = stft_oracle.wave_to_spectrogram(X, 1024, 2048)
    Ys = stft_oracle.wave_to_spectrogram(y, 1024, 2048)
    inst_frames, voc_frames = single_source_frames(Xs.shape[2], 1024, 2048, inst_end, voc_start, X.shape[1])
    assert len(inst_frames) > 50 and len(voc_frames) > 50
    for kind in KINDS:
        m = om.mask(Xs, Ys, kind)
        assert np.all(m[:, :, inst_frames] == 1.0), kind
        assert np.all(m[:, :, voc_frames] == 0.0), kind


# ---- the command line -------------------------------------------------------------------------------------------
def _listing(root, names):
    for sub in ('mixtures', 'instruments'):
        os.makedirs(os.path.join(root, sub))
        for base in names:
            open(os.path.join(root, sub, base + '.wav'), 'wb').close()


def _cli(*args, cwd=PKG):
    return subprocess.run([sys.executable, os.path.join(PKG, 'evaluate.py')] + list(args), capture_output=True,
                          text=True, cwd=cwd)


def test_cli_errors(tmp_path):
    data = str(tmp_path / 'data')
    _listing(data, ['a', 'b', 'c'])
    garbage = str(tmp_path / 'not_a_checkpoint.pth')
    with open(garbage, 'w') as f:
        f.write('not a checkpoint')
    r = _cli('-d', data, '-P', garbage, '--oracle', 'iam')
    assert r.returncode == 2 and 'not allowed with argument' in r.stderr
    r = _cli('-d', data)
    assert r.returncode == 2 and '--pretrained_model/-P' in r.stderr and '--oracle' in r.stderr
    for flag in ('-t', '-p'):
        r = _cli('-d', data, '--oracle', 'irm1', flag)
        assert r.returncode == 2 and 'cannot be used with --oracle' in r.stderr, flag
    r = _cli('-d', data, '--oracle', 'mwf', '--wiener_iterations', '1')
    assert r.returncode == 2 and '--wiener_iterations must be 0' in r.stderr
    r = _cli('-d', data, '--oracle', 'sigsep')
    assert r.returncode == 2 and 'invalid choice' in r.stderr
    r = _cli('-d', str(tmp_path / 'nowhere'), '--oracle', 'ibm')
    assert r.returncode == 2 and 'nowhere' in r.stderr


def test_cli_parser():
    import evaluate
    from lib import spec_utils
    p = evaluate.build_parser()
    assert p.parse_args(['-d', 'x', '-P', 'm.pth']).oracle is None
    for kind in spec_utils.ORACLES:
        args = p.parse_args(['-d', 'x', '--oracle', kind])
        assert args.oracle == kind and args.pretrained_model is None
    assert spec_utils.MASK_ORACLES == om.KINDS


def test_cli_without_gpu_fails_on_cuda_after_the_split(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    data = str(tmp_path / 'data')
    _listing(data, ['a', 'b', 'c', 'd', 'e'])
    r = _cli('-d', data, '--oracle', 'irm1', cwd=str(tmp_path))
    assert r.returncode != 0 and 'RuntimeError: no CUDA device' in r.stderr
    assert not [f for _, _, files in os.walk(str(tmp_path)) for f in files if f.endswith('.pth')]


def test_python_errors():
    from lib import spec_utils
    X = np.zeros((2, 1025, 4), np.complex64)
    with pytest.raises(ValueError, match='kind'):
        spec_utils.oracle_mask(X, X, 'mwf')
    with pytest.raises(ValueError, match='shape'):
        spec_utils.oracle_mask(X, X[:, :, :3], 'iam')
    with pytest.raises(ValueError, match='wiener_iterations must be 0'):
        spec_utils.oracle_spectrograms(X, X, 'mwf', 1)
    with pytest.raises(ValueError, match='kind'):
        spec_utils.oracle_separate_wave(np.zeros((2, 100), np.float32), np.zeros((2, 100), np.float32), 'ideal')
