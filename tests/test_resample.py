"""SURVEY 8(f) rank 2: the sample-rate conversion of librosa.load(res_type='kaiser_fast') = resampy.resample.

CPU part: the vectorised oracle against the literal restatement of resampy's loop, its length / dtype contract, and a
sanity anchor against scipy.signal.resample_poly (resampy itself is absent offline: parity unpinned, see the oracle's
header).  GPU part: vr_resample (csrc/resample.cu) against the oracle, through lib.audio_io."""
import os
import sys
import wave

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import resample_oracle as ro  # noqa: E402

RATES = [(48000, 44100), (22050, 44100), (44100, 48000), (32000, 44100), (96000, 44100)]


def _tones(sr, seconds, freqs=(440.0, 5000.0, 9000.0)):
    t = np.arange(int(sr * seconds)) / sr
    return sum(a * np.sin(2 * np.pi * f * t + p) for a, f, p in zip((0.5, 0.3, 0.1), freqs, (0.0, 1.0, 2.0))).astype(np.float32)


@pytest.mark.parametrize('rates', RATES)
def test_oracle_matches_literal_loop(rates):
    a, b = rates
    x = np.random.default_rng(a + b).standard_normal(257)
    y = ro.resample(x, a, b)
    assert y.shape == (int(257 * (float(b) / a)),)
    assert np.abs(y - ro.resample_literal(x, a, b)).max() < 1e-12


def test_oracle_contract_and_scipy_anchor():
    from scipy.signal import resample_poly
    x = _tones(48000, 1.0)
    y = ro.resample(np.stack([x, 0.5 * x]), 48000, 44100)
    assert y.shape == (2, 44100) and y.dtype == np.float32
    ref = resample_poly(x.astype(np.float64), 147, 160)
    assert np.abs(y[0, 2000:-2000] - ref[2000:44100 - 2000]).max() < 1e-3     # different low-pass designs, same signal
    assert np.abs(y[1] - 0.5 * y[0]).max() < 1e-6                            # linear
    with pytest.raises(ValueError):
        ro.resample(np.zeros(1), 44100, 8000)
    with pytest.raises(ValueError):
        ro.resample(np.zeros(10), 0, 8000)


@pytest.mark.parametrize('rates', [(48000, 44100), (44100, 48000)])
def test_oracle_output_range_matches_the_full_call(rates):
    """out_range computes the same samples as the full call, to the bit, for windows at both ends (where the taps are
    clipped by the signal) and inside; and it refuses a range outside the output."""
    a, b = rates
    x = np.stack([_tones(a, 0.1), _tones(a, 0.1, (1000.0, 3000.0, 7000.0))]).astype(np.float64)
    full = ro.resample(x, a, b)
    n_out = full.shape[-1]
    for t0, t1 in ((0, 37), (0, 1), (1000, 1777), (n_out - 41, n_out), (n_out, n_out), (0, n_out)):
        part = ro.resample(x, a, b, out_range=(t0, t1))
        assert part.shape == (2, t1 - t0) and np.array_equal(part, full[:, t0:t1]), (t0, t1)
    for bad in ((-1, 5), (5, 4), (0, n_out + 1)):
        with pytest.raises(ValueError):
            ro.resample(x, a, b, out_range=bad)


def test_host_table_matches_oracle_table():
    sys.path.insert(0, os.path.join(ROOT, 'vocal-remover_b200'))
    from lib import audio_io
    half, per = audio_io.kaiser_fast_table()
    ref, per_ref = ro.sinc_window(**ro.KAISER_FAST)
    assert per == per_ref == 512 and half.shape == ref.shape == (16 * 512 + 1,)
    assert np.abs(half - ref).max() == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize('rates', RATES)
def test_gpu_resample_vs_oracle(rates):
    from conftest import record_parity
    from lib import audio_io
    a, b = rates
    x = np.stack([_tones(a, 0.5), _tones(a, 0.5, (1000.0, 3000.0, 7000.0))])
    y = audio_io.resample(x, a, b)
    ref = ro.resample(x.astype(np.float64), a, b)
    assert y.shape == ref.shape and y.dtype == np.float32
    err = float(np.abs(y - ref).max())
    record_parity('resample_%d_%d' % (a, b), err, 2e-6)
    assert err < 2e-6      # fp64 accumulation on both sides, fp32 output


@pytest.mark.gpu
@pytest.mark.parametrize('rates', [(48000, 44100), (44100, 48000)])
def test_gpu_resample_four_minutes_vs_oracle(rates):
    """A 4-minute stereo track, the length real input has: the output instant t / ratio reaches ~1.1e7 there, where a
    float32 time register would keep no fraction at all.  Windows at the start, the middle and the end are compared
    with the oracle over the same output range; the oracle with its output instants rounded to float32 must miss the
    gate by a wide factor, so the windows see where the fractional table index comes from."""
    from conftest import record_parity
    from lib import audio_io
    a, b = rates
    seconds = 240.0
    x = np.stack([_tones(a, seconds), _tones(a, seconds, (1000.0, 3000.0, 7000.0))])
    y = audio_io.resample(x, a, b)
    n_out = int(x.shape[1] * (float(b) / a))
    assert y.shape == (2, n_out) and y.dtype == np.float32
    x64 = x.astype(np.float64)
    width = 4096
    for where, t0 in (('start', 0), ('middle', n_out // 2 - width // 2 + 7), ('end', n_out - width)):
        ref = ro.resample(x64, a, b, out_range=(t0, t0 + width))
        err = float(np.abs(y[:, t0:t0 + width] - ref).max())
        record_parity('resample_4min_%d_%d_%s' % (a, b, where), err, 2e-6)
        assert err < 2e-6, (where, err)
        # float32 instants miss by ~20x the gate at the start (t < 5000) and by ~4e4x from the middle on
        wrong = ro.resample(x64, a, b, out_range=(t0, t0 + width), time_dtype=np.float32)
        assert np.abs(wrong - ref).max() > (10 if where == 'start' else 1000) * 2e-6, where


@pytest.mark.gpu
def test_gpu_resample_edges_and_load(tmp_path):
    import torch
    from lib import audio_io
    # mono, a handful of samples (every tap count is clipped by the signal ends), device tensor in -> device tensor out
    x = np.random.default_rng(3).standard_normal(7).astype(np.float32)
    y = audio_io.resample(torch.from_numpy(x).cuda(), 8000, 44100)
    assert y.is_cuda and y.shape == (int(7 * 44100 / 8000),)
    assert np.abs(y.cpu().numpy() - ro.resample(x.astype(np.float64), 8000, 44100)).max() < 2e-6
    with pytest.raises(ValueError):
        audio_io.resample(np.zeros(1, np.float32), 44100, 8000)
    # a 48 kHz stereo PCM file through the reference-shaped loader
    sig = np.stack([_tones(48000, 0.25), 0.5 * _tones(48000, 0.25)])
    pcm = np.clip(np.round(sig.T * 32767.0), -32768, 32767).astype('<i2')
    path = str(tmp_path / 'in48k.wav')
    with wave.open(path, 'wb') as f:
        f.setnchannels(2)
        f.setsampwidth(2)
        f.setframerate(48000)
        f.writeframes(pcm.tobytes())
    X, sr = audio_io.load(path, sr=44100, mono=False, dtype=np.float32)
    assert sr == 44100 and X.shape == (2, int(pcm.shape[0] * 44100 / 48000)) and X.dtype == np.float32
    ref = ro.resample((pcm.T.astype(np.float32) / 32768.0).astype(np.float64), 48000, 44100)
    assert np.abs(X - ref).max() < 2e-6
