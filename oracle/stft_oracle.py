"""CPU oracle for the two external ``librosa`` calls on the hot path.  TEST INFRASTRUCTURE.

The reference calls ``librosa.stft(wave[c], n_fft=n_fft, hop_length=hop_length)``
(lib/spec_utils.py:27-28) and ``librosa.istft(spec[c], hop_length=hop_length)``
(lib/spec_utils.py:159-162).  librosa (pinned ``librosa~=0.10.0``,
requirements.txt:4) is a third-party dependency that is NOT vendored under
the reference checkout and is not installable offline, so this file restates the
published librosa 0.10 algorithm (defaults: window='hann' periodic, center=True,
pad_mode='constant', win_length=n_fft) as summarised in SURVEY.md App. A.

PARITY UNPINNED at this boundary: the reference holds no tests / golden vectors
for STFT, and librosa itself cannot be run here.  The restatement is cross-checked
against two independent implementations (``torch.stft`` / ``torch.istft`` and
``scipy.signal.stft`` / ``istft``) and by round trip in tests/test_oracle_stft.py.
"""
import numpy as np


def hann_periodic(n_fft):
    # scipy.signal.get_window('hann', n_fft, fftbins=True): periodic Hann, float64
    n = np.arange(n_fft, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * n / n_fft)


def stft(y, n_fft=2048, hop_length=None):
    """librosa.stft(y, n_fft=, hop_length=) for 1-D float32 ``y`` -> complex64 (1+n_fft//2, T).

    Zero ("constant") centre padding of n_fft//2 each side, T = 1 + len(y)//hop,
    float64 window * float32 frame -> float64 rfft -> stored complex64.
    """
    y = np.asarray(y)
    if hop_length is None:
        hop_length = n_fft // 4
    w = hann_periodic(n_fft)
    yp = np.concatenate([np.zeros(n_fft // 2, y.dtype), y, np.zeros(n_fft // 2, y.dtype)])
    n_frames = 1 + (len(yp) - n_fft) // hop_length
    out = np.empty((1 + n_fft // 2, n_frames), dtype=np.complex64)
    # block over frames to bound memory
    blk = 4096
    for s in range(0, n_frames, blk):
        e = min(n_frames, s + blk)
        idx = (np.arange(s, e)[:, None] * hop_length) + np.arange(n_fft)[None, :]
        frames = yp[idx].astype(np.float64) * w[None, :]
        out[:, s:e] = np.fft.rfft(frames, axis=1).T
    return out


def istft(S, hop_length=None):
    """librosa.istft(S, hop_length=) for complex64 (1+n_fft//2, T) -> float32 (hop*(T-1),).

    irfft (1/N normalised, float64) * periodic Hann, overlap-add at ``hop_length``
    into a float32 buffer, divide by the window-sum-square where > tiny(float32),
    trim n_fft//2 from each end (center=True, length=None).
    """
    S = np.asarray(S)
    n_fft = 2 * (S.shape[0] - 1)
    if hop_length is None:
        hop_length = n_fft // 4
    n_frames = S.shape[1]
    w = hann_periodic(n_fft)
    full_len = n_fft + hop_length * (n_frames - 1)
    y = np.zeros(full_len, dtype=np.float32)
    wss = np.zeros(full_len, dtype=np.float32)
    wsq = (w * w).astype(np.float32)
    blk = 2048
    for s in range(0, n_frames, blk):
        e = min(n_frames, s + blk)
        ytmp = np.fft.irfft(S[:, s:e].astype(np.complex128), n=n_fft, axis=0) * w[:, None]
        for t in range(s, e):
            y[t * hop_length:t * hop_length + n_fft] += ytmp[:, t - s].astype(np.float32)
            wss[t * hop_length:t * hop_length + n_fft] += wsq
    nz = wss > np.finfo(np.float32).tiny
    y[nz] /= wss[nz]
    return y[n_fft // 2: full_len - n_fft // 2]


def wave_to_spectrogram(wave, hop_length, n_fft):
    """Restates lib/spec_utils.py:26-31 over the stft restatement above."""
    return np.asarray([stft(wave[0], n_fft=n_fft, hop_length=hop_length),
                       stft(wave[1], n_fft=n_fft, hop_length=hop_length)])


def spectrogram_to_wave(spec, hop_length=1024):
    """Restates lib/spec_utils.py:157-165 (2-D mono or 3-D stereo spectrogram)."""
    if spec.ndim == 2:
        return istft(spec, hop_length=hop_length)
    return np.asarray([istft(spec[0], hop_length=hop_length),
                       istft(spec[1], hop_length=hop_length)])
