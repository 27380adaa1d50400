"""Pins oracle/stft_oracle.py (the librosa 0.10 restatement, SURVEY App. A).

librosa is absent, so the STFT boundary is 'parity unpinned' by the reference itself; these tests
cross-check the restatement against an independent implementation (torch.stft / torch.istft with
the same conventions) and by round trip.
"""
import numpy as np
import torch

from oracle import stft_oracle
from lib import synth


def test_stft_matches_torch_stft():
    x = synth.sine_mix(2.0)
    S = stft_oracle.wave_to_spectrogram(x, 1024, 2048)
    assert S.dtype == np.complex64 and S.shape == (2, 1025, 1 + x.shape[1] // 1024)
    win = torch.hann_window(2048, periodic=True, dtype=torch.float64)
    St = torch.stft(torch.from_numpy(x).double(), 2048, 1024, window=win, center=True,
                    pad_mode='constant', return_complex=True).numpy()
    assert np.abs(S - St).max() <= 2e-5 * np.abs(St).max()


def test_istft_matches_torch_istft_and_roundtrip():
    x = synth.sine_mix(2.0)
    S = stft_oracle.wave_to_spectrogram(x, 1024, 2048)
    w = stft_oracle.spectrogram_to_wave(S, 1024)
    assert w.dtype == np.float32 and w.shape == (2, 1024 * (S.shape[2] - 1))
    win = torch.hann_window(2048, periodic=True, dtype=torch.float64)
    wt = torch.istft(torch.from_numpy(S).to(torch.complex128), 2048, 1024, window=win, center=True).numpy()
    assert np.abs(w - wt).max() < 2e-6
    assert np.abs(w - x[:, :w.shape[1]]).max() < 2e-6
    # 2-D (mono) input path of lib/spec_utils.py:158-159
    w0 = stft_oracle.spectrogram_to_wave(S[0], 1024)
    assert np.array_equal(w0, w[0])


def test_small_fft_and_ragged_lengths():
    rng = np.random.default_rng(1)
    for L in (256, 1000, 4097):
        x = rng.standard_normal(L).astype(np.float32)
        S = stft_oracle.stft(x, 512, 256)
        assert S.shape == (257, 1 + L // 256)
        w = stft_oracle.istft(S, 256)
        assert w.shape == (256 * (S.shape[1] - 1),)
        assert np.abs(w - x[:len(w)]).max() < 1e-5


def test_istft_of_non_hermitian_spectra_matches_torch():
    """Spectra whose DC and Nyquist rows have imaginary parts (no real signal has them): the oracle drops those parts
    as a c2r transform does (np.fft.irfft, librosa.istft), which torch.istft / torch.fft.irfft confirm.  At hop = n_fft
    torch.istft refuses the spectrum (the window-sum-square is zero at every frame's first sample), so there the frames
    are inverted with torch.fft.irfft, windowed, and divided by the window square where it exceeds float32's tiny."""
    rng = np.random.default_rng(5)
    for n_fft, hop, T in ((64, 16, 40), (64, 64, 9), (4096, 1024, 9), (4096, 4096, 5)):
        bins = n_fft // 2 + 1
        S = (rng.standard_normal((bins, T)) + 1j * rng.standard_normal((bins, T))).astype(np.complex64)
        S[[0, -1]] += 8j   # large imaginary DC and Nyquist
        w = stft_oracle.istft(S, hop)
        assert w.shape == (hop * (T - 1),)
        win = torch.hann_window(n_fft, periodic=True, dtype=torch.float64)
        St = torch.from_numpy(S).to(torch.complex128)
        if hop < n_fft:
            ref = torch.istft(St, n_fft, hop, window=win, center=True).numpy()
        else:
            frames = torch.fft.irfft(St, n_fft, dim=0) * win[:, None]
            wsq = win * win
            frames = torch.where((wsq > np.finfo(np.float32).tiny)[:, None], frames / wsq[:, None], frames)
            ref = frames.T.reshape(-1)[n_fft // 2:n_fft // 2 + hop * (T - 1)].numpy()
        assert ref.shape == w.shape
        # relative to each sample's own size: at hop = n_fft the division by the window square scales samples by 1e7
        err = np.abs(w - ref) / np.maximum(np.abs(ref), 1.0)
        assert err.max() < 1e-6, (n_fft, hop, err.max())
        # the gate resolves perturbations of the size of those imaginary parts: the Hermitian extension's complex
        # inverse, real plus imaginary part (not what any c2r transform computes; its real part alone is the irfft)
        full = np.concatenate([S, np.conj(S[-2:0:-1])]).astype(np.complex128)
        z = np.fft.ifft(full, axis=0)
        perturbed = stft_oracle.istft(np.fft.rfft(z.real + z.imag, axis=0), hop)
        assert (np.abs(perturbed - ref) / np.maximum(np.abs(ref), 1.0)).max() > 1e-3


def test_golden_spectrogram(golden_default):
    g = golden_default
    x = synth.sine_mix(10.0)
    S = stft_oracle.wave_to_spectrogram(x, 1024, 2048)
    assert np.array_equal(S[:, ::16, :], g['X_sub'])
    assert np.float32(np.abs(S).max()) == g['absmax']


def test_stft_and_istft_match_scipy_signal():
    """Second independent implementation (scipy.signal, the library librosa builds its window on): same framing
    (zero centre padding, hop 1024, periodic Hann), scipy scales the forward transform by 1 / sum(window)."""
    from scipy import signal
    x = synth.sine_mix(2.0)
    S = stft_oracle.wave_to_spectrogram(x, 1024, 2048)
    win = signal.get_window('hann', 2048, fftbins=True)
    _, _, Z = signal.stft(x.astype(np.float64), window=win, nperseg=2048, noverlap=1024, boundary='zeros',
                          padded=False, return_onesided=True)
    Z = Z * win.sum()
    assert Z.shape == S.shape
    assert np.abs(S - Z).max() <= 2e-5 * np.abs(Z).max()
    _, w = signal.istft(S.astype(np.complex128) / win.sum(), window=win, nperseg=2048, noverlap=1024, boundary=True)
    wo = stft_oracle.spectrogram_to_wave(S, 1024)
    n = wo.shape[1]
    assert w.shape[1] >= n
    assert np.abs(wo - w[:, :n]).max() < 5e-6
