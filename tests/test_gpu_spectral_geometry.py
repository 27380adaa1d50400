"""The STFT and the inverse STFT (csrc/fft.cu) over the whole geometry the library accepts (run on an H100).

vr_create takes any power-of-two n_fft in [64, 4096] and any hop_length in (0, n_fft].  Every n_fft is run at hops
n_fft/2, n_fft/4 and n_fft/8, at an odd hop that does not divide n_fft, and at hop = n_fft, where the window-sum-square
is zero at each frame's first sample and the float32-tiny guard of the overlap-add decides the output.  n_fft = 2048 runs
the radix-8 kernels, every other n_fft the radix-2 ones.  Each comparison is against oracle/stft_oracle.py (librosa 0.10
restated in float64) and also computes, in float64 numpy, a wrong variant of the operation that must miss the gate by a
wide factor, so that no gate passes vacuously.

Metrics:
* STFT: max |S - R| / max |R| (the gate of test_gpu_parity.py).
* inverse STFT: the error of each output sample times wss / sum(w) (its window-sum-square over the sum of the windows
  that overlap it), relative to the largest windowed frame value.  Where the frames overlap well that factor is about
  one; near the zeros of the window-sum-square the output is a float32 frame error divided by the window, and the
  factor takes that division back out, so the metric measures the transform's error wherever the output exists.
"""
import numpy as np
import pytest
import torch

from conftest import record_parity

pytestmark = pytest.mark.gpu

NFFTS = (64, 128, 256, 512, 1024, 2048, 4096)
STFT_GATE = 5e-6
ISTFT_GATE = 5e-6
NONVACUOUS = 10   # a wrong variant must land at least this many gates away
SR = 44100


def _odd_hop(n_fft):
    """odd and not a divisor of n_fft (a power of two): 3 n_fft / 8 + 1"""
    return 3 * n_fft // 8 + 1


def _geometries():
    for n_fft in NFFTS:
        for hop in (n_fft // 2, n_fft // 4, n_fft // 8, _odd_hop(n_fft), n_fft):
            yield n_fft, hop


GEOMETRIES = list(_geometries())


def _lengths(n_fft, hop):
    """one sample, shorter than the centre padding, one short of and exactly k hops, and a ragged few seconds"""
    k = 5
    return (1, n_fft // 2 - 1, hop * k - 1, hop * k, 3 * SR + 37)


def _symmetric_hann_stft(y, n_fft, hop):
    """the STFT with a symmetric Hann window (np.hanning) in place of the periodic one, float64"""
    yp = np.concatenate([np.zeros(n_fft // 2), y.astype(np.float64), np.zeros(n_fft // 2)])
    T = 1 + len(y) // hop
    frames = np.lib.stride_tricks.sliding_window_view(yp, n_fft)[::hop][:T]
    return np.fft.rfft(frames * np.hanning(n_fft)[None, :], axis=1).T


def _ola_weight(n_fft, hop, T):
    """per output sample: wss / sum(w) over the frames that overlap it (1 where no window reaches it), and where the
    window-sum-square is exactly zero (hop = n_fft: every frame's first sample), which only the overlap-add's
    float32-tiny guard keeps from a 0 / 0"""
    from oracle import stft_oracle
    w = stft_oracle.hann_periodic(n_fft)
    full = n_fft + hop * (T - 1)
    wss, wsum = np.zeros(full), np.zeros(full)
    for t in range(T):
        wss[t * hop:t * hop + n_fft] += w * w
        wsum[t * hop:t * hop + n_fft] += w
    wss, wsum = wss[n_fft // 2:full - n_fft // 2], wsum[n_fft // 2:full - n_fft // 2]
    return np.where(wsum > 0, wss / np.where(wsum > 0, wsum, 1.0), 1.0), wss == 0


def _frame_scale(S):
    """largest windowed frame value of the inverse transform of S (bins, T), float64"""
    from oracle import stft_oracle
    n_fft = 2 * (S.shape[-2] - 1)
    frames = np.fft.irfft(S.astype(np.complex128), n=n_fft, axis=-2) * stft_oracle.hann_periodic(n_fft)[:, None]
    return max(float(np.abs(frames).max()), 1e-30)


def _istft_ratio(got, ref, weight, scale):
    if got.size == 0:
        return 0.0
    return float((np.abs(got.astype(np.float64) - ref.astype(np.float64)) * weight).max() / scale)


def _fold(acc, key, *ratios):
    """acc[key] = the largest of acc[key] and ratios, NaN if any of them is NaN (Python's max would drop a NaN)"""
    acc[key] = float(np.max([acc[key], *ratios]))


def _check_inverse(name, got, ref, dead):
    """finite everywhere, and exactly zero where the window-sum-square is zero (the oracle's output is zero there)"""
    assert np.isfinite(got).all(), '%s: %d non-finite samples' % (name, int((~np.isfinite(got)).sum()))
    assert not ref[..., dead].any(), name
    assert not got[..., dead].any(), '%s: nonzero where the window-sum-square is zero' % name


def _packed_istft_keeping_dc_nyquist(Ya, Yb, hop):
    """What a two-for-one inverse transform (stem a in the real part, stem b in the imaginary part) computes when it
    keeps the imaginary parts of DC and Nyquist: the frames are the complex inverse of ext(Ya) + i ext(Yb), where
    ext is the Hermitian extension with the DC and Nyquist values left as they are.  Overlap-add and normalisation are
    the oracle's (its irfft of the rfft of a real frame is that frame).  Returns the two stems, float64 frames."""
    from oracle import stft_oracle
    n_fft = 2 * (Ya.shape[0] - 1)

    def ext(Y):
        return np.concatenate([Y, np.conj(Y[-2:0:-1])]).astype(np.complex128)

    z = np.fft.ifft(ext(Ya) + 1j * ext(Yb), axis=0)
    return (stft_oracle.istft(np.fft.rfft(z.real, axis=0), hop), stft_oracle.istft(np.fft.rfft(z.imag, axis=0), hop))


def _non_hermitian_spectrum(rng, bins, T):
    """random complex spectrum (2, bins, T) whose DC and Nyquist rows carry large imaginary parts"""
    S = rng.standard_normal((2, bins, T)) + 1j * rng.standard_normal((2, bins, T))
    S[:, [0, -1]] += 6j * np.sign(rng.standard_normal((2, 2, T)))
    return S.astype(np.complex64)


def _mask_with_exact_ends(rng, shape):
    m = rng.random(shape).astype(np.float32)
    m.reshape(-1)[::7] = 0.0
    m.reshape(-1)[3::7] = 1.0
    return m


def _apply_mask_istft(n_fft, hop, X, mask):
    from lib import _native, spec_utils
    ctx = spec_utils._spectral_ctx(n_fft, hop)
    dev = torch.device('cuda', ctx.device_index)
    T = X.shape[2]
    d_x = torch.from_numpy(np.ascontiguousarray(X)).to(dev)
    d_m = torch.from_numpy(np.ascontiguousarray(mask)).to(dev)
    inst = torch.empty((2, hop * (T - 1)), dtype=torch.float32, device=dev)
    voc = torch.empty_like(inst)
    ctx.check(ctx.lib.vr_apply_mask_istft(ctx.handle, _native.ptr(d_x), _native.ptr(d_m), T, _native.ptr(inst),
                                          _native.ptr(voc), _native.stream_ptr()), 'vr_apply_mask_istft')
    return inst.cpu().numpy(), voc.cpu().numpy()


@pytest.mark.parametrize('n_fft,hop', GEOMETRIES)
def test_stft_and_istft_geometry_vs_oracle(n_fft, hop):
    """For every length of _lengths: the STFT of a random stereo signal; the inverse STFT (vr_istft) of (a) the
    oracle's spectrum of that signal and (b) a random spectrum with large imaginary DC and Nyquist parts; and the
    masked inverse STFT (vr_apply_mask_istft) of (b) under a mask in [0, 1] that holds exact zeros and ones, against
    istft(m X) and istft((1 - m) X).

    Every output must be finite, and the inverse outputs exactly zero where the window-sum-square is zero (hop =
    n_fft), so the overlap-add's float32-tiny guard is tested; the ratios are folded with a NaN-propagating maximum.

    Wrong variants: a symmetric Hann window (STFT); the masked kernels without their DC / Nyquist zeroing, i.e. the
    packed complex inverse of ext(m X) + i ext((1-m) X) (_packed_istft_keeping_dc_nyquist), which is what
    istft_frames_kernel and istft2048_frames_kernel compute with the `k == 0 || k == NF / 2` zeroing deleted, so
    deleting it fails this test.  For vr_istft that zeroing changes nothing: it transforms one channel per CTA and
    keeps only the real output, where the imaginary DC and Nyquist parts never land.  Its wrong variant (the real
    plus the imaginary part of the complex inverse) is a perturbation of the size of those parts, which shows that the
    gate resolves them, not a mutation of the kernel."""
    from lib import spec_utils
    from oracle import stft_oracle
    rng = np.random.default_rng(n_fft * 7919 + hop)
    bins = n_fft // 2 + 1
    worst = dict(stft=0.0, istft_real=0.0, istft_nonhermitian=0.0, mask_istft=0.0)
    wrong = dict(stft=0.0, istft_nonhermitian=0.0, mask_istft=0.0)
    for L in _lengths(n_fft, hop):
        T = 1 + L // hop
        x = rng.standard_normal((2, L)).astype(np.float32)
        # STFT
        S = spec_utils.wave_to_spectrogram(x, hop, n_fft)
        R = stft_oracle.wave_to_spectrogram(x, hop, n_fft)
        assert S.shape == R.shape == (2, bins, T) and S.dtype == np.complex64
        assert np.isfinite(S).all(), 'stft: %d non-finite values' % int((~np.isfinite(S)).sum())
        scale = float(np.abs(R).max())
        _fold(worst, 'stft', float(np.abs(S - R).max()) / scale)
        Rs = np.asarray([_symmetric_hann_stft(x[c], n_fft, hop) for c in range(2)])
        _fold(wrong, 'stft', float(np.abs(Rs - R).max()) / scale)

        weight, dead = _ola_weight(n_fft, hop, T)
        # (a) the spectrum of a real signal
        w = spec_utils.spectrogram_to_wave(R, hop)
        wr = stft_oracle.spectrogram_to_wave(R, hop)
        assert w.shape == wr.shape == (2, hop * (T - 1)) and w.dtype == np.float32
        _check_inverse('istft_real', w, wr, dead)
        _fold(worst, 'istft_real', _istft_ratio(w, wr, weight, _frame_scale(R)))
        # (b) a spectrum no real signal has
        X = _non_hermitian_spectrum(rng, bins, T)
        sx = _frame_scale(X)
        w = spec_utils.spectrogram_to_wave(X, hop)
        wr = stft_oracle.spectrogram_to_wave(X, hop)
        _check_inverse('istft_nonhermitian', w, wr, dead)
        _fold(worst, 'istft_nonhermitian', _istft_ratio(w, wr, weight, sx))
        for c in range(2):
            full = np.concatenate([X[c], np.conj(X[c, -2:0:-1])]).astype(np.complex128)
            z = np.fft.ifft(full, axis=0)
            perturbed = stft_oracle.istft(np.fft.rfft(z.real + z.imag, axis=0), hop)
            _fold(wrong, 'istft_nonhermitian', _istft_ratio(perturbed, wr[c], weight, sx))
        # (b) through the masked inverse
        m = _mask_with_exact_ends(rng, X.shape)
        inst, voc = _apply_mask_istft(n_fft, hop, X, m)
        X64 = X.astype(np.complex128)
        ref_i = stft_oracle.spectrogram_to_wave(m * X64, hop)
        ref_v = stft_oracle.spectrogram_to_wave((1.0 - m) * X64, hop)
        _check_inverse('mask_istft instruments', inst, ref_i, dead)
        _check_inverse('mask_istft vocals', voc, ref_v, dead)
        _fold(worst, 'mask_istft', _istft_ratio(inst, ref_i, weight, sx), _istft_ratio(voc, ref_v, weight, sx))
        for c in range(2):
            bad_i, bad_v = _packed_istft_keeping_dc_nyquist(m[c] * X64[c], (1.0 - m[c]) * X64[c], hop)
            _fold(wrong, 'mask_istft', _istft_ratio(bad_i, ref_i[c], weight, sx),
                  _istft_ratio(bad_v, ref_v[c], weight, sx))

    gates = dict(stft=STFT_GATE, istft_real=ISTFT_GATE, istft_nonhermitian=ISTFT_GATE, mask_istft=ISTFT_GATE)
    failed = []
    for name, r in worst.items():
        record_parity('%s_nfft%d_hop%d' % (name, n_fft, hop), r, gates[name])
        if not r <= gates[name]:
            failed.append('%s: %.4g > gate %.4g' % (name, r, gates[name]))
    for name, r in wrong.items():
        if not r >= NONVACUOUS * gates[name]:
            failed.append('%s wrong variant only %.4g (needs >= %.4g)' % (name, r, NONVACUOUS * gates[name]))
    assert not failed, '\n'.join(failed)
