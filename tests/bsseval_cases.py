"""Seeded signals with known BSS Eval answers, shared by tests/test_bsseval_host.py (against the float64 oracle) and
tests/test_gpu_bsseval.py (the GPU against the oracle)."""
import numpy as np

SR = 44100


def spatial(K=2, C=2, seconds=5.0, L=512, taps=300, seed=11):
    """Every estimate is its own source filtered by a seeded FIR of ``taps`` <= L taps per channel pair:
    shat_ji = sum_c h_jic * s_jc.  The references are white noise with their last L samples silent, so that the filtered
    signals end inside the track and lie exactly in the span of the delayed references.  Returns (s, shat) float32."""
    rng = np.random.default_rng(seed)
    N = int(seconds * SR)
    s = rng.standard_normal((K, C, N)).astype(np.float32)
    s[:, :, N - L:] = 0
    e = np.zeros((K, C, N))
    for j in range(K):
        for i in range(C):
            for c in range(C):
                h = rng.standard_normal(taps) * np.exp(-np.arange(taps) / 40.0) * 0.3
                if c == i:
                    h[0] += 1.0
                e[j, i] += np.convolve(s[j, c].astype(np.float64), h)[:N]
    return s, e.astype(np.float32)


def interference(alpha=0.3, seconds=10.0, seed=12):
    """Two independent white-noise stereo sources; shat_j = s_j + alpha s_k (k the other source)."""
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((2, 2, int(seconds * SR))).astype(np.float32)
    e = (s + np.float32(alpha) * s[::-1]).astype(np.float32)
    return s, e


def artifacts(level=0.2, seconds=10.0, seed=13):
    """shat_j = s_j + n_j with n independent white noise."""
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((2, 2, int(seconds * SR))).astype(np.float32)
    n = (level * rng.standard_normal(s.shape)).astype(np.float32)
    return s, (s + n).astype(np.float32), n


def frame_energy(x, window, hop, nwin):
    """(K, nwin) sums of x^2 over each frame and the channels of each source, float64."""
    x = np.asarray(x, dtype=np.float64)
    return np.stack([np.sum(x[:, :, w * hop:w * hop + window] ** 2, axis=(1, 2)) for w in range(nwin)], axis=1)


# frame rules: N = 5500 is not a multiple of hop = 700; window 1000 -> 7 frames, starting 0, 700, ..., 4200
RULES_N, RULES_WINDOW, RULES_HOP, RULES_NWIN = 5500, 1000, 700, 7
RULES_NAN_FRAMES = (2, 5)


def frame_rules(seed=14):
    """Noise references and noisy estimates with source 0's reference silent over frame 2 ([1400, 2400)) and source 1's
    estimate silent over frame 5 ([3500, 4500)): frames 2 and 5 are NaN for both sources, the rest finite."""
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((2, 2, RULES_N)).astype(np.float32)
    e = (s + 0.5 * rng.standard_normal(s.shape) + 0.3 * s[::-1]).astype(np.float32)
    s[0, :, 1400:2400] = 0
    e[1, :, 3500:4500] = 0
    return s, e


def duplicated(seconds=5.0, seed=15):
    """A mono track duplicated to both channels (what evaluate.py makes of a mono file): white-noise references whose
    two channels are equal, so the Gram matrix is exactly singular, and estimates with interference and noise."""
    rng = np.random.default_rng(seed)
    s = np.repeat(rng.standard_normal((2, 1, int(seconds * SR))), 2, axis=1).astype(np.float32)
    e = s + 0.3 * s[::-1] + np.repeat(0.1 * rng.standard_normal((2, 1, s.shape[2])), 2, axis=1)
    return s, e.astype(np.float32)


def band_limited(cutoff=0.5, seconds=5.0, seed=16):
    """float32 references band-limited to ``cutoff`` of Nyquist (as resampled or filtered stems are), so the Gram
    matrix is singular to rounding, and full-band estimates with interference and noise."""
    import scipy.signal
    rng = np.random.default_rng(seed)
    b, a = scipy.signal.butter(12, cutoff)
    s = scipy.signal.lfilter(b, a, rng.standard_normal((2, 2, int(seconds * SR)))).astype(np.float32)
    e = s + 0.3 * s[::-1] + 0.1 * rng.standard_normal(s.shape)
    return s, e.astype(np.float32)
