"""The multichannel Wiener filter of ``--wiener_iterations`` (DESIGN.md §11) in float64 numpy.

norbert 0.2's ``wiener(v, x, iterations, use_softmask=False)`` restricted to 2 channels and 2 sources, with the masked
spectrograms as the initial estimates.  norbert is not installed, so this restatement of the contract is the
definition the GPU (csrc/wiener.cu) is checked against.  ``round32=True`` stores the estimates as complex64 where the
GPU does: y / s at the start, after every iteration, and s * y at the end.
"""
import numpy as np

EPS = 2.0 ** -23          # float32 machine epsilon, as norbert takes it from a complex64 mixture
REG = np.sqrt(EPS)        # the loading of the mixture covariance


def scale(X):
    """s = max(1, max|X| / 10), max|X| the float32 magnitude over both channels, all bins and all frames."""
    X = np.asarray(X, dtype=np.complex64)
    m = float(np.abs(X).max()) if X.size else 0.0
    return max(1.0, m / 10.0)


def covariance(y):
    """v (bins, T) = (|y0|^2 + |y1|^2) / 2 and R (bins, 2, 2) = sum_t y y^H / (eps + sum_t v) of one source."""
    v = (np.abs(y[0]) ** 2 + np.abs(y[1]) ** 2) / 2
    R = np.einsum('cft,dft->fcd', y, y.conj()) / (EPS + v.sum(axis=1))[:, None, None]
    return v, R


def em_step(x, ys):
    """One iteration on the scaled mixture x and estimates ys (each complex (2, bins, T)): (new estimates, u = C^-1 x)."""
    vR = [covariance(y) for y in ys]
    c = [[sum(v * R[:, a, b, None] for v, R in vR) + (REG if a == b else 0.0) for b in range(2)] for a in range(2)]
    det = c[0][0] * c[1][1] - c[0][1] * c[1][0]
    u = np.stack([(c[1][1] * x[0] - c[0][1] * x[1]) / det, (c[0][0] * x[1] - c[1][0] * x[0]) / det])
    out = [np.stack([v * (R[:, k, 0, None] * u[0] + R[:, k, 1, None] * u[1]) for k in range(2)]) for v, R in vR]
    return out, u


def wiener(X, y_spec, v_spec, iterations=1, round32=False):
    """Refined (y_spec, v_spec): complex128, or complex64 with ``round32``.  iterations = 0 returns the inputs."""
    if iterations < 0:
        raise ValueError('iterations must be >= 0')
    if iterations == 0:
        return np.array(y_spec), np.array(v_spec)
    s = scale(X)
    x = np.asarray(X, dtype=np.complex128) / s
    ys = [np.asarray(y, dtype=np.complex128) / s for y in (y_spec, v_spec)]
    for _ in range(iterations):
        if round32:
            ys = [y.astype(np.complex64).astype(np.complex128) for y in ys]
        ys, _ = em_step(x, ys)
    if round32:
        return tuple((s * y.astype(np.complex64).astype(np.complex128)).astype(np.complex64) for y in ys)
    return tuple(s * y for y in ys)
