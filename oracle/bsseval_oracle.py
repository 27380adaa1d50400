"""BSS Eval images with time-invariant distortion filters, restated in float64 numpy / scipy straight from the formulas of
DESIGN.md section 10: the same contract lib/bsseval.py computes on the GPU (bsseval.cu).

Explicit correlations, the dense Gram matrix, ``scipy.linalg.solve`` and ``np.convolve`` projections; slow on purpose
(test infrastructure, and the CPU time the measurement script reports).  Parity with museval is unpinned: museval is not
available here, so this file is the reference of the GPU path, not a copy of museval.
"""
import numpy as np
import scipy.linalg

METRICS = ('sdr', 'isr', 'sir', 'sar')
# diagonal loading eps = scale * max diag G: the first scale, the factor between tries, the last scale tried
LOADING_FIRST, LOADING_STEP, LOADING_LAST = 2.0 ** -40, 2.0 ** 8, 2.0 ** -20


def check(references, estimates, window, hop, filters_len):
    s = np.asarray(references)
    e = np.asarray(estimates)
    if s.shape != e.shape or s.ndim != 3:
        raise ValueError('references and estimates must both have shape (K, C, N), got %s and %s' % (s.shape, e.shape))
    if s.shape[2] < window:
        raise ValueError('the signals (%d samples) are shorter than one window (%d)' % (s.shape[2], window))
    if not np.any(s):
        raise ValueError('every reference is zero')
    if not (np.all(np.isfinite(s)) and np.all(np.isfinite(e))):
        raise ValueError('the references and estimates must be finite (no NaN or Inf)')
    if filters_len < 1 or window < 1 or hop < 1:
        raise ValueError('filters_len, window and hop must be positive')
    return s.astype(np.float32).astype(np.float64), e.astype(np.float32).astype(np.float64)


def correlations(s, e, L):
    """R[a][b][l] = sum_u s_a(u) y_b(u + l), l < L, for the M = K*C references s_a and y = references then estimates:
    (M, 2M, L) float64, one explicit dot product per lag."""
    K, C, N = s.shape
    S = s.reshape(K * C, N)
    Y = np.concatenate([S, e.reshape(K * C, N)])
    R = np.zeros((K * C, 2 * K * C, L))
    for lag in range(min(L, N)):
        R[:, :, lag] = S[:, :N - lag] @ Y[:, lag:].T
    return R


def gram(R, L):
    """G[(a, t), (b, t')] = r[a][b](t - t'), with r[a][b](-l) = r[b][a](l): (M*L, M*L)."""
    M = R.shape[0]
    lag = np.arange(L)[:, None] - np.arange(L)[None, :]
    G = np.empty((M * L, M * L))
    for a in range(M):
        for b in range(M):
            G[a * L:(a + 1) * L, b * L:(b + 1) * L] = np.where(lag >= 0, R[a, b][np.maximum(lag, 0)],
                                                               R[b, a][np.maximum(-lag, 0)])
    return G


def rhs(R, L):
    """d[(k, c, t)] for every estimate channel e: (M*L, M)."""
    M = R.shape[0]
    return R[:, M:, :].transpose(0, 2, 1).reshape(M * L, M)


def loading_scale(A, base):
    """The first of LOADING_FIRST, LOADING_FIRST * LOADING_STEP, ... up to LOADING_LAST for which A + scale * base * I
    has a Cholesky factor.  A Gram matrix is only positive semidefinite (a duplicated channel makes it singular,
    band-limited references singular to rounding); 2^-40 of its largest diagonal value is above the rounding of the
    factorisation at these sizes, so the later scales are a fallback that well-formed input does not reach."""
    scale = LOADING_FIRST
    while scale <= LOADING_LAST:
        try:
            scipy.linalg.cholesky(A + scale * base * np.eye(A.shape[0]), lower=True)
            return scale
        except np.linalg.LinAlgError:
            scale *= LOADING_STEP
    raise ValueError('the Gram matrix is not positive definite even with a loading of %g of its largest diagonal '
                     'value' % LOADING_LAST)


def decompose(s, e, L, scales=None):
    """(s_true, e_spat, e_interf, e_artif), each (K, C, N) float64, on the samples [0, N) the frames cover.
    ``scales``: the loading scale of the full system and of each source's block (K + 1 values), found by
    loading_scale when None."""
    K, C, N = s.shape
    M = K * C
    R = correlations(s, e, L)
    G = gram(R, L)
    d = rhs(R, L)
    base = np.max(np.diag(G))
    blocks = [slice(j * C * L, (j + 1) * C * L) for j in range(K)]
    if scales is None:
        scales = [loading_scale(G, base)] + [loading_scale(G[r, r], base) for r in blocks]
    a_all = scipy.linalg.solve(G + scales[0] * base * np.eye(M * L), d)
    S = s.reshape(M, N)
    P_all = np.zeros((M, N))
    P_j = np.zeros((M, N))
    for j in range(K):
        rows = blocks[j]
        a_j = scipy.linalg.solve(G[rows, rows] + scales[1 + j] * base * np.eye(C * L), d[rows, j * C:(j + 1) * C])
        for i in range(C):
            ej = j * C + i
            for kc in range(M):
                P_all[ej] += np.convolve(S[kc], a_all[kc * L:(kc + 1) * L, ej])[:N]
            for c in range(C):
                P_j[ej] += np.convolve(S[j * C + c], a_j[c * L:(c + 1) * L, i])[:N]
    P_all = P_all.reshape(K, C, N)
    P_j = P_j.reshape(K, C, N)
    return s, P_j - s, P_all - P_j, e - P_all


def bss_eval(references, estimates, window, hop, filters_len=512, scales=None):
    """dict of (K, nwin) float64 arrays 'sdr', 'isr', 'sir', 'sar' (dB per frame, NaN for silent frames).
    ``scales`` fixes the diagonal loadings (see decompose)."""
    s, e = check(references, estimates, window, hop, filters_len)
    K, C, N = s.shape
    s_true, e_spat, e_interf, e_artif = decompose(s, e, filters_len, scales)
    nwin = (N - window + hop) // hop
    out = {m: np.full((K, nwin), np.nan) for m in METRICS}

    def energy(x, sl):
        return np.sum(x[:, :, sl] ** 2, axis=(1, 2))   # over the frame and the channels of each source

    with np.errstate(divide='ignore', invalid='ignore'):
        for w in range(nwin):
            sl = slice(w * hop, w * hop + window)
            if np.any(energy(s, sl) == 0) or np.any(energy(e, sl) == 0):
                continue
            out['isr'][:, w] = 10 * np.log10(energy(s_true, sl) / energy(e_spat, sl))
            out['sdr'][:, w] = 10 * np.log10(energy(s_true, sl) / energy(e_spat + e_interf + e_artif, sl))
            out['sir'][:, w] = 10 * np.log10(energy(s_true + e_spat, sl) / energy(e_interf, sl))
            out['sar'][:, w] = 10 * np.log10(energy(s_true + e_spat + e_interf, sl) / energy(e_artif, sl))
    return out
