"""BSS Eval v3 (framewise distortion filters) in float64 numpy / scipy, from the contract of DESIGN.md section 10,
"Framewise filters (v3)": the reference of lib/bsseval.py's ``framewise=True`` path.

Every frame that is not silent is scored as a signal of its own with the functions of oracle/bsseval_oracle.py,
unchanged: the frame's slices are zero-padded by L - 1 samples, so that ``decompose`` (which keeps its projections to
the length of its input) projects on the frame's whole timeline of window + L - 1 samples.  The padding adds nothing to
the correlations, so the frame's Gram matrix and right-hand sides are those of its window samples.  Slow on purpose:
one dense solve per system and frame.
"""
import numpy as np

from oracle import bsseval_oracle as bo


def _frames(s, e, window, hop, L):
    """Yield (w, slice of s, slice of e) for every frame, the slices zero-padded to window + L - 1 samples, or None
    for a frame in which a reference source or an estimate is all zeros."""
    K, C, N = s.shape
    nwin = (N - window + hop) // hop
    pad = ((0, 0), (0, 0), (0, L - 1))
    for w in range(nwin):
        ss = s[:, :, w * hop:w * hop + window]
        ee = e[:, :, w * hop:w * hop + window]
        if np.any(np.sum(ss ** 2, axis=(1, 2)) == 0) or np.any(np.sum(ee ** 2, axis=(1, 2)) == 0):
            yield w, None, None
        else:
            yield w, np.pad(ss, pad), np.pad(ee, pad)


def _check(references, estimates, window, hop, filters_len):
    s, e = bo.check(references, estimates, window, hop, filters_len)
    if window < filters_len:
        raise ValueError('with framewise filters the window (%d samples) must not be shorter than filters_len (%d)'
                         % (window, filters_len))
    return s, e


def frame_loading(sp, ep, L):
    """The K + 1 loading scales of one frame's systems (all unknowns, then each source), from its padded slices."""
    K, C, _ = sp.shape
    G = bo.gram(bo.correlations(sp, ep, L), L)
    base = np.max(np.diag(G))
    blocks = [slice(j * C * L, (j + 1) * C * L) for j in range(K)]
    return [bo.loading_scale(G, base)] + [bo.loading_scale(G[r, r], base) for r in blocks]


def loading(references, estimates, window, hop, filters_len=512):
    """(nwin, K + 1) loading scales of every frame's systems, NaN rows for silent frames."""
    s, e = _check(references, estimates, window, hop, filters_len)
    K, C, N = s.shape
    out = np.full(((N - window + hop) // hop, K + 1), np.nan)
    for w, sp, ep in _frames(s, e, window, hop, filters_len):
        if sp is not None:
            out[w] = frame_loading(sp, ep, filters_len)
    return out


def bss_eval_framewise(references, estimates, window, hop, filters_len=512, scales=None):
    """dict of (K, nwin) float64 arrays 'sdr', 'isr', 'sir', 'sar' (dB per frame, NaN for silent frames), every frame
    with its own distortion filters.  ``scales``: (nwin, K + 1) loading scales to use instead of the schedule's."""
    s, e = _check(references, estimates, window, hop, filters_len)
    K, C, N = s.shape
    L = filters_len
    nwin = (N - window + hop) // hop
    out = {m: np.full((K, nwin), np.nan) for m in bo.METRICS}

    def energy(x):
        return np.sum(x ** 2, axis=(1, 2))   # over the frame's timeline and the channels of each source

    with np.errstate(divide='ignore', invalid='ignore'):
        for w, sp, ep in _frames(s, e, window, hop, L):
            if sp is None:
                continue
            sc = list(scales[w]) if scales is not None else frame_loading(sp, ep, L)
            s_true, e_spat, e_interf, e_artif = bo.decompose(sp, ep, L, sc)
            out['isr'][:, w] = 10 * np.log10(energy(s_true) / energy(e_spat))
            out['sdr'][:, w] = 10 * np.log10(energy(s_true) / energy(e_spat + e_interf + e_artif))
            out['sir'][:, w] = 10 * np.log10(energy(s_true + e_spat) / energy(e_interf))
            out['sar'][:, w] = 10 * np.log10(energy(s_true + e_spat + e_interf) / energy(e_artif))
    return out
