"""The BSS Eval v3 (framewise filters) oracle without a GPU: against an explicit least-squares formulation, a closed
form, the slicing of a track into frames, the silence rule and the errors; and the command line's check of
--framewise_filters before the model loads."""
import os
import subprocess
import sys

import numpy as np
import pytest

import bsseval_cases as cases
import bsseval_framewise_oracle as fo
from conftest import PKG
from oracle import bsseval_oracle as bo


def _delays(x, L, length):
    """(length, C * L) matrix of the channels of x (C, n) delayed by 0 .. L - 1 samples, zero outside [0, n)."""
    C, n = x.shape
    A = np.zeros((length, C * L))
    for c in range(C):
        for tau in range(L):
            A[tau:tau + n, c * L + tau] = x[c]
    return A


def _lstsq_frame(s, e, L):
    """Ratios of one frame (K, C, n) from np.linalg.lstsq on the explicit (n + L - 1) x K*C*L matrix of delays."""
    K, C, n = s.shape
    T = n + L - 1
    A = _delays(s.reshape(K * C, n), L, T)
    y = np.zeros((K * C, T))
    y[:, :n] = e.reshape(K * C, n)
    st = np.zeros((K * C, T))
    st[:, :n] = s.reshape(K * C, n)
    P_all = (A @ np.linalg.lstsq(A, y.T, rcond=None)[0]).T
    P_j = np.zeros_like(P_all)
    for j in range(K):
        Aj = A[:, j * C * L:(j + 1) * C * L]
        rows = slice(j * C, (j + 1) * C)
        P_j[rows] = (Aj @ np.linalg.lstsq(Aj, y[rows].T, rcond=None)[0]).T

    def energy(x):
        return np.sum(x.reshape(K, C, T) ** 2, axis=(1, 2))
    e_spat, e_interf, e_artif = P_j - st, P_all - P_j, y - P_all
    return {'isr': 10 * np.log10(energy(st) / energy(e_spat)),
            'sdr': 10 * np.log10(energy(st) / energy(e_spat + e_interf + e_artif)),
            'sir': 10 * np.log10(energy(st + e_spat) / energy(e_interf)),
            'sar': 10 * np.log10(energy(st + e_spat + e_interf) / energy(e_artif))}


def test_oracle_against_explicit_least_squares():
    rng = np.random.default_rng(31)
    window, hop, L = 2000, 1500, 64
    s = rng.standard_normal((2, 2, 5000)).astype(np.float32)
    e = (s + 0.3 * s[::-1] + 0.2 * rng.standard_normal(s.shape)).astype(np.float32)
    got = fo.bss_eval_framewise(s, e, window, hop, L)
    nwin = (5000 - window + hop) // hop
    assert nwin == 3
    worst = 0.0
    for w in range(nwin):
        sl = slice(w * hop, w * hop + window)
        want = _lstsq_frame(s[:, :, sl].astype(np.float64), e[:, :, sl].astype(np.float64), L)
        for m in bo.METRICS:
            worst = max(worst, float(np.abs(got[m][:, w] - want[m]).max()))
    assert worst < 1e-9, worst


def test_closed_form_filtered_sources():
    """Abutting frames, every reference silent over the last L samples of each frame, every estimate its own source
    filtered by short FIRs: the estimate lies in the span of the frame's delayed references, so ISR is known in closed
    form and SIR and SAR measure only rounding."""
    rng = np.random.default_rng(32)
    K, C, window, L, taps, nwin = 2, 2, 3000, 64, 40, 3
    N = window * nwin
    s = rng.standard_normal((K, C, N)).astype(np.float32)
    for w in range(nwin):
        s[:, :, (w + 1) * window - L:(w + 1) * window] = 0
    P = np.zeros((K, C, N))
    for j in range(K):
        for i in range(C):
            for c in range(C):
                h = rng.standard_normal(taps) * np.exp(-np.arange(taps) / 8.0) * 0.3
                if c == i:
                    h[0] += 1.0
                P[j, i] += np.convolve(s[j, c].astype(np.float64), h)[:N]
    e = P.astype(np.float32)
    got = fo.bss_eval_framewise(s, e, window, window, L)
    sd = s.astype(np.float64)
    for w in range(nwin):
        sl = slice(w * window, (w + 1) * window)
        want_isr = 10 * np.log10(np.sum(sd[:, :, sl] ** 2, axis=(1, 2)) / np.sum((P - sd)[:, :, sl] ** 2, axis=(1, 2)))
        assert np.abs(got['isr'][:, w] - want_isr).max() < 1e-4, (w, got['isr'][:, w], want_isr)
        assert np.all(got['sir'][:, w] > 100) and np.all(got['sar'][:, w] > 100), (got['sir'][:, w], got['sar'][:, w])


def test_frame_equals_its_slice():
    rng = np.random.default_rng(33)
    window, hop, L = 1500, 1100, 48
    s = rng.standard_normal((2, 1, 5000)).astype(np.float32)
    e = (s + 0.4 * s[::-1] + 0.1 * rng.standard_normal(s.shape)).astype(np.float32)
    whole = fo.bss_eval_framewise(s, e, window, hop, L)
    for w in range(whole['sdr'].shape[1]):
        sl = slice(w * hop, w * hop + window)
        one = fo.bss_eval_framewise(s[:, :, sl], e[:, :, sl], window, hop, L)
        for m in bo.METRICS:
            assert np.array_equal(whole[m][:, w], one[m][:, 0]), (m, w)


def test_silence_rule_and_errors():
    s, e = cases.frame_rules()
    L = 32
    got = fo.bss_eval_framewise(s, e, cases.RULES_WINDOW, cases.RULES_HOP, L)
    nan_frames = [w for w in range(cases.RULES_NWIN) if np.isnan(got['sdr'][:, w]).any()]
    assert nan_frames == list(cases.RULES_NAN_FRAMES)
    for m in bo.METRICS:
        assert got[m].shape == (2, cases.RULES_NWIN)
        assert np.all(np.isnan(got[m][:, list(cases.RULES_NAN_FRAMES)]))
        finite = [w for w in range(cases.RULES_NWIN) if w not in cases.RULES_NAN_FRAMES]
        assert np.all(np.isfinite(got[m][:, finite]))
    load = fo.loading(s, e, cases.RULES_WINDOW, cases.RULES_HOP, L)
    assert load.shape == (cases.RULES_NWIN, 3)
    assert np.all(np.isnan(load[list(cases.RULES_NAN_FRAMES)]))
    assert np.all(load[finite] == bo.LOADING_FIRST)
    with pytest.raises(ValueError, match='filters_len'):
        fo.bss_eval_framewise(s, e, 500, 500, 512)
    with pytest.raises(ValueError, match='shorter than one window'):
        fo.bss_eval_framewise(s[:, :, :900], e[:, :, :900], 1000, 1000, 32)


def test_python_checks_window_before_the_device():
    from lib import bsseval
    s, e = cases.frame_rules()
    with pytest.raises(ValueError, match='filters_len'):
        bsseval.frame_sums(s, e, 500, 500, 512, framewise=True)
    with pytest.raises(ValueError, match='filters_len'):
        bsseval.bss_eval(s, e, 500, 500, 512, framewise=True)


def test_cli_flag(tmp_path):
    import evaluate
    p = evaluate.build_parser()
    assert p.parse_args(['-d', 'x', '-P', 'y']).framewise_filters is False
    assert p.parse_args(['-d', 'x', '-P', 'y', '--framewise_filters']).framewise_filters is True
    data = str(tmp_path / 'data')
    for sub in ('mixtures', 'instruments'):
        os.makedirs(os.path.join(data, sub))
        for base in 'abcde':
            open(os.path.join(data, sub, base + '.wav'), 'wb').close()
    garbage = str(tmp_path / 'not_a_checkpoint.pth')
    with open(garbage, 'w') as f:
        f.write('not a checkpoint')
    # 0.01 s = 441 samples < 512 taps: an argument error, before the model loads
    r = subprocess.run([sys.executable, os.path.join(PKG, 'evaluate.py'), '-d', data, '-P', garbage, '--window', '0.01',
                        '--framewise_filters'], capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 2 and '--framewise_filters' in r.stderr, r.stderr
