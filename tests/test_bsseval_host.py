"""BSS Eval without a GPU: the float64 oracle (oracle/bsseval_oracle.py) on signals with known answers, the frame and
NaN rules, the errors of the oracle and of lib/bsseval.py's host-side checks, the median rules, and the evaluate.py
command line up to the point where it needs a device."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import bsseval_cases as cases
from conftest import PKG

SR = cases.SR


def test_spatial_distortion_only():
    from oracle import bsseval_oracle
    s, e = cases.spatial()
    r = bsseval_oracle.bss_eval(s, e, SR, SR, 512)
    nwin = r['sdr'].shape[1]
    assert nwin == 5
    direct = 10 * np.log10(cases.frame_energy(s, SR, SR, nwin) / cases.frame_energy(e.astype(np.float64) - s, SR, SR, nwin))
    np.testing.assert_allclose(r['isr'], direct, rtol=0, atol=1e-6)
    np.testing.assert_allclose(r['sdr'], direct, rtol=0, atol=1e-6)
    assert np.all(r['sir'] > 100) and np.all(r['sar'] > 100), (r['sir'].min(), r['sar'].min())


def test_interference():
    from oracle import bsseval_oracle
    alpha = 0.3
    s, e = cases.interference(alpha)
    r = bsseval_oracle.bss_eval(s, e, SR, SR, 512)
    nwin = r['sir'].shape[1]
    want = 10 * np.log10(cases.frame_energy(s, SR, SR, nwin) / cases.frame_energy(alpha * s[::-1].astype(np.float64),
                                                                                  SR, SR, nwin))
    assert np.abs(r['sir'] - want).max() < 0.1, np.abs(r['sir'] - want).max()


def test_artifacts():
    from oracle import bsseval_oracle
    s, e, n = cases.artifacts()
    r = bsseval_oracle.bss_eval(s, e, SR, SR, 512)
    nwin = r['sar'].shape[1]
    snr = 10 * np.log10(cases.frame_energy(s, SR, SR, nwin) / cases.frame_energy(n, SR, SR, nwin))
    assert np.abs(r['sar'] - snr).max() < 0.1, np.abs(r['sar'] - snr).max()


def test_frame_rules():
    from lib import bsseval
    from oracle import bsseval_oracle
    s, e = cases.frame_rules()
    assert bsseval.frame_count(cases.RULES_N, cases.RULES_WINDOW, cases.RULES_HOP) == cases.RULES_NWIN
    r = bsseval_oracle.bss_eval(s, e, cases.RULES_WINDOW, cases.RULES_HOP, 32)
    for m in bsseval.METRICS:
        assert r[m].shape == (2, cases.RULES_NWIN)
        nan_cols = sorted(set(np.flatnonzero(np.isnan(r[m]).any(axis=0)).tolist()))
        assert nan_cols == list(cases.RULES_NAN_FRAMES), (m, nan_cols)
        assert np.isnan(r[m][:, list(cases.RULES_NAN_FRAMES)]).all()
    # one window exactly: one frame; a hop longer than the window leaves gaps
    assert bsseval.frame_count(1000, 1000, 300) == 1
    assert bsseval.frame_count(10000, 1000, 3000) == 4


@pytest.mark.parametrize('case', ['duplicated', 'band_limited'])
def test_semidefinite_gram_gets_a_larger_loading(case):
    """A singular (duplicated channel) or numerically singular (band-limited) Gram matrix has no Cholesky factor at
    2^-52 of its largest diagonal value; the first loading of the schedule, 2^-40, factors it, and the metrics are
    finite."""
    from oracle import bsseval_oracle
    s, e = getattr(cases, case)()
    L = 512
    R = bsseval_oracle.correlations(s.astype(np.float64), e.astype(np.float64), L)
    G = bsseval_oracle.gram(R, L)
    base = np.max(np.diag(G))
    with pytest.raises(np.linalg.LinAlgError):
        np.linalg.cholesky(G + 2.0 ** -52 * base * np.eye(G.shape[0]))
    assert bsseval_oracle.loading_scale(G, base) == bsseval_oracle.LOADING_FIRST
    r = bsseval_oracle.bss_eval(s, e, SR, SR, L)
    assert all(np.isfinite(r[m]).all() for m in bsseval_oracle.METRICS)
    # the interference is 0.3 of the other source: SIR near 10 log10(1 / 0.09) in every frame
    assert np.abs(r['sir'] - 10 * np.log10(1 / 0.09)).max() < 0.5


def test_metrics_from_sums_and_medians():
    from lib import bsseval
    q = np.ones((2, 3, 8))
    q[..., 1] = 0.1    # ISR 10 dB
    q[..., 2] = 0.01   # SDR 20 dB
    q[..., 4] = 1e-3   # SIR 30 dB
    q[..., 6] = 1e-4   # SAR 40 dB
    q[1, 1, 7] = 0     # source 1's estimate silent in frame 1: frame 1 NaN for both sources
    r = bsseval.metrics(q)
    np.testing.assert_allclose(r['isr'][:, [0, 2]], 10)
    np.testing.assert_allclose(r['sdr'][:, [0, 2]], 20)
    np.testing.assert_allclose(r['sir'][:, [0, 2]], 30)
    np.testing.assert_allclose(r['sar'][:, [0, 2]], 40)
    assert all(np.isnan(r[m][:, 1]).all() for m in bsseval.METRICS)
    med = bsseval.track_medians({'sdr': np.array([[1.0, np.nan, 3.0, 10.0], [np.nan] * 4]),
                                 'isr': np.zeros((2, 4)), 'sir': np.zeros((2, 4)), 'sar': np.zeros((2, 4))})
    assert med['sdr'][0] == 3.0 and np.isnan(med['sdr'][1])


def test_errors():
    from lib import bsseval
    from oracle import bsseval_oracle
    s = np.ones((2, 2, 1000), np.float32)
    for fn in (bsseval_oracle.bss_eval, bsseval.bss_eval):
        with pytest.raises(ValueError, match='shape'):
            fn(s, s[:, :, :999], 100, 100)
        with pytest.raises(ValueError, match='shape'):
            fn(s[0], s[0], 100, 100)
        with pytest.raises(ValueError, match='shorter than one window'):
            fn(s, s, 1001, 100)
        with pytest.raises(ValueError, match='every reference is zero'):
            fn(np.zeros_like(s), s, 100, 100)
        bad = s.copy()
        bad[1, 0, 500] = np.nan
        with pytest.raises(ValueError, match='NaN or Inf'):
            fn(s, bad, 100, 100)
        bad[1, 0, 500] = np.inf
        with pytest.raises(ValueError, match='NaN or Inf'):
            fn(bad, s, 100, 100)
    with pytest.raises(ValueError, match='K \\* C'):
        bsseval.bss_eval(np.ones((3, 3, 1000), np.float32), np.ones((3, 3, 1000), np.float32), 100, 100)
    with pytest.raises(ValueError, match='filters_len'):
        bsseval.bss_eval(s, s, 100, 100, filters_len=1025)
    with pytest.raises(ValueError, match='window and hop'):
        bsseval.bss_eval(s, s, 100, 0)


def _listing(root, names):
    for sub in ('mixtures', 'instruments'):
        os.makedirs(os.path.join(root, sub))
        for base in names:
            open(os.path.join(root, sub, base + '.wav'), 'wb').close()


def _cli(*args):
    return subprocess.run([sys.executable, os.path.join(PKG, 'evaluate.py')] + list(args), capture_output=True,
                          text=True, cwd=PKG)


def test_cli_errors_come_before_the_model_loads(tmp_path):
    data = str(tmp_path / 'data')
    _listing(data, ['a', 'b', 'c', 'd', 'e'])
    garbage = str(tmp_path / 'not_a_checkpoint.pth')
    with open(garbage, 'w') as f:
        f.write('not a checkpoint')
    vlist = str(tmp_path / 'val.json')
    with open(vlist, 'w') as f:
        json.dump([['x.wav', 'y.wav']], f)

    r = _cli('-d', data)
    assert r.returncode == 2 and '--pretrained_model/-P' in r.stderr
    r = _cli('-d', data, '-P', str(tmp_path / 'missing.pth'))
    assert r.returncode == 2 and 'no such file' in r.stderr
    r = _cli('-d', data, '-P', garbage, '-S', 'subdirs', '-V', vlist)
    assert r.returncode == 2 and '`val_filelist` option is not available with `subdirs` mode' in r.stderr
    r = _cli('-d', str(tmp_path / 'nowhere'), '-P', garbage)
    assert r.returncode == 2 and 'nowhere' in r.stderr
    r = _cli('-d', data, '-P', garbage, '-c', '128')
    assert r.returncode == 2 and '--cropsize' in r.stderr
    r = _cli('-d', data, '-P', garbage, '-B', '0')
    assert r.returncode == 2 and '--batchsize' in r.stderr
    r = _cli('-d', data, '-P', garbage, '--hop', '0')
    assert r.returncode == 2 and '--window and --hop' in r.stderr
    r = _cli('-d', data, '-P', garbage, '--filters_len', '2000')
    assert r.returncode == 2 and '--filters_len' in r.stderr
    r = _cli('-d', data, '-P', garbage, '--json', str(tmp_path / 'no' / 'dir.json'))
    assert r.returncode == 2 and '--json' in r.stderr
    r = _cli('-d', data, '-P', garbage, '-E', '3')
    assert r.returncode == 2 and 'unrecognized arguments' in r.stderr


def test_cli_pair_selection(tmp_path):
    import argparse
    import evaluate
    data = str(tmp_path / 'data')
    _listing(data, ['a', 'b', 'c', 'd', 'e'])
    p = evaluate.build_parser()
    val = evaluate.select_pairs(p, p.parse_args(['-d', data, '-P', 'x', '-s', '3', '-v', '0.4']))
    assert len(val) == 2
    every = evaluate.select_pairs(p, p.parse_args(['-d', data, '-P', 'x', '--all']))
    assert [os.path.basename(a) for a, _ in every] == ['a.wav', 'b.wav', 'c.wav', 'd.wav', 'e.wav']
    assert all(pair in every for pair in val)
    args = p.parse_args(['-d', data, '-P', 'x'])
    assert (args.window, args.hop, args.filters_len, args.json, args.all) == (1.0, 1.0, 512, None, False)
    assert isinstance(args, argparse.Namespace)


def test_cli_without_gpu_fails_on_cuda_after_the_split(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    data = str(tmp_path / 'data')
    _listing(data, ['a', 'b', 'c', 'd', 'e'])
    garbage = str(tmp_path / 'not_a_checkpoint.pth')
    with open(garbage, 'w') as f:
        f.write('not a checkpoint')
    r = _cli('-d', data, '-P', garbage)
    assert r.returncode != 0 and 'RuntimeError: no CUDA device' in r.stderr
