"""BSS Eval v3 (framewise filters) on the GPU (run on an H100): lib/bsseval.py's ``framewise=True`` against the
float64 oracle (tests/bsseval_framewise_oracle.py) on the analytic, odd-size, semidefinite and separated cases; bit
identity for every batch size and across calls; each frame's loadings and correlations; silent frames; and
evaluate.py --framewise_filters end to end.

The gate is that of tests/test_gpu_bsseval.py: 1e-3 dB on every frame value below 100 dB, and both above 100 dB
otherwise.
"""
import json
import os

import numpy as np
import pytest
import torch

import bsseval_cases as cases
import bsseval_framewise_oracle as fo
from conftest import record_parity
from oracle import bsseval_oracle as bo
from test_gpu_bsseval import _cli, _compare, _separated_pair, _write_pairs

pytestmark = pytest.mark.gpu

SR = cases.SR


def _dev():
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def model():
    from lib import nets, synth
    m = nets.CascadedNet(2048, 1024, 32, 128)
    m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    m.to(_dev())
    return m


@pytest.fixture(scope='module')
def separated(model):
    return _separated_pair(model)


def _case(name, s, e, window, hop, L):
    from lib import bsseval
    got = bsseval.bss_eval(s, e, window, hop, L, framewise=True)
    want = fo.bss_eval_framewise(s, e, window, hop, L)
    return _compare('framewise_' + name, got, want)


def _odd(name):
    s, e, _ = cases.artifacts(seconds=5.0)
    return {'k1_c1': (s[:1, :1], e[:1, :1], SR // 2, SR // 4, 100),      # overlapping frames, L not a tile multiple
            'k2_c1': (s[:, :1], e[:, :1], SR, SR, 512),                   # mono
            'k2_c2_gaps': (s, e, 20000, 30000, 1024)}[name]               # hop > window, the longest filter


@pytest.mark.parametrize('name', ['spatial', 'interference', 'artifacts', 'frame_rules', 'duplicated',
                                  'band_limited', 'k1_c1', 'k2_c1', 'k2_c2_gaps'])
def test_against_oracle(name):
    if name == 'spatial':
        s, e = cases.spatial()
        args = (SR, SR, 512)
    elif name in ('interference', 'artifacts'):
        s, e = getattr(cases, name)(seconds=5.0)[:2]
        args = (SR, SR, 512)
    elif name == 'frame_rules':
        s, e = cases.frame_rules()
        args = (cases.RULES_WINDOW, cases.RULES_HOP, 32)
    elif name in ('duplicated', 'band_limited'):
        s, e = getattr(cases, name)()
        args = (SR, SR, 512)
    else:
        s, e, *args = _odd(name)
    _case(name, s, e, *args)


def test_separated_pair_against_oracle(separated):
    s, e = separated
    _case('sine_mix_30s', s, e, SR, SR, 512)


def _sums(s, e, frames_per_batch, correlations=True):
    from lib import bsseval
    return bsseval.frame_sums(s, e, SR, SR, 512, correlations=correlations, framewise=True,
                              frames_per_batch=frames_per_batch)


@pytest.mark.parametrize('name', ['separated', 'duplicated', 'band_limited'])
def test_bit_identical_for_every_batch(name, request):
    from lib import bsseval
    s, e = request.getfixturevalue('separated') if name == 'separated' else getattr(cases, name)()
    nwin = bsseval.frame_count(s.shape[2], SR, SR)
    first = _sums(s, e, 1)
    for fpb in (7, nwin, nwin):
        out = _sums(s, e, fpb)
        for k in ('sums', 'corr', 'loading'):
            assert out[k].tobytes() == first[k].tobytes(), (name, fpb, k)
    auto = bsseval.frame_sums(s, e, SR, SR, 512, framewise=True)
    assert 1 <= auto['frames_per_batch'] <= nwin
    assert auto['sums'].tobytes() == first['sums'].tobytes()


@pytest.mark.parametrize('name', ['duplicated', 'band_limited'])
def test_loading_of_every_frame(name):
    s, e = getattr(cases, name)()
    got = _sums(s, e, None, correlations=False)['loading']
    want = fo.loading(s, e, SR, SR, 512)
    assert got.shape == want.shape and np.array_equal(got, want), (got, want)


def test_correlations_against_explicit_float64():
    from lib import bsseval
    s, e = cases.interference(seconds=3.0)
    window, hop, L = SR, SR // 2, 512
    got = bsseval.frame_sums(s, e, window, hop, L, correlations=True, framewise=True, frames_per_batch=2)['corr']
    nwin = bsseval.frame_count(s.shape[2], window, hop)
    assert got.shape == (nwin, 4, 8, L)
    M = 4
    worst = 0.0
    for w in range(nwin):
        ss = s[:, :, w * hop:w * hop + window].astype(np.float64)
        ee = e[:, :, w * hop:w * hop + window].astype(np.float64)
        want = bo.correlations(ss, ee, L)
        y = np.concatenate([ss.reshape(M, -1), ee.reshape(M, -1)])
        scale = np.sqrt(np.sum(y[:M] ** 2, axis=1)[:, None] * np.sum(y ** 2, axis=1)[None, :])[:, :, None]
        worst = max(worst, float((np.abs(got[w] - want) / scale).max()))
    record_parity('bsseval_framewise_correlation_rel_err', worst, 1e-13)
    assert worst < 1e-13


def test_silent_vocals_intro():
    """Vocals silent through the first three seconds: those frames are NaN, the rest finite, no error."""
    from lib import bsseval
    rng = np.random.default_rng(41)
    s = rng.standard_normal((2, 2, 8 * SR)).astype(np.float32)
    s[1, :, :3 * SR] = 0
    e = (s + 0.3 * s[::-1] + 0.1 * rng.standard_normal(s.shape)).astype(np.float32)
    out = _sums(s, e, 3, correlations=False)
    got = bsseval.metrics(out['sums'])
    for m in bsseval.METRICS:
        assert np.all(np.isnan(got[m][:, :3])) and np.all(np.isfinite(got[m][:, 3:])), m
    assert np.all(np.isnan(out['loading'][:3])) and np.all(out['loading'][3:] == bo.LOADING_FIRST)
    _compare('framewise_silent_intro', got, fo.bss_eval_framewise(s, e, SR, SR, 512))


def test_cli_end_to_end(model, tmp_path):
    import evaluate
    import inference
    import validate
    from lib import bsseval, synth
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
    pairs = _write_pairs(str(tmp_path / 'data'), {'': [0, 1]})['']
    sp = inference.Separator(model, _dev(), 4, 256, False)

    def expect(framewise):
        res = []
        for X_path, y_path in pairs:
            X, y = evaluate.pair_waves(X_path, y_path, SR, 0)
            res.append(evaluate.score_pair(sp, X, y, SR, SR, 512, framewise=framewise))
        lines = (['{} {} {}'.format(i + 1, validate.pair_name(*pair), evaluate.format_values(bsseval.track_medians(r)))
                  for i, (pair, r) in enumerate(zip(pairs, res))],
                 'median of {} pairs: {}'.format(len(res), evaluate.format_values(evaluate.dataset_medians(res))))
        return res, lines

    for framewise in (True, False):
        js = str(tmp_path / ('v3.json' if framewise else 'v4.json'))
        flag = ['--framewise_filters'] if framewise else []
        got = _cli('-d', str(tmp_path / 'data'), '-P', ckpt, '--all', '--json', js, *flag)
        res, lines = expect(framewise)
        assert got == lines, (framewise, got, lines)
        with open(js) as f:
            doc = json.load(f)
        assert doc.get('framewise_filters') is (True if framewise else None)
        for t, r in zip(doc['tracks'], res):
            for k, stem in enumerate(evaluate.STEMS):
                for m in bsseval.METRICS:
                    v = np.array([np.nan if x is None else x for x in t['frames'][stem][m]])
                    assert np.array_equal(v, r[m][k], equal_nan=True), (framewise, stem, m)
    # the two modes are different metrics
    assert expect(True)[1] != expect(False)[1]
