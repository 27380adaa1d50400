"""BSS Eval on the GPU (run on an H100): lib/bsseval.py against the float64 oracle (oracle/bsseval_oracle.py) on the
analytic cases, references whose Gram matrix is singular (a duplicated channel) or singular to rounding (band-limited),
a separated synthetic pair and the K = 1 / C = 1 shapes; bit-identical repeats; the correlation kernel against explicit
float64 correlations; the error of non-finite input; and evaluate.py end to end, with a mono pair and with two ranks.

The metric gate is 1e-3 dB on every frame value below 100 dB.  Above that (the SIR and SAR of an estimate that lies in
the span of its own references) both sides measure rounding noise, and the test asks only that both stay above 100 dB.
"""
import json
import os
import random
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import bsseval_cases as cases
from conftest import PKG, record_parity

pytestmark = pytest.mark.gpu

SR = cases.SR
GATE_DB = 1e-3


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


def _compare(name, got, want):
    """Same NaN pattern exactly; finite values below 100 dB within GATE_DB; both above 100 dB otherwise."""
    from lib import bsseval
    worst = 0.0
    for m in bsseval.METRICS:
        g, w = got[m], want[m]
        assert g.shape == w.shape, (name, m, g.shape, w.shape)
        assert np.array_equal(np.isnan(g), np.isnan(w)), (name, m)
        ok = ~np.isnan(w)
        high = ok & (w > 100)
        assert np.all(g[high] > 100), (name, m, g[high].min() if high.any() else None)
        low = ok & ~high
        if low.any():
            worst = max(worst, float(np.abs(g[low] - w[low]).max()))
    record_parity('bsseval_%s_max_abs_db' % name, worst, GATE_DB)
    assert worst <= GATE_DB, (name, worst)
    return worst


def _case(name, s, e, window, hop, L):
    from lib import bsseval
    from oracle import bsseval_oracle
    got = bsseval.bss_eval(s, e, window, hop, L)
    want = bsseval_oracle.bss_eval(s, e, window, hop, L)
    return _compare(name, got, want)


def test_spatial_against_oracle():
    s, e = cases.spatial()
    _case('spatial', s, e, SR, SR, 512)


def test_interference_against_oracle():
    s, e = cases.interference()
    _case('interference', s, e, SR, SR, 512)


def test_artifacts_against_oracle():
    s, e, _ = cases.artifacts()
    _case('artifacts', s, e, SR, SR, 512)


def test_frame_rules_against_oracle():
    s, e = cases.frame_rules()
    _case('frame_rules', s, e, cases.RULES_WINDOW, cases.RULES_HOP, 32)


def test_shapes_and_odd_sizes_against_oracle():
    s, e, _ = cases.artifacts(seconds=5.0)
    _case('k1_c2', s[:1], e[:1], SR, SR, 512)                         # one source
    _case('k2_c1', s[:, :1], e[:, :1], SR, SR, 512)                   # mono
    _case('k1_c1', s[:1, :1], e[:1, :1], SR // 2, SR // 4, 100)       # overlapping frames, L not a tile multiple
    _case('k2_c2_gaps', s, e, 20000, 30000, 1024)                     # hop > window, the longest filter


@pytest.mark.parametrize('case', ['duplicated', 'band_limited'])
def test_semidefinite_gram_against_oracle(case):
    """Systems that 2^-52 of max diag G does not factor: the GPU factors them at the schedule's first loading, as
    the oracle's LAPACK Cholesky does, and the metrics agree within the gate."""
    from lib import bsseval
    from oracle import bsseval_oracle
    s, e = getattr(cases, case)()
    out = bsseval.frame_sums(s, e, SR, SR, 512)
    R = bsseval_oracle.correlations(s.astype(np.float64), e.astype(np.float64), 512)
    G = bsseval_oracle.gram(R, 512)
    base = np.max(np.diag(G))
    want_scales = [bsseval_oracle.loading_scale(G, base)] + [
        bsseval_oracle.loading_scale(G[j * 1024:(j + 1) * 1024, j * 1024:(j + 1) * 1024], base) for j in range(2)]
    assert out['loading'].tolist() == want_scales == [bsseval_oracle.LOADING_FIRST] * 3, (out['loading'], want_scales)
    got = bsseval.metrics(out['sums'])
    assert all(np.isfinite(got[m]).all() for m in bsseval.METRICS)
    _compare(case, got, bsseval_oracle.bss_eval(s, e, SR, SR, 512))


def _separated_pair(model, seconds=30.0):
    """Instruments and vocals of a synthetic 30 s pair, and the seeded checkpoint's estimates of both."""
    import inference
    from lib import synth
    inst = 0.5 * synth.sine_mix(seconds, seed=1)
    voc = 0.5 * synth.sine_mix(seconds / 2, sr=2 * SR, seed=2)[:, :inst.shape[1]]   # the same sines an octave down
    X = (inst + voc).astype(np.float32)
    sp = inference.Separator(model, _dev(), 4, 256, False)
    est_i, est_v = sp.separate_wave(X)
    n = est_i.shape[1]
    return np.stack([inst[:, :n], (X - inst)[:, :n]]), np.stack([est_i, est_v])


def test_separated_pair_against_oracle(model):
    s, e = _separated_pair(model)
    _case('sine_mix_30s', s, e, SR, SR, 512)


def test_deterministic(model):
    from lib import bsseval
    s, e = _separated_pair(model, 10.0)
    a = bsseval.frame_sums(s, e, SR, SR, 512)['sums']
    b = bsseval.frame_sums(torch.from_numpy(s).to(_dev()), torch.from_numpy(e).to(_dev()), SR, SR, 512)['sums']
    assert a.tobytes() == b.tobytes()


def test_correlations_against_explicit_float64():
    from lib import bsseval
    from oracle import bsseval_oracle
    s, e = cases.interference(seconds=5.0)
    L = 512
    got = bsseval.frame_sums(s, e, SR, SR, L, correlations=True)['corr']
    want = bsseval_oracle.correlations(s.astype(np.float64), e.astype(np.float64), L)
    # fp64 rounding of N-term sums, on the scale Cauchy-Schwarz gives every r[a][b](l)
    M = s.shape[0] * s.shape[1]
    y = np.concatenate([s.reshape(M, -1), e.reshape(M, -1)]).astype(np.float64)
    scale = np.sqrt(np.sum(y[:M] ** 2, axis=1)[:, None] * np.sum(y ** 2, axis=1)[None, :])[:, :, None]
    err = float((np.abs(got - want) / scale).max())
    record_parity('bsseval_correlation_rel_err', err, 1e-13)
    assert err < 1e-13


def test_non_finite_input_is_an_error():
    from lib import _native, bsseval
    s, e = cases.interference(seconds=2.0)
    dev = _dev()
    for which in (0, 1):
        x = [s.copy(), e.copy()]
        x[which][1, 0, 1000] = np.nan if which else np.inf
        with pytest.raises(ValueError, match='NaN or Inf'):
            bsseval.bss_eval(x[0], x[1], SR, SR, 64)
        with pytest.raises(ValueError, match='NaN or Inf'):   # device tensors are checked on the device
            bsseval.bss_eval(torch.from_numpy(x[0]).to(dev), torch.from_numpy(x[1]).to(dev), SR, SR, 64)
    # the C entry point checks on its own
    lib = _native.load_library()
    bad = torch.from_numpy(e).to(dev)
    bad[0, 1, 5] = float('nan')
    ref = torch.from_numpy(s).to(dev)
    nbytes = lib.vr_bss_eval_workspace(2, 2, s.shape[2], 64, SR, SR)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    sums = np.empty((2, 2, 8))
    rc = lib.vr_bss_eval(None, _native.ptr(ref), _native.ptr(bad), 2, 2, s.shape[2], 64, SR, SR, _native.ptr(ws), nbytes,
                         sums.ctypes.data, None, None, None, _native.stream_ptr())
    assert rc != 0 and b'NaN or Inf' in lib.vr_last_error(None)
    assert np.isfinite(bsseval.bss_eval(s, e, SR, SR, 64)['sdr']).all()   # and the next call is fine


# ---- evaluate.py -------------------------------------------------------------------------------------------------
def _write_pairs(root, layout, seconds=6.0, mono=()):
    """{subdir: [pair indices]} -> WAV pairs (mixture = instruments + vocals) under root/subdir/{mixtures,instruments};
    the pairs with an index in ``mono`` are written as mono files (the left channel)."""
    from lib import audio_io, synth
    pairs = {}
    for sub, idx in layout.items():
        for k in idx:
            inst = 0.4 * synth.sine_mix(seconds, seed=10 + k)
            voc = 0.4 * synth.sine_mix(seconds / (2 + k % 2), sr=(2 + k % 2) * SR, seed=20 + k)[:, :inst.shape[1]]
            pair = []
            for kind, w in (('mixtures', inst + voc), ('instruments', inst)):
                d = os.path.join(root, sub, kind)
                os.makedirs(d, exist_ok=True)
                path = os.path.join(d, 'track%d.wav' % k)
                audio_io.write(path, w[0] if k in mono else w.T, SR)
                pair.append(path)
            pairs.setdefault(sub, []).append(pair)
    return pairs


def _parse(stdout):
    lines = stdout.strip().splitlines()
    pairs = [l for l in lines if re.match(r'\d+ \S+\.wav \S+\.wav instruments SDR ', l)]
    assert lines[-1].startswith('median of %d pairs: ' % len(pairs)), r.stdout
    return pairs, lines[-1]


def _cli(*args):
    r = subprocess.run([sys.executable, os.path.join(PKG, 'evaluate.py'), '-g', '0'] + list(args),
                       capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 0, r.stderr
    return _parse(r.stdout)


def test_cli_end_to_end(model, tmp_path):
    import evaluate
    import inference
    import validate
    from lib import bsseval, dataset, synth
    dev = _dev()
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)

    def direct(filelist, tta=False, postprocess=False):
        sp = inference.Separator(model, dev, 4, 256, postprocess)
        out = []
        for X_path, y_path in filelist:
            X, y = evaluate.pair_waves(X_path, y_path, SR, 0)
            out.append(evaluate.score_pair(sp, X, y, SR, SR, 512, tta))
        return out

    def expect_lines(filelist, results):
        return (['{} {} {}'.format(i + 1, validate.pair_name(*pair), evaluate.format_values(bsseval.track_medians(r)))
                 for i, (pair, r) in enumerate(zip(filelist, results))],
                'median of {} pairs: {}'.format(len(results), evaluate.format_values(evaluate.dataset_medians(results))))

    # random split: the reference's shuffle of 4 pairs with seed 3, half of them scored
    flat = _write_pairs(str(tmp_path / 'flat'), {'': [0, 1, 2, 3]})['']
    random.seed(3)
    _, val = dataset.train_val_split(str(tmp_path / 'flat'), 'random', 0.5, [])
    val = [list(p) for p in val]
    assert len(val) == 2
    res = direct(val)
    js = str(tmp_path / 'frames.json')
    pairs, last = _cli('-d', str(tmp_path / 'flat'), '-P', ckpt, '-s', '3', '-v', '0.5', '--json', js)
    want_pairs, want_last = expect_lines(val, res)
    assert pairs == want_pairs and last == want_last
    with open(js) as f:
        doc = json.load(f)
    assert [[t['mixture'], t['instruments']] for t in doc['tracks']] == val
    for t, r in zip(doc['tracks'], res):
        for k, stem in enumerate(evaluate.STEMS):
            for m in ('sdr', 'isr', 'sir', 'sar'):
                got = np.array([np.nan if v is None else v for v in t['frames'][stem][m]])
                assert got.shape == r[m][k].shape and got.size >= 4
                assert np.array_equal(got, r[m][k], equal_nan=True)
    med = evaluate.dataset_medians(res)
    assert doc['median']['vocals']['sdr'] == pytest.approx(float(med['sdr'][1]), abs=0)

    # -t and -p: the estimates of Separator(postprocess=True).separate_wave(X, tta=True)
    res_tp = direct(val, tta=True, postprocess=True)
    pairs_tp, last_tp = _cli('-d', str(tmp_path / 'flat'), '-P', ckpt, '-s', '3', '-v', '0.5', '-t', '-p')
    assert (pairs_tp, last_tp) == expect_lines(val, res_tp)
    assert pairs_tp != pairs

    # --val_filelist: the given pairs, in the given order
    vlist = str(tmp_path / 'val.json')
    with open(vlist, 'w') as f:
        json.dump([flat[3], flat[1]], f)
    pairs, last = _cli('-d', str(tmp_path / 'flat'), '-P', ckpt, '-V', vlist)
    assert (pairs, last) == expect_lines([flat[3], flat[1]], direct([flat[3], flat[1]]))

    # subdirs: validation/ only
    sub = _write_pairs(str(tmp_path / 'split'), {'training': [0], 'validation': [1, 2, 3]})
    pairs, last = _cli('-d', str(tmp_path / 'split'), '-P', ckpt, '-S', 'subdirs')
    assert (pairs, last) == expect_lines(sub['validation'], direct(sub['validation']))


def test_cli_mono_pair_and_two_ranks(model, tmp_path):
    """A mono pair (duplicated to two channels, so its Gram matrix is singular) scores like any other, and two gloo
    ranks sharing the GPU print exactly what one rank prints."""
    import socket
    import evaluate
    import inference
    import validate
    from lib import bsseval, synth
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
    pairs = _write_pairs(str(tmp_path / 'data'), {'': [0, 1, 2]}, mono=(1,))['']
    sp = inference.Separator(model, _dev(), 4, 256, False)
    results = []
    for X_path, y_path in pairs:
        X, y = evaluate.pair_waves(X_path, y_path, SR, 0)
        results.append(evaluate.score_pair(sp, X, y, SR, SR, 512))
    assert all(np.isfinite(results[1][m]).all() for m in bsseval.METRICS)
    want = (['{} {} {}'.format(i + 1, validate.pair_name(*pair), evaluate.format_values(bsseval.track_medians(r)))
             for i, (pair, r) in enumerate(zip(pairs, results))],
            'median of 3 pairs: ' + evaluate.format_values(evaluate.dataset_medians(results)))
    args = ['-d', str(tmp_path / 'data'), '-P', ckpt, '--all']
    assert _cli(*args) == want

    with socket.socket() as sock:
        sock.bind(('127.0.0.1', 0))
        port = sock.getsockname()[1]
    procs = []
    for rank in range(2):
        env = dict(os.environ, WORLD_SIZE='2', RANK=str(rank), LOCAL_RANK='0', MASTER_ADDR='127.0.0.1',
                   MASTER_PORT=str(port), GLOO_SOCKET_IFNAME='lo')
        procs.append(subprocess.Popen([sys.executable, os.path.join(PKG, 'evaluate.py')] + args, cwd=PKG, env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    outs = [p.communicate(timeout=600) for p in procs]
    for p, (_, err) in zip(procs, outs):
        assert p.returncode == 0, err
    assert _parse(outs[0][0]) == want
    assert outs[1][0].strip() == ''   # rank 1 prints nothing
