"""The Wiener filter oracle (tests/wiener_oracle.py) on the CPU: against a literal per-(bin, frame) loop with
np.linalg.inv, the mixture identity sum_j y_j = x - reg C^-1 x, the no-op, silent and mono-duplicated input, the gain
on a synthetic spatial mixture, and how far a mask error of the GPU's size moves the filtered stems.  Also the
--wiener_iterations flags of inference.py and evaluate.py, without a device."""
import numpy as np
import pytest

import wiener_oracle as wo

# the GPU mask's measured error against the oracle is about 2e-4 (DESIGN.md §7); its gate is 1e-3
MASK_ERROR = 2e-4


def _random(shape, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)


def spatial_case(seed=0, bins=257, T=400):
    """Two sparse gamma-power sources with random phases, panned (0.9, 0.35) and (0.3, 0.95): (X, sources, ratio
    mask averaged over the channels)."""
    rng = np.random.default_rng(seed)
    srcs = []
    for pan in ((0.9, 0.35), (0.3, 0.95)):
        s = np.sqrt(rng.gamma(0.3, 1.0, (bins, T))) * np.exp(2j * np.pi * rng.random((bins, T)))
        srcs.append(np.stack([pan[0] * s, pan[1] * s]).astype(np.complex64))
    X = (srcs[0] + srcs[1]).astype(np.complex64)
    P = [np.mean(np.abs(s) ** 2, axis=0) for s in srcs]
    m = (P[0] / (P[0] + P[1])).astype(np.float32)
    return X, srcs, np.stack([m, m])


def masked(X, m):
    return (m * X).astype(np.complex64), ((1 - m) * X).astype(np.complex64)


def sdr(ref, est):
    return 10 * np.log10(np.sum(np.abs(ref) ** 2) / np.sum(np.abs(ref - est) ** 2))


def _literal_step(x, ys):
    """One iteration as the contract states it, one bin and one frame at a time."""
    bins, T = x.shape[1:]
    out = [np.zeros_like(y) for y in ys]
    for f in range(bins):
        R, v = [], []
        for y in ys:
            vj = [(abs(y[0, f, t]) ** 2 + abs(y[1, f, t]) ** 2) / 2 for t in range(T)]
            S = sum(np.outer(y[:, f, t], y[:, f, t].conj()) for t in range(T))
            R.append(S / (wo.EPS + sum(vj)))
            v.append(vj)
        for t in range(T):
            C = sum(v[j][t] * R[j] for j in range(2)) + wo.REG * np.eye(2)
            Ci = np.linalg.inv(C)
            for j in range(2):
                out[j][:, f, t] = v[j][t] * R[j] @ Ci @ x[:, f, t]
    return out


def test_matches_a_literal_loop():
    X = 30 * _random((2, 5, 7), 1)
    Y = 30 * _random((2, 5, 7), 2)
    V = (X - Y).astype(np.complex64)
    s = wo.scale(X)
    assert s > 1
    x, ys = X.astype(np.complex128) / s, [Y.astype(np.complex128) / s, V.astype(np.complex128) / s]
    for it in range(3):
        want = _literal_step(x, ys)
        got, _ = wo.em_step(x, ys)
        for g, w in zip(got, want):
            assert np.abs(g - w).max() <= 1e-12 * np.abs(w).max(), it
        ys = want
    # wiener() is s times the iterated steps
    y3, v3 = wo.wiener(X, Y, V, 3)
    assert np.abs(y3 - s * ys[0]).max() <= 1e-12 * np.abs(X).max()
    assert np.abs(v3 - s * ys[1]).max() <= 1e-12 * np.abs(X).max()


def test_mixture_identity():
    X, _, m = spatial_case(bins=33, T=50)
    s = wo.scale(X)
    x = X.astype(np.complex128) / s
    ys = [y.astype(np.complex128) / s for y in masked(X, m)]
    for _ in range(2):
        ys, u = wo.em_step(x, ys)
        resid = ys[0] + ys[1] - (x - wo.REG * u)
        assert np.abs(resid).max() <= 1e-12 * np.abs(x).max()


def test_zero_iterations_returns_the_inputs():
    X = _random((2, 9, 11), 3)
    Y, V = _random((2, 9, 11), 4), _random((2, 9, 11), 5)
    for round32 in (False, True):
        y, v = wo.wiener(X, Y, V, 0, round32=round32)
        assert np.array_equal(y, Y) and np.array_equal(v, V)
    with pytest.raises(ValueError):
        wo.wiener(X, Y, V, -1)


def test_silence_and_mono():
    Z = np.zeros((2, 17, 23), np.complex64)
    assert wo.scale(Z) == 1.0
    for round32 in (False, True):
        y, v = wo.wiener(Z, Z, Z, 3, round32=round32)
        assert np.isfinite(y).all() and np.isfinite(v).all() and not y.any() and not v.any()
    # a mono track duplicated to stereo: every R_j is singular, reg keeps C invertible
    mono = 40 * _random((1, 17, 23), 6)
    X = np.concatenate([mono, mono])
    m = np.random.default_rng(7).random((1, 17, 23)).astype(np.float32)
    Y, V = masked(X, np.concatenate([m, m]))
    for round32 in (False, True):
        for it in (1, 3):
            y, v = wo.wiener(X, Y, V, it, round32=round32)
            assert np.isfinite(y).all() and np.isfinite(v).all()
            assert np.array_equal(y[0], y[1]) and np.array_equal(v[0], v[1])


def test_one_iteration_raises_the_sdr():
    """Measured: the ratio mask gives 7.09 / 7.40 dB, one iteration 10.87 / 11.18 dB, three 11.70 / 12.01 dB; the
    mask pulled halfway to 0.5 gives 5.59 / 5.89, 11.87 / 12.17 and 15.74 / 16.04 dB."""
    X, srcs, m = spatial_case()
    for pull, gain in ((0.0, 2.5), (0.5, 5.0)):
        mm = (m + pull * (0.5 - m)).astype(np.float32)
        y0, v0 = masked(X, mm)
        y1, v1 = wo.wiener(X, y0, v0, 1, round32=True)
        y3, v3 = wo.wiener(X, y0, v0, 3, round32=True)
        for ref, e0, e1, e3 in ((srcs[0], y0, y1, y3), (srcs[1], v0, v1, v3)):
            assert sdr(ref, e1) >= sdr(ref, e0) + gain, pull
            assert sdr(ref, e3) >= sdr(ref, e1), pull


def test_mask_error_sensitivity():
    """A mask error of the GPU's size moves the filtered stems by about as much as it moves the masked ones:
    max|dY| / max|X| measured 2.0e-4 after one iteration and 5.1e-4 after three, for +-2e-4 on every mask value.  So
    the end-to-end gate of tests/test_gpu_wiener.py is the mask gate (1e-3) times 1.5 at one iteration."""
    X, _, m = spatial_case()
    rng = np.random.default_rng(5)
    ref = {it: wo.wiener(X, *masked(X, m), it) for it in (1, 3)}
    worst = {1: 0.0, 3: 0.0}
    for _ in range(3):
        mp = (m + rng.choice([-MASK_ERROR, MASK_ERROR], m.shape)).astype(np.float32)
        for it in (1, 3):
            got = wo.wiener(X, *masked(X, mp), it)
            d = max(np.abs(g - r).max() for g, r in zip(got, ref[it])) / np.abs(X).max()
            worst[it] = max(worst[it], d)
    print('wiener sensitivity to a %.0e mask error: %.3g (1 iteration), %.3g (3 iterations)'
          % (MASK_ERROR, worst[1], worst[3]))
    assert worst[1] <= 1.5 * MASK_ERROR
    assert worst[3] <= 4 * MASK_ERROR


def test_cli_flags():
    import evaluate
    import inference
    p = inference.build_parser()
    assert p.parse_args(['-i', 'x.wav']).wiener_iterations == 0
    assert p.parse_args(['-i', 'x.wav', '--wiener_iterations', '3']).wiener_iterations == 3
    assert "norbert's default" in p.format_help()
    e = evaluate.build_parser()
    assert e.parse_args(['-d', 'd', '-P', 'm.pth']).wiener_iterations == 0
    assert e.parse_args(['-d', 'd', '-P', 'm.pth', '--wiener_iterations', '1']).wiener_iterations == 1
    for parser, args in ((p, ['-i', 'x.wav']), (e, ['-d', 'd', '-P', 'm.pth'])):
        with pytest.raises(SystemExit):
            parser.parse_args(args + ['--wiener_iterations', '-1'])
