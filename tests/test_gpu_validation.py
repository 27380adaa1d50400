"""validate.py on the GPU (run on an H100): vr_validation_loss against the reference's own per-patch losses
(tests/golden/ref_validation, oracle/validation_oracle.py), the L1 kernel against a float64 numpy sum over the mask
the net gives, determinism, a silent pair, and the CLI in its three split modes.

The gate of patch j follows from the mask gate of the separation parity tests (max |mask - reference| < 1e-3):
|m'x - y| and |mx - y| differ by at most |m' - m| x, so the two losses differ by at most 1e-3 * mean_j(|X| / coef)
over the patch's (2, bins, roi) kept frames.
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

from conftest import PKG, load_golden, record_parity

pytestmark = pytest.mark.gpu

ROI = 128


def _dev():
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def golden_validation():
    return load_golden('ref_validation')


@pytest.fixture(scope='module')
def model():
    from lib import nets, synth
    m = nets.CascadedNet(2048, 1024, 32, 128)
    m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    m.to(_dev())
    return m


@pytest.fixture(scope='module')
def specs():
    from oracle import validation_oracle
    return validation_oracle.spectrograms()


def _patch_gates(X, y):
    """1e-3 * mean over (2, bins, roi) of |X| / coef per patch (frames past T count as zero)."""
    coef = max(np.abs(X).max(), np.abs(y).max())
    a = np.abs(X).astype(np.float64) / coef
    n = -(-X.shape[2] // ROI)
    a = np.pad(a, ((0, 0), (0, 0), (0, n * ROI - X.shape[2])))
    return 1e-3 * a.reshape(2, X.shape[1], n, ROI).mean(axis=(0, 1, 3))


def test_patch_losses_match_reference(model, specs, golden_validation):
    import validate
    g = golden_validation
    v = validate.Validator(model, _dev(), 256, 4)
    got, gates, sums = [], [], []
    for name, X, y in specs:
        s = v.window_sums(X, y, name)
        assert s.dtype == np.float64 and s.shape == (-(-X.shape[2] // ROI),), (name, s.shape)
        sums.append(s)
        got.append(v.patch_losses(s))
        gates.append(_patch_gates(X, y))
    got, gates = np.concatenate(got), np.concatenate(gates)
    err = np.abs(got - g['patch_losses'])
    record_parity('validation_patch_loss_max_abs_err', err.max())
    record_parity('validation_patch_loss_err_over_gate', (err / gates).max(), 1.0)
    assert np.all(err <= gates), (err, gates)
    total = validate.combine(v, sums)
    total_err = abs(total - float(g['total_b4']))
    record_parity('validation_total_b4_abs_err', total_err, gates.mean())
    assert total_err <= gates.mean()


def test_kernel_matches_float64_sum_over_the_mask(model, specs):
    """The mask from vr_separate_windows with the same normaliser and padding, then the L1 sums in float64 numpy."""
    from lib import _native
    dev = _dev()
    ctx = model.native_context(256, 4)
    worst = 0.0
    for name, X, y in specs:
        T = X.shape[2]
        n = -(-T // ROI)
        d_x, d_y = torch.from_numpy(X).to(dev), torch.from_numpy(y).to(dev)
        coef = torch.empty(1, dtype=torch.float32, device=dev)
        sums = torch.empty(n, dtype=torch.float64, device=dev)
        ctx.check(ctx.lib.vr_validation_loss(ctx.handle, _native.ptr(d_x), _native.ptr(d_y), T, _native.ptr(coef),
                                             _native.ptr(sums), _native.stream_ptr()), 'vr_validation_loss')
        c = float(coef.item())
        np.testing.assert_allclose(c, max(np.abs(X).max(), np.abs(y).max()), rtol=1e-6)
        mask = torch.empty((2, X.shape[1], n * ROI), dtype=torch.float32, device=dev)
        ctx.check(ctx.lib.vr_separate_windows(ctx.handle, _native.ptr(d_x), T, _native.ptr(coef), 64, 0, n,
                                              _native.ptr(mask), n * ROI, 0, 0, _native.stream_ptr()),
                  'vr_separate_windows')
        m = mask.cpu().numpy().astype(np.float64)[:, :, :T]
        terms = np.abs(m * np.abs(X).astype(np.float64) / c - np.abs(y).astype(np.float64) / c)
        terms = np.pad(terms, ((0, 0), (0, 0), (0, n * ROI - T)))
        want = terms.reshape(2, X.shape[1], n, ROI).sum(axis=(0, 1, 3))
        rel = np.abs(sums.cpu().numpy() - want) / want
        worst = max(worst, float(rel.max()))
    record_parity('validation_kernel_vs_float64_rel_err', worst, 1e-6)
    assert worst < 1e-6


def test_deterministic_and_batch_size(model, specs):
    import validate
    dev = _dev()
    v4 = validate.Validator(model, dev, 256, 4)
    v1 = validate.Validator(model, dev, 256, 1)
    gap = 0.0
    for name, X, y in specs:
        a = v4.window_sums(X, y, name)
        b = v4.window_sums(torch.from_numpy(X).to(dev), torch.from_numpy(y).to(dev), name)
        assert a.tobytes() == b.tobytes(), name   # bit-identical from call to call, host or device input
        c = v1.window_sums(X, y, name)
        gap = max(gap, float((np.abs(c - a) / a).max()))
    record_parity('validation_batch1_vs_batch4_rel_gap', gap, 1e-5)
    assert gap < 1e-5


def test_silent_pair_raises_and_leaves_the_context_clean(model, specs, golden_validation):
    import validate
    v = validate.Validator(model, _dev(), 256, 4)
    name, X, y = specs[0]
    first = v.window_sums(X, y, name)
    silent = np.zeros((2, 1025, 200), np.complex64)
    with pytest.raises(ValueError, match='quiet.wav quiet_inst.wav'):
        v.window_sums(silent, silent, 'quiet.wav quiet_inst.wav')
    again = v.window_sums(X, y, name)
    assert again.tobytes() == first.tobytes()
    n = len(first)
    gates = _patch_gates(X, y)
    assert np.all(np.abs(v.patch_losses(again) - golden_validation['patch_losses'][:n]) <= gates)


def _dataset(root, specs, layout):
    """Empty audio files plus the reference's spectrogram caches; layout: {subdir: [pair indices]}."""
    pairs = {}
    for sub, idx in layout.items():
        for k in idx:
            name, X, y = specs[k]
            pair = []
            for kind, s in (('mixtures', X), ('instruments', y)):
                d = os.path.join(root, sub, kind)
                os.makedirs(os.path.join(d, 'sr44100_hl1024_nf2048'), exist_ok=True)
                open(os.path.join(d, name + '.wav'), 'wb').close()
                np.save(os.path.join(d, 'sr44100_hl1024_nf2048', name + '.npy'), s.transpose(2, 0, 1))
                pair.append(os.path.join(d, name + '.wav'))
            pairs.setdefault(sub, []).append(pair)
    return pairs


def _cli_loss(*args):
    r = subprocess.run([sys.executable, os.path.join(PKG, 'validate.py'), '-g', '0'] + list(args),
                       capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    m = re.fullmatch(r'validation loss = (\d+\.\d{6})', lines[-1])
    assert m, r.stdout
    return m.group(1), [l for l in lines if re.match(r'\d+ \S+\.wav \S+\.wav \d+\.\d{6}$', l)]


def test_cli_end_to_end(model, specs, tmp_path):
    import validate
    from lib import dataset, synth
    dev = _dev()
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)

    def expect(filelist, batchsize=4):
        return '{:.6f}'.format(validate.validation_loss(model, dev, filelist, 44100, 1024, 2048, 256, batchsize))

    # random: the reference's shuffle of 4 pairs with seed 3, half of them validation pairs
    flat = _dataset(str(tmp_path / 'flat'), specs, {'': [0, 1, 2, 3]})['']
    random.seed(3)
    _, val = dataset.train_val_split(str(tmp_path / 'flat'), 'random', 0.5, [])
    assert len(val) == 2
    loss, pairs = _cli_loss('-d', str(tmp_path / 'flat'), '-P', ckpt, '-s', '3', '-v', '0.5')
    assert loss == expect(val) and len(pairs) == 2
    assert pairs[0].startswith('1 %s %s ' % (os.path.basename(val[0][0]), os.path.basename(val[0][1])))
    loss_b1, _ = _cli_loss('-d', str(tmp_path / 'flat'), '-P', ckpt, '-s', '3', '-v', '0.5', '-b', '1')
    assert loss_b1 == expect(val, 1)

    # --val_filelist: the given pairs, in the given order
    vlist = str(tmp_path / 'val.json')
    with open(vlist, 'w') as f:
        json.dump([flat[3], flat[1]], f)
    loss, pairs = _cli_loss('-d', str(tmp_path / 'flat'), '-P', ckpt, '-V', vlist)
    assert loss == expect([flat[3], flat[1]]) and len(pairs) == 2

    # subdirs: validation/ only
    sub = _dataset(str(tmp_path / 'split'), specs, {'training': [0], 'validation': [1, 2, 3]})
    loss, pairs = _cli_loss('-d', str(tmp_path / 'split'), '-P', ckpt, '-S', 'subdirs')
    assert loss == expect(sub['validation']) and len(pairs) == 3
    assert not any(d.startswith('cs256_sr') for d in os.listdir(PKG))   # no patch cache in the working directory
