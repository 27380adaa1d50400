"""validate.py without a GPU: the numpy validation-loss oracle against the reference's own validate_epoch
(tests/golden/ref_validation, oracle/validation_oracle.py), the reference's train / validation split, the patch count,
the rank-0 combination of per-window sums over gloo, and the CLI's error order."""
import math
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from conftest import PKG, checksum, load_golden


@pytest.fixture(scope='module')
def golden_validation():
    return load_golden('ref_validation')


def test_validation_oracle_equals_reference(golden_validation):
    from lib import synth
    from oracle import validation_oracle
    g = golden_validation
    sd = synth.to_torch_state_dict(synth.make_state_dict())
    losses = []
    for (name, X, y), (_, a, b) in zip(validation_oracle.spectrograms(), validation_oracle.validation_cases()):
        # the seeded waves regenerate bit for bit, their spectrograms to rounding
        assert np.array_equal(np.stack([checksum(a), checksum(b)]), g[name + '_wave_sum']), name
        np.testing.assert_allclose(np.stack([checksum(X), checksum(y)]), g[name + '_spec_sum'], rtol=1e-6, atol=1e-6)
        losses.append(validation_oracle.patch_losses(sd, X, y))
    assert [len(l) for l in losses] == [math.ceil(T / 128) for T in g['T']]
    losses = np.concatenate(losses)
    np.testing.assert_allclose(losses, g['patch_losses'], rtol=1e-5, atol=0)
    np.testing.assert_allclose(losses.mean(), g['total_b4'], rtol=1e-5, atol=0)


def _listing(root, names):
    for sub in ('mixtures', 'instruments'):
        os.makedirs(os.path.join(root, sub))
        for base in names:
            open(os.path.join(root, sub, base + '.wav'), 'wb').close()
        open(os.path.join(root, sub, 'notes.txt'), 'w').close()


def test_train_val_split_matches_reference(golden_validation, tmp_path):
    from lib import dataset
    from oracle import validation_oracle
    g = golden_validation
    root = str(tmp_path / 'split')
    _listing(root, validation_oracle.split_names())
    random.seed(validation_oracle.SPLIT_SEED)
    train, val = dataset.train_val_split(root, 'random', validation_oracle.SPLIT_RATE, [])
    base = lambda lst: [[os.path.basename(a), os.path.basename(b)] for a, b in lst]   # noqa: E731
    assert base(train) == g['split_train'].tolist() and base(val) == g['split_val'].tolist()
    assert len(val) == 2 and all(os.path.dirname(a) == os.path.join(root, 'mixtures') for a, _ in val)
    # a given validation list is used as it stands; the training set is every other pair
    given = [list(p) for p in val]
    train2, val2 = dataset.train_val_split(root, 'random', 0.2, given)
    assert val2 is given and sorted(train2) == sorted(train)


def test_train_val_split_subdirs(tmp_path):
    from lib import dataset
    _listing(str(tmp_path / 'training'), ['a', 'b', 'c'])
    _listing(str(tmp_path / 'validation'), ['d', 'e'])
    train, val = dataset.train_val_split(str(tmp_path), 'subdirs', 0.2, [])
    assert [os.path.basename(a) for a, _ in train] == ['a.wav', 'b.wav', 'c.wav']
    assert [os.path.basename(b) for _, b in val] == ['d.wav', 'e.wav']
    with pytest.raises(ValueError, match='`val_filelist` option is not available with `subdirs` mode'):
        dataset.train_val_split(str(tmp_path), 'subdirs', 0.2, [['x.wav', 'y.wav']])


def test_validation_patch_count():
    from lib import dataset, distributed
    for T in (1, 2, 127, 128, 129, 255, 256, 257, 383, 384, 385, 10000):
        n = dataset.validation_patch_count(T, 256, 64)
        assert n == math.ceil(T / 128), T
        # Separator cuts one window more exactly when T is a multiple of roi (lib/dataset.py:236 vs inference.py:44)
        assert distributed.window_count(T, 256, 64)[0] == n + (T % 128 == 0), T
    assert dataset.validation_patch_count(300, 192, 64) == 5   # roi 64


_WORKER = r'''
import os, sys
import numpy as np
import torch.distributed as dist
sys.path.insert(0, os.getcwd())
import validate
from lib import dataset, nets
world, rank, init, out = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4]
rng = np.random.default_rng(5)
sums = [rng.uniform(0, 300, size=n) for n in (3, 1, 4, 2, 2)]   # per-file window sums, global file order
if world > 1:
    dist.init_process_group('gloo', init_method=init, world_size=world, rank=rank)
got = validate.gather_window_sums(dataset.shard_files(sums, world, rank), world, rank)
if rank == 0:
    assert len(got) == len(sums) and all(np.array_equal(a, b) for a, b in zip(got, sums))
    v = validate.Validator(nets.CascadedNet(2048, 1024), None, 256, 4)
    np.save(out, np.float64(validate.combine(v, got)))
else:
    assert got is None
if world > 1:
    dist.destroy_process_group()
'''


def test_rank0_combination_is_independent_of_world_size(tmp_path):
    env = dict(os.environ, GLOO_SOCKET_IFNAME='lo', CUDA_VISIBLE_DEVICES='')
    results = {}
    for world in (1, 2):
        init = 'file://' + str(tmp_path / ('init%d' % world))
        out = str(tmp_path / ('loss%d.npy' % world))
        procs = [subprocess.Popen([sys.executable, '-c', _WORKER, str(world), str(rank), init, out], cwd=PKG, env=env,
                                  stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for rank in range(world)]
        for p in procs:
            _, err = p.communicate(timeout=300)
            assert p.returncode == 0, err
        results[world] = np.load(out)
    assert results[1].tobytes() == results[2].tobytes()
    rng = np.random.default_rng(5)
    sums = np.concatenate([rng.uniform(0, 300, size=n) for n in (3, 1, 4, 2, 2)])
    np.testing.assert_allclose(results[1], (sums / (2 * 1025 * 128)).mean(), rtol=1e-15)


def _cli(*args, cwd=None):
    return subprocess.run([sys.executable, os.path.join(PKG, 'validate.py')] + list(args), capture_output=True,
                          text=True, cwd=cwd or PKG)


def test_cli_errors_come_before_the_model_loads(tmp_path):
    data = str(tmp_path / 'data')
    _listing(data, ['a', 'b', 'c', 'd', 'e'])
    garbage = str(tmp_path / 'not_a_checkpoint.pth')
    with open(garbage, 'w') as f:
        f.write('not a checkpoint')
    vlist = str(tmp_path / 'val.json')
    with open(vlist, 'w') as f:
        f.write('[["x.wav", "y.wav"]]')

    r = _cli('-d', data)
    assert r.returncode == 2 and '--pretrained_model/-P' in r.stderr
    r = _cli('-d', data, '-P', str(tmp_path / 'missing.pth'))
    assert r.returncode == 2 and 'no such file' in r.stderr and 'missing.pth' in r.stderr
    r = _cli('-d', data, '-P', garbage, '-S', 'subdirs', '-V', vlist)
    assert r.returncode == 2 and '`val_filelist` option is not available with `subdirs` mode' in r.stderr
    r = _cli('-d', data, '-P', garbage, '-S', 'folds')
    assert r.returncode == 2 and 'invalid choice' in r.stderr
    r = _cli('-d', str(tmp_path / 'nowhere'), '-P', garbage)
    assert r.returncode == 2 and 'nowhere' in r.stderr
    r = _cli('-d', data, '-P', garbage, '-c', '128')
    assert r.returncode == 2 and '--val_cropsize' in r.stderr
    # training-only flags of train.py are not taken
    r = _cli('-d', data, '-P', garbage, '-E', '3')
    assert r.returncode == 2 and 'unrecognized arguments' in r.stderr


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
