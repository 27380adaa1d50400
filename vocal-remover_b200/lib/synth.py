"""Synthetic inputs and synthetic checkpoints for parity tests and benchmarks.

No pretrained ``baseline.pth`` ships with the reference (models/.gitkeep only;
inference.py:104-105 expects a GitHub-release download) and there is no network, so
every parity / timing run uses the seeded recipes below.  Both the unmodified reference
(oracle side) and the H100 path load the same ``state_dict``.

* ``sine_mix``            - SURVEY.md section 8(d) synthetic 44.1 kHz stereo sine mix + 1 % noise.
* ``state_dict_spec``     - (key, shape, kind) for every entry of ``CascadedNet.state_dict()``
                            (689 keys for the default net; lib/nets.py:44-80, SURVEY App. C).
* ``make_state_dict``     - seeded, name-keyed values: He-uniform conv / linear weights so every
                            layer carries signal, torch-style LSTM init, non-trivial BatchNorm
                            statistics; ``out.weight`` is scaled so the mask logits have
                            std ~= 3 (masks span (0,1); otherwise the 1e-3 gate is vacuous).
"""
import zlib

import numpy as np


def sine_mix(seconds, sr=44100, seed=0):
    """float32 (2, L) stereo sine mix + low-level noise (SURVEY.md 8(d))."""
    L = int(round(seconds * sr))
    rng = np.random.default_rng(seed)
    out = np.empty((2, L), dtype=np.float32)
    blk = 1 << 22
    for s in range(0, L, blk):
        e = min(L, s + blk)
        t = np.arange(s, e, dtype=np.float64) / sr
        n = rng.standard_normal((2, e - s))
        out[0, s:e] = (0.30 * np.sin(2 * np.pi * 440 * t) + 0.20 * np.sin(2 * np.pi * 1000 * t)
                       + 0.10 * np.sin(2 * np.pi * 3000 * t) + 0.01 * n[0])
        out[1, s:e] = (0.30 * np.sin(2 * np.pi * 440 * t + 0.3) + 0.20 * np.sin(2 * np.pi * 1500 * t)
                       + 0.10 * np.sin(2 * np.pi * 5000 * t) + 0.01 * n[1])
    return out


def _cba(prefix, cin, cout, k):
    """Conv2DBNActiv at ``prefix`` (lib/layers.py:8-26): conv.0 = Conv2d(bias=False), conv.1 = BatchNorm2d."""
    yield prefix + '.conv.0.weight', (cout, cin, k, k), 'conv'
    yield from _bn(prefix + '.conv.1', cout)


def _bn(prefix, c):
    yield prefix + '.weight', (c,), 'bn_weight'
    yield prefix + '.bias', (c,), 'bn_bias'
    yield prefix + '.running_mean', (c,), 'bn_mean'
    yield prefix + '.running_var', (c,), 'bn_var'
    yield prefix + '.num_batches_tracked', (), 'bn_count'


def _basenet(prefix, nin, n, nin_lstm, nout_lstm):
    """BaseNet children (lib/nets.py:10-24)."""
    yield from _cba(prefix + '.enc1', nin, n, 3)
    cprev = n
    for i, mult in zip((2, 3, 4, 5), (2, 4, 6, 8)):
        yield from _cba(f'{prefix}.enc{i}.conv1', cprev, n * mult, 3)
        yield from _cba(f'{prefix}.enc{i}.conv2', n * mult, n * mult, 3)
        cprev = n * mult
    c8 = n * 8
    yield from _cba(prefix + '.aspp.conv1.1', c8, c8, 1)
    yield from _cba(prefix + '.aspp.conv2', c8, c8, 1)
    for i in (3, 4, 5):
        yield from _cba(f'{prefix}.aspp.conv{i}', c8, c8, 3)
    yield from _cba(prefix + '.aspp.bottleneck', c8 * 5, c8, 1)
    yield from _cba(prefix + '.dec4.conv1', n * 14, n * 6, 3)
    yield from _cba(prefix + '.dec3.conv1', n * 10, n * 4, 3)
    yield from _cba(prefix + '.dec2.conv1', n * 6, n * 2, 3)
    p = prefix + '.lstm_dec2'
    yield from _cba(p + '.conv', n * 2, 1, 1)
    hid = nout_lstm // 2
    for sfx in ('', '_reverse'):
        yield f'{p}.lstm.weight_ih_l0{sfx}', (4 * hid, nin_lstm), 'lstm'
        yield f'{p}.lstm.weight_hh_l0{sfx}', (4 * hid, hid), 'lstm'
        yield f'{p}.lstm.bias_ih_l0{sfx}', (4 * hid,), 'lstm'
        yield f'{p}.lstm.bias_hh_l0{sfx}', (4 * hid,), 'lstm'
    yield p + '.dense.0.weight', (nin_lstm, nout_lstm), 'linear'
    yield p + '.dense.0.bias', (nin_lstm,), 'linear_bias'
    yield from _bn(p + '.dense.1', nin_lstm)
    yield from _cba(prefix + '.dec1.conv1', n * 3 + 1, n, 3)


def state_dict_spec(n_fft=2048, nout=32, nout_lstm=128):
    """[(key, shape, kind)] of CascadedNet(n_fft, hop, nout, nout_lstm).state_dict() (lib/nets.py:46-80)."""
    max_bin = n_fft // 2
    nin_lstm = max_bin // 2
    nin = 2
    spec = []
    spec += _basenet('stg1_low_band_net.0', nin, nout // 2, nin_lstm // 2, nout_lstm)
    spec += _cba('stg1_low_band_net.1', nout // 2, nout // 4, 1)
    spec += _basenet('stg1_high_band_net', nin, nout // 4, nin_lstm // 2, nout_lstm // 2)
    spec += _basenet('stg2_low_band_net.0', nout // 4 + nin, nout, nin_lstm // 2, nout_lstm)
    spec += _cba('stg2_low_band_net.1', nout, nout // 2, 1)
    spec += _basenet('stg2_high_band_net', nout // 4 + nin, nout // 2, nin_lstm // 2, nout_lstm // 2)
    spec += _basenet('stg3_full_band_net', 3 * nout // 4 + nin, nout, nin_lstm, nout_lstm)
    spec.append(('out.weight', (nin, nout, 1, 1), 'conv'))
    spec.append(('aux_out.weight', (nin, 3 * nout // 4, 1, 1), 'conv'))
    return spec


# ``out.weight`` multiplier that brings std(logit) of the first 256-frame window of the 10 s
# ``sine_mix`` to ~3 for seed 0 / default net.  Measured once with the unmodified reference
# (oracle/make_golden.py prints it); a constant so the product never needs an oracle pass.
OUT_LOGIT_GAIN = {(2048, 32, 128, 0): 3.3}


def make_state_dict(n_fft=2048, nout=32, nout_lstm=128, seed=0, out_gain=None):
    """Seeded synthetic checkpoint as {key: numpy array}; dtypes follow torch (float32 / int64)."""
    sd = {}
    for key, shape, kind in state_dict_spec(n_fft, nout, nout_lstm):
        rng = np.random.default_rng([seed, zlib.crc32(key.encode())])
        if kind == 'conv':
            fan_in = shape[1] * shape[2] * shape[3]
            b = np.sqrt(6.0 / fan_in)
            v = rng.uniform(-b, b, size=shape)
        elif kind == 'linear':
            b = np.sqrt(6.0 / shape[1])
            v = rng.uniform(-b, b, size=shape)
        elif kind == 'linear_bias':
            v = rng.uniform(-0.1, 0.1, size=shape)
        elif kind == 'lstm':
            hid = shape[0] // 4
            b = 1.0 / np.sqrt(hid)
            v = rng.uniform(-b, b, size=shape)
        elif kind == 'bn_weight':
            v = rng.uniform(0.5, 1.5, size=shape)
        elif kind == 'bn_bias':
            v = rng.uniform(-0.1, 0.1, size=shape)
        elif kind == 'bn_mean':
            v = rng.uniform(-0.1, 0.1, size=shape)
        elif kind == 'bn_var':
            v = rng.uniform(0.5, 1.5, size=shape)
        elif kind == 'bn_count':
            sd[key] = np.asarray(1, dtype=np.int64)
            continue
        else:
            raise ValueError(kind)
        sd[key] = v.astype(np.float32)
    if out_gain is None:
        out_gain = OUT_LOGIT_GAIN.get((n_fft, nout, nout_lstm, seed), 1.0)
    sd['out.weight'] = (sd['out.weight'] * np.float32(out_gain)).astype(np.float32)
    return sd


def to_torch_state_dict(sd):
    import torch
    return {k: torch.from_numpy(np.array(v, copy=True)) for k, v in sd.items()}
