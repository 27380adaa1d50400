"""H100-native mirror of the reference's lib/spec_utils.py for the inference path.

wave_to_spectrogram / spectrogram_to_wave keep the reference signatures and numpy in / numpy out
contract (lib/spec_utils.py:26-31, 157-165) but run the framed FFT / inverse FFT + overlap-add on the
GPU through libvr_b200.so (csrc/fft.cu) instead of librosa on the host.  spectrogram_to_image (--output_image) builds
its uint8 image on the GPU as well (csrc/elementwise.cu).

Run as a script, it is the reference's pair check (lib/spec_utils.py:168-198): one (mixture, instruments) pair is
loaded at 44.1 kHz and aligned, and test_X / test_y / test_v .jpg and .wav, of the mixture, the instruments and
their difference v = X - y, are written to the working directory::

    python lib/spec_utils.py <mix> <inst>        (or python -m lib.spec_utils ...)
"""
import os
import sys

if __name__ == '__main__' and not __package__:
    # run as a file: import the package this file belongs to instead of its modules as top-level ones
    _LIB_DIR = os.path.dirname(os.path.abspath(__file__))
    if sys.path and os.path.abspath(sys.path[0] or os.curdir) == _LIB_DIR:
        del sys.path[0]
    sys.path.insert(0, os.path.dirname(_LIB_DIR))
    __package__ = 'lib'

import numpy as np
import torch

from . import _native

_DEVICE_INDEX = 0
_ctx_cache = {}


def set_device(index):
    """GPU used by the module-level spectral functions (default cuda:0)."""
    global _DEVICE_INDEX
    _DEVICE_INDEX = int(index)


def _spectral_ctx(n_fft, hop_length):
    key = (_DEVICE_INDEX, int(n_fft), int(hop_length))
    ctx = _ctx_cache.get(key)
    if ctx is None:
        # a context without weights: only the FFT tables are allocated until weights are finalized
        ctx = _native.Context(_DEVICE_INDEX, n_fft, hop_length, 32, 128, 256, 1)
        _ctx_cache[key] = ctx
    return ctx


def crop_center(h1, h2):
    """lib/spec_utils.py:8-23: centre-crop h1 on the time axis (dim 3) to h2's width."""
    w1, w2 = h1.size()[3], h2.size()[3]
    if w1 == w2:
        return h1
    if w1 < w2:
        raise ValueError('h1_shape[3] must be greater than h2_shape[3]')
    start = (w1 - w2) // 2
    return h1[:, :, :, start:start + w2]


def wave_to_spectrogram(wave, hop_length, n_fft):
    """float32 (2, L) -> complex64 (2, n_fft//2+1, 1 + L//hop_length)   (lib/spec_utils.py:26-31)."""
    wave = np.ascontiguousarray(np.asarray(wave, dtype=np.float32))
    if wave.ndim != 2 or wave.shape[0] != 2:
        raise ValueError('wave must have shape (2, L)')
    ctx = _spectral_ctx(n_fft, hop_length)
    dev = torch.device('cuda', ctx.device_index)
    L = wave.shape[1]
    T = 1 + L // hop_length
    with torch.cuda.device(dev):
        d_wave = torch.from_numpy(wave).to(dev)
        d_spec = torch.empty((2, n_fft // 2 + 1, T), dtype=torch.complex64, device=dev)
        ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(d_wave), L, _native.ptr(d_spec), T, None,
                                  _native.stream_ptr()), 'vr_stft')
        return d_spec.cpu().numpy()


def spectrogram_to_wave(spec, hop_length=1024):
    """complex64 (2, bins, T) or (bins, T) -> float32 (2, hop*(T-1)) or (hop*(T-1),)   (lib/spec_utils.py:157-165)."""
    spec = np.asarray(spec)
    mono = spec.ndim == 2
    if mono:
        spec = np.asarray([spec, spec])
    elif spec.ndim != 3:
        raise ValueError('spec must be 2-D or 3-D')
    spec = np.ascontiguousarray(spec.astype(np.complex64, copy=False))
    n_fft = 2 * (spec.shape[1] - 1)
    T = spec.shape[2]
    ctx = _spectral_ctx(n_fft, hop_length)
    dev = torch.device('cuda', ctx.device_index)
    with torch.cuda.device(dev):
        d_spec = torch.from_numpy(spec).to(dev)
        d_wave = torch.empty((2, hop_length * (T - 1)), dtype=torch.float32, device=dev)
        ctx.check(ctx.lib.vr_istft(ctx.handle, _native.ptr(d_spec), T, _native.ptr(d_wave),
                                   _native.stream_ptr()), 'vr_istft')
        out = d_wave.cpu().numpy()
    return out[0] if mono else out


def spectrogram_to_image(spec, mode='magnitude'):
    """complex (2, bins, T) -> uint8 (bins, T, 3) image {max(L, R), L, R} of the log power   (lib/spec_utils.py:34-57).

    Built on the GPU (vr_spec_image).  A numpy array gives a numpy image, a CUDA complex64 tensor a CUDA uint8 tensor.
    A constant spectrogram (e.g. silence) gives an all-zero image where the reference's uint8 cast sees NaN.
    """
    if mode != 'magnitude':
        raise NotImplementedError("spectrogram_to_image: only mode='magnitude' (the --output_image path) is supported")
    on_device = torch.is_tensor(spec)
    if not on_device:
        spec = np.asarray(spec)
    if not (spec.is_complex() if on_device else np.iscomplexobj(spec)):
        raise NotImplementedError('spectrogram_to_image: only complex spectrograms (the --output_image path)')
    if spec.ndim != 3 or spec.shape[0] != 2:
        raise NotImplementedError('spectrogram_to_image: only (2, bins, T) stereo spectrograms (the --output_image path)')
    bins, T = spec.shape[1], spec.shape[2]
    ctx = _spectral_ctx(2 * (bins - 1), bins - 1)
    dev = torch.device('cuda', ctx.device_index)
    with torch.cuda.device(dev):
        d_spec = _to_device(spec, dev, 'spectrogram_to_image')
        img = torch.empty((bins, T, 3), dtype=torch.uint8, device=dev)
        ctx.check(ctx.lib.vr_spec_image(ctx.handle, _native.ptr(d_spec), None, T, _native.ptr(img), None,
                                        _native.stream_ptr()), 'vr_spec_image')
        return img if on_device else img.cpu().numpy()


def _to_device(spec, dev, what):
    """A contiguous complex64 copy (or the tensor itself) of ``spec`` on ``dev``."""
    if torch.is_tensor(spec):
        if spec.device != dev:
            raise ValueError('%s: spec is on %s, the spectral functions use %s' % (what, spec.device, dev))
        return spec.to(torch.complex64).contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(spec, dtype=np.complex64))).to(dev)


def spectrogram_difference(a, b):
    """complex (2, bins, T) a - b, the pair check's v_spec = X_spec - y_spec (lib/spec_utils.py:186), on the GPU
    (vr_spec_sub): complex64 with numpy's bits.  Numpy arrays give a numpy array, CUDA tensors a CUDA tensor."""
    on_device = torch.is_tensor(a)
    if torch.is_tensor(b) != on_device:
        raise TypeError('spectrogram_difference: a and b must both be numpy arrays or both CUDA tensors')
    if not on_device:
        a, b = np.asarray(a), np.asarray(b)
    if a.ndim != 3 or a.shape[0] != 2 or tuple(a.shape) != tuple(b.shape):
        raise ValueError('spectrogram_difference: a and b must both have shape (2, bins, T), got %s and %s'
                         % (tuple(a.shape), tuple(b.shape)))
    bins, T = a.shape[1], a.shape[2]
    ctx = _spectral_ctx(2 * (bins - 1), bins - 1)
    dev = torch.device('cuda', ctx.device_index)
    with torch.cuda.device(dev):
        d_a, d_b = (_to_device(s, dev, 'spectrogram_difference') for s in (a, b))
        out = torch.empty((2, bins, T), dtype=torch.complex64, device=dev)
        ctx.check(ctx.lib.vr_spec_sub(ctx.handle, _native.ptr(d_a), _native.ptr(d_b), T, _native.ptr(out),
                                      _native.stream_ptr()), 'vr_spec_sub')
        return out if on_device else out.cpu().numpy()


def wiener(X_spec, y_spec, v_spec, iterations=1):
    """The two stems refined by a multichannel Wiener filter (expectation-maximisation, norbert 0.2's
    ``wiener(v, x, iterations)`` for 2 channels and 2 sources; DESIGN.md §11), on the GPU (vr_wiener).

    X_spec is the mixture, y_spec / v_spec the initial estimates (the masked spectrograms), each complex (2, bins, T).
    Numpy arrays give numpy arrays, CUDA tensors new CUDA tensors; the inputs are not modified.  Returns
    (y_spec, v_spec) as complex64; ``iterations = 0`` returns them unchanged.
    """
    if iterations < 0:
        raise ValueError('wiener: iterations must be >= 0, got %d' % iterations)
    on_device = torch.is_tensor(X_spec)
    if torch.is_tensor(y_spec) != on_device or torch.is_tensor(v_spec) != on_device:
        raise TypeError('wiener: X_spec, y_spec and v_spec must all be numpy arrays or all CUDA tensors')
    if not on_device:
        X_spec, y_spec, v_spec = np.asarray(X_spec), np.asarray(y_spec), np.asarray(v_spec)
    if X_spec.ndim != 3 or X_spec.shape[0] != 2 or X_spec.shape[2] < 1 or \
            not tuple(X_spec.shape) == tuple(y_spec.shape) == tuple(v_spec.shape):
        raise ValueError('wiener: X_spec, y_spec and v_spec must all have shape (2, bins, T >= 1), got %s, %s and %s'
                         % (tuple(X_spec.shape), tuple(y_spec.shape), tuple(v_spec.shape)))
    bins, T = X_spec.shape[1], X_spec.shape[2]
    ctx = _spectral_ctx(2 * (bins - 1), bins - 1)
    dev = torch.device('cuda', ctx.device_index)
    with torch.cuda.device(dev):
        d_x = _to_device(X_spec, dev, 'wiener')
        d_y, d_v = (_to_device(s, dev, 'wiener').clone() for s in (y_spec, v_spec))
        ctx.check(ctx.lib.vr_wiener(ctx.handle, _native.ptr(d_x), _native.ptr(d_y), _native.ptr(d_v), T,
                                    int(iterations), _native.stream_ptr()), 'vr_wiener')
        return (d_y, d_v) if on_device else (d_y.cpu().numpy(), d_v.cpu().numpy())


# evaluate.py --oracle (DESIGN.md §12): the masks vr_oracle_mask computes, by kind number, then the oracle MWF
MASK_ORACLES = ('iam', 'ibm', 'irm1', 'irm2')
ORACLES = MASK_ORACLES + ('mwf',)


def current_device():
    """The CUDA device of the module-level spectral functions (set_device)."""
    return torch.device('cuda', _DEVICE_INDEX)


def oracle_mask(X_spec, y_spec, kind):
    """The instruments mask of an ideal separation (DESIGN.md §12), on the GPU (vr_oracle_mask): float32 (2, bins, T)
    in [0, 1] from the mixture X_spec and the true instruments y_spec, each complex (2, bins, T); the vocals' mask is
    ``1 - mask``.  ``kind`` is one of MASK_ORACLES: 'iam' clip(|Y| / |X|, 0, 1), 'ibm' the dominant source, 'irm1'
    |Y| / (|Y| + |V|), 'irm2' |Y|^2 / (|Y|^2 + |V|^2), with V = X - Y.  Numpy arrays give a numpy array, CUDA tensors a
    CUDA tensor; the inputs are not modified."""
    if kind not in MASK_ORACLES:
        raise ValueError('oracle_mask: kind must be one of %s, got %r' % (', '.join(MASK_ORACLES), kind))
    on_device = torch.is_tensor(X_spec)
    if torch.is_tensor(y_spec) != on_device:
        raise TypeError('oracle_mask: X_spec and y_spec must both be numpy arrays or both CUDA tensors')
    if not on_device:
        X_spec, y_spec = np.asarray(X_spec), np.asarray(y_spec)
    if X_spec.ndim != 3 or X_spec.shape[0] != 2 or X_spec.shape[2] < 1 or tuple(X_spec.shape) != tuple(y_spec.shape):
        raise ValueError('oracle_mask: X_spec and y_spec must both have shape (2, bins, T >= 1), got %s and %s'
                         % (tuple(X_spec.shape), tuple(y_spec.shape)))
    bins, T = X_spec.shape[1], X_spec.shape[2]
    ctx = _spectral_ctx(2 * (bins - 1), bins - 1)
    dev = torch.device('cuda', ctx.device_index)
    with torch.cuda.device(dev):
        d_x, d_y = (_to_device(s, dev, 'oracle_mask') for s in (X_spec, y_spec))
        mask = torch.empty((2, bins, T), dtype=torch.float32, device=dev)
        ctx.check(ctx.lib.vr_oracle_mask(ctx.handle, _native.ptr(d_x), _native.ptr(d_y), T, MASK_ORACLES.index(kind),
                                         _native.ptr(mask), _native.stream_ptr()), 'vr_oracle_mask')
        return mask if on_device else mask.cpu().numpy()


def _check_oracle(kind, wiener_iterations):
    if kind not in ORACLES:
        raise ValueError('oracle: kind must be one of %s, got %r' % (', '.join(ORACLES), kind))
    if wiener_iterations < 0:
        raise ValueError('oracle: wiener_iterations must be >= 0, got %d' % wiener_iterations)
    if kind == 'mwf' and wiener_iterations > 0:
        raise ValueError('oracle: mwf is one Wiener iteration from the true stems; wiener_iterations must be 0')


def oracle_spectrograms(X_spec, y_spec, kind, wiener_iterations=0):
    """The oracle estimates (y_spec, v_spec) of the mixture X_spec given the true instruments y_spec (DESIGN.md §12):
    a mask oracle applies ``oracle_mask`` as the Separator applies the net's mask (vr_apply_mask), refined by
    ``wiener_iterations`` of the Wiener filter; 'mwf' is one Wiener iteration (vr_wiener) started from the true stems
    y_spec and X_spec - y_spec.  Numpy arrays give numpy arrays, CUDA tensors CUDA tensors; the inputs are not
    modified."""
    _check_oracle(kind, wiener_iterations)
    on_device = torch.is_tensor(X_spec)
    if torch.is_tensor(y_spec) != on_device:
        raise TypeError('oracle_spectrograms: X_spec and y_spec must both be numpy arrays or both CUDA tensors')
    if not on_device:
        X_spec, y_spec = np.asarray(X_spec), np.asarray(y_spec)
    if X_spec.ndim != 3 or X_spec.shape[0] != 2 or X_spec.shape[2] < 1 or tuple(X_spec.shape) != tuple(y_spec.shape):
        raise ValueError('oracle_spectrograms: X_spec and y_spec must both have shape (2, bins, T >= 1), got %s and %s'
                         % (tuple(X_spec.shape), tuple(y_spec.shape)))
    bins = X_spec.shape[1]
    ctx = _spectral_ctx(2 * (bins - 1), bins - 1)
    dev = torch.device('cuda', ctx.device_index)
    with torch.cuda.device(dev):
        d_x, d_y = (_to_device(s, dev, 'oracle_spectrograms') for s in (X_spec, y_spec))
        y, v = _oracle_specs(ctx, d_x, d_y, kind, wiener_iterations)
        return (y, v) if on_device else (y.cpu().numpy(), v.cpu().numpy())


def _oracle_specs(ctx, d_x, d_y, kind, wiener_iterations):
    """oracle_spectrograms on device complex64 tensors, into new tensors."""
    T = d_x.shape[2]
    y, v = torch.empty_like(d_x), torch.empty_like(d_x)
    if kind == 'mwf':
        y.copy_(d_y)
        ctx.check(ctx.lib.vr_spec_sub(ctx.handle, _native.ptr(d_x), _native.ptr(d_y), T, _native.ptr(v),
                                      _native.stream_ptr()), 'vr_spec_sub')
        iterations = 1
    else:
        mask = torch.empty(d_x.shape, dtype=torch.float32, device=d_x.device)
        ctx.check(ctx.lib.vr_oracle_mask(ctx.handle, _native.ptr(d_x), _native.ptr(d_y), T, MASK_ORACLES.index(kind),
                                         _native.ptr(mask), _native.stream_ptr()), 'vr_oracle_mask')
        ctx.check(ctx.lib.vr_apply_mask(ctx.handle, _native.ptr(d_x), _native.ptr(mask), T, _native.ptr(y),
                                        _native.ptr(v), _native.stream_ptr()), 'vr_apply_mask')
        iterations = wiener_iterations
    if iterations > 0:
        ctx.check(ctx.lib.vr_wiener(ctx.handle, _native.ptr(d_x), _native.ptr(y), _native.ptr(v), T, iterations,
                                    _native.stream_ptr()), 'vr_wiener')
    return y, v


def oracle_separate_wave(X, y, kind, n_fft=2048, hop_length=1024, wiener_iterations=0):
    """The oracle stems (instruments, vocals), float32 (2, hop * (L // hop)) each, of the mixture wave X given the
    true instruments wave y, both float32 (2, L), at the STFT (n_fft, hop_length) - what ``Separator.separate_wave``
    returns with the net's mask replaced by the oracle's (DESIGN.md §12).  A mask oracle without the Wiener filter runs
    the Separator's masked inverse STFT (vr_apply_mask_istft); otherwise both estimates of ``oracle_spectrograms`` are
    inverted (vr_istft).  CUDA tensors give CUDA tensors, numpy arrays numpy arrays."""
    _check_oracle(kind, wiener_iterations)
    on_device = torch.is_tensor(X)
    if torch.is_tensor(y) != on_device:
        raise TypeError('oracle_separate_wave: X and y must both be numpy arrays or both CUDA tensors')
    if tuple(X.shape) != tuple(y.shape) or len(X.shape) != 2 or X.shape[0] != 2 or X.shape[1] < 1:
        raise ValueError('oracle_separate_wave: X and y must both have shape (2, L >= 1), got %s and %s'
                         % (tuple(X.shape), tuple(y.shape)))
    ctx = _spectral_ctx(n_fft, hop_length)
    dev = torch.device('cuda', ctx.device_index)
    with torch.cuda.device(dev):
        waves = []
        for w in (X, y):
            if on_device:
                if w.device != dev:
                    raise ValueError('oracle_separate_wave: wave is on %s, the spectral functions use %s'
                                     % (w.device, dev))
                waves.append(w.contiguous().float())
            else:
                waves.append(torch.from_numpy(np.ascontiguousarray(np.asarray(w, dtype=np.float32))).to(dev))
        L = waves[0].shape[1]
        T = 1 + L // hop_length
        d_x, d_y = (torch.empty((2, n_fft // 2 + 1, T), dtype=torch.complex64, device=dev) for _ in range(2))
        for w, spec in zip(waves, (d_x, d_y)):
            ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(w), L, _native.ptr(spec), T, None,
                                      _native.stream_ptr()), 'vr_stft')
        inst = torch.empty((2, hop_length * (T - 1)), dtype=torch.float32, device=dev)
        voc = torch.empty_like(inst)
        if kind in MASK_ORACLES and wiener_iterations == 0:
            mask = torch.empty((2, n_fft // 2 + 1, T), dtype=torch.float32, device=dev)
            ctx.check(ctx.lib.vr_oracle_mask(ctx.handle, _native.ptr(d_x), _native.ptr(d_y), T,
                                             MASK_ORACLES.index(kind), _native.ptr(mask), _native.stream_ptr()),
                      'vr_oracle_mask')
            ctx.check(ctx.lib.vr_apply_mask_istft(ctx.handle, _native.ptr(d_x), _native.ptr(mask), T,
                                                  _native.ptr(inst), _native.ptr(voc), _native.stream_ptr()),
                      'vr_apply_mask_istft')
        else:
            for spec, wave_out in zip(_oracle_specs(ctx, d_x, d_y, kind, wiener_iterations), (inst, voc)):
                ctx.check(ctx.lib.vr_istft(ctx.handle, _native.ptr(spec), T, _native.ptr(wave_out),
                                           _native.stream_ptr()), 'vr_istft')
        return (inst, voc) if on_device else (inst.cpu().numpy(), voc.cpu().numpy())


def artifact_weights(frame_min, thres=0.05, min_range=64, fade_size=32):
    """Per-frame fade weight of ``merge_artifacts`` from the per-frame minimum of the mask over (channel, bin).

    Frames whose minimum exceeds ``thres`` for runs longer than ``min_range`` are treated as vocal-free; the weight
    ramps 0 -> 1 over ``fade_size`` frames into such a run and 1 -> 0 out of it (reference lib/spec_utils.py:60-93,
    including its handling of runs that touch either end of the track or follow each other closely).
    """
    if min_range < fade_size * 2:
        raise ValueError('min_range must be >= fade_size * 2')
    frame_min = np.asarray(frame_min)
    n_frames = frame_min.shape[0]
    weight = np.zeros(n_frames, dtype=np.float32)
    idx = np.flatnonzero(frame_min > thres)
    if idx.size:
        breaks = np.flatnonzero(np.diff(idx) != 1)
        starts = np.concatenate([[idx[0]], idx[breaks + 1]])
        ends = np.concatenate([idx[breaks], [idx[-1]]])
        prev_end = None
        for s, e in zip(starts, ends):
            if e - s <= min_range:
                continue
            s, e = int(s), int(e)
            if prev_end is not None and s - prev_end < fade_size:
                s = prev_end - fade_size * 2
            if s != 0:
                weight[s:s + fade_size] = np.linspace(0, 1, fade_size)
            else:
                s -= fade_size
            if e != n_frames:
                weight[e - fade_size:e] = np.linspace(1, 0, fade_size)
            else:
                e += fade_size
            weight[s + fade_size:e - fade_size] = 1
            prev_end = e
    return weight


def merge_artifacts(y_mask, thres=0.05, min_range=64, fade_size=32):
    """``--postprocess`` mask clean-up (reference lib/spec_utils.py:60-93) on a host array, in place."""
    weight = artifact_weights(y_mask.min(axis=(0, 1)), thres, min_range, fade_size)
    y_mask += weight[None, None, :] * (1 - y_mask)
    return y_mask


def _trim_silence(y, top_db=60, frame_length=2048, hop_length=512):
    """Restatement of ``librosa.effects.trim(y)`` (librosa 0.10 defaults; librosa is absent offline: parity unpinned like
    the STFT): frame RMS (centred frames, zero padding) -> dB relative to the maximum -> first / last frame above
    -top_db, per channel with the maximum taken across channels.  Returns (trimmed, (start, end))."""
    y = np.asarray(y)
    L = y.shape[-1]
    yp = np.pad(y.reshape(-1, L).astype(np.float64), ((0, 0), (frame_length // 2, frame_length // 2)))
    n_frames = 1 + (yp.shape[1] - frame_length) // hop_length
    csum = np.concatenate([np.zeros((yp.shape[0], 1)), np.cumsum(yp ** 2, axis=1)], axis=1)
    starts = np.arange(n_frames) * hop_length
    power = (csum[:, starts + frame_length] - csum[:, starts]) / frame_length
    rms = np.sqrt(np.maximum(power, 0.0))
    ref = rms.max()
    db = 20.0 * np.log10(np.maximum(1e-5, rms)) - 20.0 * np.log10(np.maximum(1e-5, ref))
    non_silent = (db > -top_db).max(axis=0)
    nz = np.flatnonzero(non_silent)
    if nz.size == 0:
        return y[..., 0:0], (0, 0)
    start = int(nz[0]) * hop_length
    end = min(L, (int(nz[-1]) + 1) * hop_length)
    return y[..., start:end], (start, end)


def align_wave_head_and_tail(a, b, sr):
    """lib/spec_utils.py:96-119: trim both tracks, estimate their delay from the cross-correlation of the first four
    seconds (mono sums, mean removed) and crop them to the common aligned span."""
    a, _ = _trim_silence(a)
    b, _ = _trim_silence(b)
    a_mono = a[:, :sr * 4].sum(axis=0)
    b_mono = b[:, :sr * 4].sum(axis=0)
    a_mono = a_mono - a_mono.mean()
    b_mono = b_mono - b_mono.mean()
    offset = len(a_mono) - 1
    # np.correlate(a, b, 'full') through the FFT (the direct form is O(n^2) on 4 s of audio)
    n = len(a_mono) + len(b_mono) - 1
    nfft = 1 << (n - 1).bit_length()
    corr = np.fft.irfft(np.fft.rfft(a_mono, nfft) * np.conj(np.fft.rfft(b_mono, nfft)), nfft)
    corr = np.concatenate([corr[nfft - (len(b_mono) - 1):], corr[:len(a_mono)]])
    delay = int(np.argmax(corr)) - offset   # as the reference: offset = len(a_mono) - 1
    if delay > 0:
        a = a[:, delay:]
    else:
        b = b[:, np.abs(delay):]
    if a.shape[1] < b.shape[1]:
        b = b[:, :a.shape[1]]
    else:
        a = a[:, :b.shape[1]]
    return a, b


def cache_or_load(mix_path, inst_path, sr, hop_length, n_fft):
    """lib/spec_utils.py:122-154: spectrograms of a (mixture, instruments) pair, cached next to the audio.

    The cache layout is the reference's - ``<dir>/sr{sr}_hl{hop}_nf{n_fft}/<basename>.npy`` holding the spectrogram
    transposed to (T, 2, bins) - so caches written by either implementation are interchangeable.  On a miss both files
    are decoded (non-``sr`` input is converted on the GPU, lib/audio_io.py), aligned and transformed with the GPU STFT.
    Returns (X, y, mix_cache_path, inst_cache_path) with X, y complex64 of shape (2, bins, T)."""
    import os
    from . import audio_io
    cache_dir = 'sr{}_hl{}_nf{}'.format(sr, hop_length, n_fft)
    paths = []
    for src in (mix_path, inst_path):
        d = os.path.join(os.path.dirname(src), cache_dir)
        os.makedirs(d, exist_ok=True)
        paths.append(os.path.join(d, os.path.splitext(os.path.basename(src))[0] + '.npy'))
    mix_cache_path, inst_cache_path = paths
    if os.path.exists(mix_cache_path) and os.path.exists(inst_cache_path):
        X = np.load(mix_cache_path).transpose(1, 2, 0)
        y = np.load(inst_cache_path).transpose(1, 2, 0)
    else:
        X, _ = audio_io.load(mix_path, sr=sr, mono=False, dtype=np.float32, device=_DEVICE_INDEX)
        y, _ = audio_io.load(inst_path, sr=sr, mono=False, dtype=np.float32, device=_DEVICE_INDEX)
        X, y = align_wave_head_and_tail(X, y, sr)
        X = wave_to_spectrogram(X, hop_length, n_fft)
        y = wave_to_spectrogram(y, hop_length, n_fft)
        np.save(mix_cache_path, X.transpose(2, 0, 1))
        np.save(inst_cache_path, y.transpose(2, 0, 1))
    assert X.shape == y.shape
    return X, y, mix_cache_path, inst_cache_path


def main(argv=None):
    """The reference's pair check: test_X / test_y / test_v .jpg and .wav of one aligned pair, in the working
    directory."""
    import argparse
    from . import audio_io, utils
    p = argparse.ArgumentParser(prog='lib/spec_utils.py',
                                description='aligns one (mixture, instruments) pair and writes test_X, test_y and '
                                            'test_v (= X - y) .jpg and .wav to the working directory')
    p.add_argument('mix')
    p.add_argument('inst')
    args = p.parse_args(argv)

    # missing requirements fail before any file is written
    try:
        import cv2  # noqa: F401  (the JPEG encoder of lib/utils.imwrite)
    except ImportError as e:
        raise ImportError('the pair check needs OpenCV (the cv2 module) to encode the JPGs: %s' % e) from e
    if not torch.cuda.is_available():
        raise RuntimeError('no CUDA device: the H100 build of vocal-remover has no CPU path')

    sr, hop_length, n_fft = 44100, 1024, 2048
    X, _ = audio_io.load(args.mix, sr=sr, mono=False, dtype=np.float32, device=_DEVICE_INDEX)
    y, _ = audio_io.load(args.inst, sr=sr, mono=False, dtype=np.float32, device=_DEVICE_INDEX)
    X, y = align_wave_head_and_tail(X, y, sr)
    X_spec = wave_to_spectrogram(X, hop_length, n_fft)
    y_spec = wave_to_spectrogram(y, hop_length, n_fft)
    v_spec = spectrogram_difference(X_spec, y_spec)

    specs = (('X', X_spec), ('y', y_spec), ('v', v_spec))
    if X_spec.shape[2] > utils.JPEG_MAX_WIDTH:
        # the encoder refuses the images: no JPG, the WAVs are still written
        print('skipping test_X.jpg, test_y.jpg and test_v.jpg: {} frames exceed the {}-pixel width limit of '
              'JPEG'.format(X_spec.shape[2], utils.JPEG_MAX_WIDTH))
    else:
        for name, spec in specs:
            utils.imwrite('test_{}.jpg'.format(name), spectrogram_to_image(spec))
    for name, spec in specs:
        audio_io.write('test_{}.wav'.format(name), spectrogram_to_wave(spec, hop_length).T, sr)


if __name__ == '__main__':
    main()
