"""H100-native mirror of the reference's lib/spec_utils.py for the inference path.

wave_to_spectrogram / spectrogram_to_wave keep the reference signatures and numpy in / numpy out
contract (lib/spec_utils.py:26-31, 157-165) but run the framed FFT / inverse FFT + overlap-add on the
GPU through libvr_b200.so (csrc/fft.cu) instead of librosa on the host.  spectrogram_to_image (--output_image) builds
its uint8 image on the GPU as well (csrc/elementwise.cu).
"""
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
        if on_device:
            if spec.device != dev:
                raise ValueError('spectrogram_to_image: spec is on %s, the spectral functions use %s' % (spec.device, dev))
            d_spec = spec.to(torch.complex64).contiguous()
        else:
            d_spec = torch.from_numpy(np.ascontiguousarray(np.asarray(spec, dtype=np.complex64))).to(dev)
        img = torch.empty((bins, T, 3), dtype=torch.uint8, device=dev)
        ctx.check(ctx.lib.vr_spec_image(ctx.handle, _native.ptr(d_spec), None, T, _native.ptr(img), None,
                                        _native.stream_ptr()), 'vr_spec_image')
        return img if on_device else img.cpu().numpy()


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
