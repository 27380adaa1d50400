"""Audio file I/O either side of the hot path (SURVEY 8(f) rank 2).

The reference uses ``librosa.load(path, sr=sr, mono=False, dtype=np.float32, res_type='kaiser_fast')`` and
``soundfile.write`` (inference.py:136-138,173,178).  FLAC and MP3 input are decoded on the GPU when there is one
(lib/flac.py, csrc/flac.cu; lib/mp3.py, csrc/mp3.cu), M4A / MP4 (AAC-LC) input always is (lib/aac.py, csrc/aac.cu),
and FLAC output encoded on it (csrc/flac_encode.cu); other
decoding and encoding stay on the host (soundfile when installed, else a stdlib ``wave``
reader for 8/16/24/32-bit PCM WAV and writer for 16-bit), except the samples of a 24-bit WAV, which are quantised and
packed on the GPU like the FLAC encoder's (``vr_pcm_pack``); the sample-rate conversion of non-``sr`` input - the
expensive part of ``librosa.load`` - runs on the GPU (``vr_resample``, csrc/resample.cu): resampy 0.4's algorithm with the
``kaiser_fast`` table taken from an installed resampy, or regenerated from its documented parameters otherwise
(oracle/resample_oracle.py states what is and is not pinned).
"""
import wave as _wave

import numpy as np

# resampy's documentation of the pre-computed 'kaiser_fast' filter: 16 zero crossings, Kaiser beta, roll-off x Nyquist
KAISER_FAST = dict(num_zeros=16, precision=9, rolloff=0.85, beta=8.555504641634386)


def kaiser_fast_table():
    """(half window float64, table entries per zero crossing) of resampy's 'kaiser_fast' filter."""
    try:
        import resampy
        half, per_crossing, _ = resampy.filters.get_filter('kaiser_fast')
        return np.asarray(half, np.float64), int(per_crossing)
    except ImportError:
        pass
    # resampy.filters.sinc_window with a Kaiser window
    per_crossing = 2 ** KAISER_FAST['precision']
    n = per_crossing * KAISER_FAST['num_zeros']
    sinc_win = KAISER_FAST['rolloff'] * np.sinc(KAISER_FAST['rolloff'] * np.linspace(0, KAISER_FAST['num_zeros'], num=n + 1,
                                                                                  endpoint=True))
    return np.kaiser(2 * n + 1, KAISER_FAST['beta'])[n:] * sinc_win, per_crossing


def resample(y, orig_sr, target_sr, device=None, filt=None):
    """resampy.resample(y, orig_sr, target_sr, filter='kaiser_fast', axis=-1) on the GPU.

    y: (n,) or (channels, n) float array (numpy, or a CUDA torch tensor to stay on the device); returns the same kind.
    filt: optional (half_window, entries_per_crossing) to override the table."""
    import torch
    from . import _native
    if orig_sr <= 0 or target_sr <= 0:
        raise ValueError('Invalid sample rate')
    is_tensor = isinstance(y, torch.Tensor)
    if not torch.cuda.is_available():
        raise RuntimeError('resample: no CUDA device (this package has no CPU path); install librosa + resampy to load '
                           'non-%d Hz input on the host' % target_sr)
    dev = y.device if is_tensor and y.is_cuda else torch.device(device if device is not None else 'cuda:0')
    x = (y if is_tensor else torch.from_numpy(np.ascontiguousarray(y, np.float32))).to(dev, torch.float32)
    squeeze = x.dim() == 1
    x = x.reshape(1, -1) if squeeze else x.reshape(-1, x.shape[-1])
    x = x.contiguous()
    ratio = float(target_sr) / float(orig_sr)
    n_in = x.shape[-1]
    n_out = int(n_in * ratio)
    if n_out < 1:
        raise ValueError('Input signal length=%d is too small to resample from %s->%s' % (n_in, orig_sr, target_sr))
    half, per_crossing = kaiser_fast_table() if filt is None else (np.asarray(filt[0], np.float64), int(filt[1]))
    if ratio < 1:
        half = ratio * half
    delta = np.diff(half, append=half[-1])
    lib = _native.load_library()
    with torch.cuda.device(dev):
        d_win = torch.from_numpy(half).to(dev)
        d_delta = torch.from_numpy(delta).to(dev)
        out = torch.empty((x.shape[0], n_out), dtype=torch.float32, device=dev)
        _native.check(lib, lib.vr_resample(None, _native.ptr(x), x.shape[0], n_in, _native.ptr(out), n_out, ratio,
                                           _native.ptr(d_win), _native.ptr(d_delta), int(half.shape[0]), per_crossing,
                                           _native.stream_ptr()), 'vr_resample')
        torch.cuda.current_stream().synchronize()   # d_win / d_delta go out of scope
    out = out[0] if squeeze else out.reshape(tuple(y.shape[:-1]) + (n_out,))
    return out if is_tensor else out.cpu().numpy().astype(np.asarray(y).dtype if np.asarray(y).dtype.kind == 'f' else np.float32)


def _decode(path, device=None):
    """(channels, n) float32 at the file's own rate.  FLAC, MPEG-1 Layer III and MP4 (recognised by content, in that
    order) are decoded on the GPU whenever a CUDA device is visible (lib/flac.py, lib/mp3.py, lib/aac.py); otherwise
    soundfile reads FLAC and MP3 if it is installed.  libsndfile has no MP4 reader, so an M4A without a CUDA device
    raises RuntimeError."""
    from . import aac, flac, mp3
    # (sniff, decode, what the file is, the decoder's source, soundfile reads it) in detection order
    formats = ((flac.sniff, flac.decode, 'a FLAC file', 'lib/flac.py', True),
               (mp3.sniff, mp3.decode, 'an MP3 file', 'lib/mp3.py', True),
               (aac.sniff, aac.decode, 'an MP4 / M4A file', 'lib/aac.py', False))
    fmt = next((f for f in formats if f[0](path)), None)
    if fmt is not None:
        import torch
        _, decode, what, source, soundfile_reads = fmt
        if torch.cuda.is_available():
            x, rate, _ = decode(path, device)
            return x.cpu().numpy(), rate
        if not soundfile_reads:
            raise RuntimeError('%s is %s: decoding it needs a CUDA device (%s; soundfile has no MP4 reader), and none '
                               'is visible' % (path, what, source))
    try:
        import soundfile as sf
        data, rate = sf.read(path, dtype='float32', always_2d=True)
        return np.ascontiguousarray(data.T), rate
    except ImportError:
        pass
    if fmt is not None:
        raise RuntimeError('%s is %s: decoding it needs a CUDA device (%s) or the soundfile module, and neither is '
                           'available' % (path, what, source))
    with _wave.open(path, 'rb') as f:
        nch, width, rate, nframes = f.getnchannels(), f.getsampwidth(), f.getframerate(), f.getnframes()
        raw = f.readframes(nframes)
    if width == 2:
        x = np.frombuffer(raw, dtype='<i2').astype(np.float32) / 32768.0
    elif width == 3:
        b = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        x = ((b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)) << 8 >> 8).astype(np.float32) / 8388608.0
    elif width == 4:
        x = np.frombuffer(raw, dtype='<i4').astype(np.float32) / 2147483648.0
    elif width == 1:
        x = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    else:
        raise RuntimeError('unsupported WAV sample width %d' % width)
    return np.ascontiguousarray(x.reshape(-1, nch).T), rate


def load(path, sr, mono=False, dtype=np.float32, device=None):
    """librosa.load(path, sr=sr, mono=mono, dtype=dtype, res_type='kaiser_fast'): (channels, n) or (n,) array, sr.
    As in librosa, the channels are averaged first (mono=True) and the result is then resampled."""
    x, rate = _decode(path, device)
    if mono or x.shape[0] == 1:
        x = x.mean(axis=0)
    if sr is not None and rate != sr:
        x = resample(x, rate, sr, device=device)
        rate = sr
    return np.ascontiguousarray(x.astype(dtype)), rate


def _write_wav24(path, data, sr):
    """24-bit PCM WAV of (L, channels) or (L,) float samples, a CUDA tensor or an array: clip(rint(x * 8388607)) in fp32,
    NaN -> 0.  With a CUDA device the samples are quantised and packed to 3 bytes there (lib/flac.pcm_bytes), soundfile
    or not, so that the file holds the integers a 24-bit FLAC of the same data does."""
    import torch
    if torch.cuda.is_available():
        from . import flac
        x = data if torch.is_tensor(data) else np.asarray(data, np.float32)
        channels = 1 if x.ndim == 1 else x.shape[1]
        raw = flac.pcm_bytes(x[None] if x.ndim == 1 else x.T, 24)   # (channels, L)
    else:
        data = data.cpu().numpy() if torch.is_tensor(data) else np.asarray(data)
        try:
            import soundfile as sf
            sf.write(path, data, sr, subtype='PCM_24')
            return
        except ImportError:
            pass
        v = np.rint(data.astype(np.float32) * np.float32(8388607.0))
        q = np.clip(np.where(np.isnan(v), np.float32(0.0), v), -8388608, 8388607).astype('<i4')
        channels = 1 if q.ndim == 1 else q.shape[1]
        raw = np.ascontiguousarray(q).view(np.uint8).reshape(-1, 4)[:, :3].tobytes()
    with open(path, 'wb') as fh, _wave.open(fh, 'wb') as f:
        f.setnchannels(channels)
        f.setsampwidth(3)
        f.setframerate(sr)
        f.writeframes(raw)


def write(path, data, sr, bits=16):
    """data: (L, channels) float array, like soundfile.write; ``bits``: 16 or 24 bits per written sample.  A ``.flac``
    path is encoded on the GPU whenever a CUDA device is visible (lib/flac.py), else by soundfile; with neither it
    raises before creating the file.  A 24-bit ``.wav`` is packed on the GPU when there is one (_write_wav24)."""
    if bits not in (16, 24):
        raise ValueError('%s: output samples are 16 or 24 bits wide, not %r' % (path, bits))
    if str(path).lower().endswith('.flac'):
        import torch
        if torch.cuda.is_available():
            from . import flac
            x = data if torch.is_tensor(data) else np.asarray(data, np.float32)
            flac.encode(x[None] if x.ndim == 1 else x.T, sr, path, bits=bits)   # (channels, L)
            return
        try:
            import soundfile as sf
        except ImportError:
            raise RuntimeError('%s: writing FLAC needs a CUDA device (lib/flac.py) or the soundfile module, and neither '
                               'is available' % path) from None
        if bits == 24:
            sf.write(path, data, sr, subtype='PCM_24')
        else:
            sf.write(path, data, sr)
        return
    if bits == 24:
        _write_wav24(path, data, sr)
        return
    try:
        import soundfile as sf
        sf.write(path, data, sr)
        return
    except ImportError:
        pass
    data = np.asarray(data)
    if data.ndim == 1:
        data = data[:, None]
    pcm = np.clip(np.round(data * 32767.0), -32768, 32767).astype('<i2')
    with open(path, 'wb') as fh, _wave.open(fh, 'wb') as f:   # a bad path fails in open(), before a Wave_write exists
        f.setnchannels(pcm.shape[1])
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes(pcm.tobytes())


class AsyncWriter(object):
    """Encode and write stems on worker threads while the caller carries on (the two ``sf.write`` calls of
    inference.py:173,178 are independent of each other and of the next file's separation); ``join`` re-raises the first
    failure.  The arrays are written as passed: do not modify them before ``join``."""

    def __init__(self):
        import threading
        self._threading = threading
        self._jobs = []

    def write(self, path, data, sr, bits=16):
        self.run(write, path, data, sr, bits)

    def run(self, fn, *args):
        """Runs ``fn(*args)`` on a worker thread (e.g. lib.utils.imwrite of the --output_image JPGs)."""
        box = {}

        def run():
            try:
                fn(*args)
            except BaseException as exc:   # handed to join()
                box['exc'] = exc

        t = self._threading.Thread(target=run, name='vr-write')
        t.start()
        self._jobs.append((t, box))

    def join(self):
        jobs, self._jobs = self._jobs, []
        first = None
        for t, box in jobs:
            t.join()
            if first is None and 'exc' in box:
                first = box['exc']
        if first is not None:
            raise first
