"""BSS Eval energy ratios of separated stems against true stems, on the GPU (csrc/bsseval.cu, DESIGN.md section 10).

The SiSEC convention: bss_eval_images with one set of time-invariant distortion filters per track.  Every estimate
channel is projected on the ``filters_len`` delays of every reference channel (P_all) and of its own source's channels
(P_j) by least squares, and each frame's SDR, ISR, SIR and SAR in dB follow from the energies of

    s_true = s,  e_spat = P_j - s,  e_interf = P_all - P_j,  e_artif = shat - P_all

over the frame and the source's channels.  A frame in which any reference source or any estimate is all zeros is NaN
for every source.  ``track_medians`` gives the per-track value: the median over the frames that are not NaN.

With ``framewise=True`` the metric is BSS Eval v3 instead (museval's mode 'v3', the SiSEC campaigns before 2018):
every frame is scored as a signal of its own, with distortion filters solved on its samples alone and projections on
its timeline of window + filters_len - 1 samples.
"""
import numpy as np
import torch

from . import _native

METRICS = ('sdr', 'isr', 'sir', 'sar')
MAX_SIGNALS = 8        # K * C, BSS_EVAL_MAX_SIGNALS of include/vr_b200.h
MAX_FILTER = 1024      # filters_len, BSS_EVAL_MAX_FILTER


def frame_count(n_samples, window, hop):
    """Frames of a track of ``n_samples``: frame w covers [w * hop, w * hop + window), none reaches past the end."""
    return (int(n_samples) - int(window) + int(hop)) // int(hop)


def _as_device(x, dev, what):
    if torch.is_tensor(x):
        if not x.is_cuda or x.device != dev:
            raise ValueError('%s is on %s, the evaluation runs on %s' % (what, x.device, dev))
        return x.to(torch.float32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32))).to(dev)


def _device_of(references, estimates, device):
    if device is not None:
        dev = torch.device(device) if not isinstance(device, int) else torch.device('cuda', device)
        if dev.type != 'cuda':
            raise ValueError('bss_eval runs on a CUDA device, not %s' % dev)
        return dev if dev.index is not None else torch.device('cuda', torch.cuda.current_device())
    for x in (references, estimates):
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    return torch.device('cuda', torch.cuda.current_device())


def _check_sizes(shape_s, shape_e, window, hop, filters_len):
    if tuple(shape_s) != tuple(shape_e) or len(shape_s) != 3:
        raise ValueError('references and estimates must both have shape (K, C, N), got %s and %s'
                         % (tuple(shape_s), tuple(shape_e)))
    K, C, N = shape_s
    if K < 1 or C < 1 or K * C > MAX_SIGNALS:
        raise ValueError('K * C (sources x channels) must be in [1, %d], got %d x %d' % (MAX_SIGNALS, K, C))
    if not 1 <= filters_len <= MAX_FILTER:
        raise ValueError('filters_len must be in [1, %d], got %r' % (MAX_FILTER, filters_len))
    if window < 1 or hop < 1:
        raise ValueError('window and hop must be positive, got %r and %r' % (window, hop))
    if N < window:
        raise ValueError('the signals (%d samples) are shorter than one window (%d)' % (N, window))


WORKSPACE_CAP = 4 << 30   # the framewise workspace budget: a quarter of the free device memory, at most this


def framewise_batch(lib, K, C, N, window, hop, filters_len, budget):
    """The largest number of frames per batch, at most the frame count, whose framewise workspace fits ``budget``
    bytes; ValueError if even one frame does not."""
    def need(f):
        nbytes = lib.vr_bss_eval_framewise_workspace(K, C, N, filters_len, window, hop, f)
        if nbytes < 0:
            raise ValueError(lib.vr_last_error(None).decode())
        return nbytes

    lo, hi = 1, min(frame_count(N, window, hop), 4096)
    if need(lo) > budget:
        raise ValueError('one frame of framewise BSS Eval needs %d bytes of device workspace, over the budget of %d'
                         % (need(lo), budget))
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if need(mid) <= budget:
            lo = mid
        else:
            hi = mid - 1
    return lo


def frame_sums(references, estimates, window, hop, filters_len=512, device=None, correlations=False, timings=False,
               framewise=False, frames_per_batch=None):
    """The device evaluation without the ratios: a dict with 'sums', float64 (K, nwin, 8), the per-frame sums over the
    source's channels of s^2, (P_j - s)^2, (shat - s)^2, P_j^2, (P_all - P_j)^2, P_all^2, (shat - P_all)^2 and shat^2;
    'loading', the K + 1 diagonal loading scales the systems were solved with (all unknowns, then each source: eps =
    scale * max diag G, 2^-40 unless a factorisation needed more); with ``correlations`` also 'corr',
    (K*C, 2*K*C, filters_len) r[a][b](l) = sum_u s_a(u) y_b(u + l) with y the references then the estimates (G and d);
    with ``timings`` also 'phase_ms', the CUDA-event times of correlations,
    solves, projections and the whole call.

    ``framewise``: BSS Eval v3, every frame scored as a signal of its own (DESIGN.md section 10, "Framewise filters
    (v3)"), ``window >= filters_len``.  The sums are then over each frame's timeline of window + filters_len - 1
    samples, 'loading' is (nwin, K + 1) with NaN rows for silent frames, 'corr' is (nwin, K*C, 2*K*C, filters_len) and
    'frames_per_batch' the batch the frames were solved in: ``frames_per_batch``, or when None the largest that fits a
    quarter of the device's free memory, at most WORKSPACE_CAP bytes.  The results do not depend on it."""
    window, hop, filters_len = int(window), int(hop), int(filters_len)
    _check_sizes(np.shape(references), np.shape(estimates), window, hop, filters_len)
    if framewise and window < filters_len:
        raise ValueError('with framewise filters the window (%d samples) must not be shorter than filters_len (%d)'
                         % (window, filters_len))
    K, C, N = (int(v) for v in np.shape(references))
    if not torch.is_tensor(references) and not np.any(references):
        raise ValueError('every reference is zero: the ratios are undefined')
    for x, what in ((references, 'references'), (estimates, 'estimates')):
        if not torch.is_tensor(x) and not np.all(np.isfinite(x)):
            raise ValueError('the %s hold NaN or Inf' % what)
    dev = _device_of(references, estimates, device)
    lib = _native.load_library()
    with torch.cuda.device(dev):
        s = _as_device(references, dev, 'references')
        e = _as_device(estimates, dev, 'estimates')
        if not bool(torch.any(s != 0)):
            raise ValueError('every reference is zero: the ratios are undefined')
        for x, what in ((s, 'references'), (e, 'estimates')):
            if not bool(torch.isfinite(x).all()):
                raise ValueError('the %s hold NaN or Inf' % what)
        nwin = frame_count(N, window, hop)
        sums = np.empty((K, nwin, 8), dtype=np.float64)
        phase = np.empty(4, dtype=np.float64) if timings else None
        if framewise:
            if frames_per_batch is None:
                free, _ = torch.cuda.mem_get_info(dev)
                frames_per_batch = framewise_batch(lib, K, C, N, window, hop, filters_len,
                                                   min(free // 4, WORKSPACE_CAP))
            frames_per_batch = int(frames_per_batch)
            name, batch, per_frame = 'vr_bss_eval_framewise', (frames_per_batch,), (nwin,)
        else:
            name, batch, per_frame = 'vr_bss_eval', (), ()
        nbytes = getattr(lib, name + '_workspace')(K, C, N, filters_len, window, hop, *batch)
        if nbytes < 0:
            raise ValueError(lib.vr_last_error(None).decode())
        ws = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
        corr = np.empty(per_frame + (K * C, 2 * K * C, filters_len), dtype=np.float64) if correlations else None
        loading = np.empty(per_frame + (K + 1,), dtype=np.float64)
        rc = getattr(lib, name)(None, _native.ptr(s), _native.ptr(e), K, C, N, filters_len, window, hop, *batch,
                                _native.ptr(ws), int(nbytes), sums.ctypes.data,
                                None if corr is None else corr.ctypes.data, loading.ctypes.data,
                                None if phase is None else phase.ctypes.data, _native.stream_ptr())
        _native.check(lib, rc, name)
    out = {'sums': sums, 'loading': loading}
    if framewise:
        out['frames_per_batch'] = frames_per_batch
    if correlations:
        out['corr'] = corr
    if timings:
        out['phase_ms'] = phase
    return out


def metrics(sums):
    """(K, nwin, 8) frame sums -> dict of (K, nwin) float64 'sdr', 'isr', 'sir', 'sar' in dB, NaN in every frame where
    some reference source or some estimate is all zeros."""
    q = np.asarray(sums, dtype=np.float64)
    with np.errstate(divide='ignore', invalid='ignore'):
        out = {'isr': 10 * np.log10(q[..., 0] / q[..., 1]),
               'sdr': 10 * np.log10(q[..., 0] / q[..., 2]),
               'sir': 10 * np.log10(q[..., 3] / q[..., 4]),
               'sar': 10 * np.log10(q[..., 5] / q[..., 6])}
    silent = np.any((q[..., 0] == 0) | (q[..., 7] == 0), axis=0)
    for m in out:
        out[m][:, silent] = np.nan
    return {m: out[m] for m in METRICS}


def bss_eval(references, estimates, window, hop, filters_len=512, device=None, framewise=False):
    """SDR, ISR, SIR and SAR of every frame of ``estimates`` against ``references``.

    references, estimates: (K, C, N) float32 numpy arrays or CUDA tensors (K sources of C channels, K * C <= 8).
    window, hop: frame length and advance in samples; filters_len: taps of the distortion filters (<= 1024).
    framewise: BSS Eval v3 (museval's mode 'v3'), distortion filters solved for each frame on its own samples,
    instead of one set per track (v4); needs window >= filters_len.
    Returns a dict of (K, nwin) float64 numpy arrays 'sdr', 'isr', 'sir', 'sar' (dB), nwin = frame_count(N, window,
    hop).  Raises ValueError for different shapes, N < window, all-zero references or NaN / Inf input."""
    return metrics(frame_sums(references, estimates, window, hop, filters_len, device, framewise=framewise)['sums'])


def track_medians(result):
    """Per-track values: the median of each source's frames that are not NaN (NaN if there is none); dict of (K,)."""
    out = {}
    for m in METRICS:
        v = np.asarray(result[m], dtype=np.float64)
        med = np.full(v.shape[0], np.nan)
        for k in range(v.shape[0]):
            ok = v[k][~np.isnan(v[k])]
            if ok.size:
                med[k] = np.median(ok)
        out[m] = med
    return out
