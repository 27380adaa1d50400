"""CPU restatement of the sample-rate conversion the reference applies to non-44.1 kHz input:
``librosa.load(path, sr=args.sr, mono=False, dtype=np.float32, res_type='kaiser_fast')`` (reference
inference.py:136-138, pseudo.py:47-50), i.e. ``resampy.resample(y, orig_sr, sr, filter='kaiser_fast', axis=-1)``.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): the product path is vocal-remover_b200/csrc/resample.cu.

PARITY UNPINNED.  resampy (requirements.txt: ``resampy~=0.4.0``) is a third-party dependency that is neither under
the reference checkout nor installed offline, and the reference holds no golden vectors for this step.  What is restated here
is resampy 0.4's published algorithm:

* ``resampy.filters.sinc_window``: half of a Kaiser-windowed sinc, ``num_zeros`` zero crossings, ``2**precision`` table
  entries per crossing, cut-off ``rolloff`` x Nyquist;
* ``resampy.core.resample``: the table is scaled by the rate ratio when down-sampling, ``interp_delta`` is its first
  difference, ``t_out = arange(n_out) / ratio`` in float64, ``n_out = int(n_in * ratio)``;
* ``resampy.interpn._resample_loop``: for every output instant the left and the right wing of the filter are walked with
  stride ``int(scale * 2**precision)`` table entries, the table being interpolated linearly.

The pre-computed ``kaiser_fast`` table is described by resampy's documentation as 16 zero crossings, a Kaiser window of
beta = 8.555504641634386 and a roll-off of 0.85 x Nyquist; it is regenerated from those numbers with ``precision = 9``
(sinc_window's default).  A user with resampy installed can pass the exact table
(``resampy.filters.get_filter('kaiser_fast')[:2]``) as ``filt=(half_window, table_per_crossing)``.
The sanity anchor available offline is ``scipy.signal.resample_poly`` (tests/test_resample.py).
"""
import numpy as np

KAISER_FAST = dict(num_zeros=16, precision=9, rolloff=0.85, beta=8.555504641634386)


def sinc_window(num_zeros=16, precision=9, rolloff=0.85, beta=8.555504641634386):
    """resampy.filters.sinc_window with window = scipy.signal.windows.kaiser(., beta): (half window, entries per crossing)."""
    num_bits = 2 ** precision
    n = num_bits * num_zeros
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    taper = np.kaiser(2 * n + 1, beta)[n:]
    return taper * sinc_win, num_bits


def prepare(sr_orig, sr_new, filt=None):
    """(interp_win, interp_delta, num_table, scale, sample_ratio) as resampy.core.resample builds them."""
    if sr_orig <= 0 or sr_new <= 0:
        raise ValueError('Invalid sample rate')
    sample_ratio = float(sr_new) / sr_orig
    interp_win, num_table = sinc_window(**KAISER_FAST) if filt is None else (np.asarray(filt[0], np.float64), int(filt[1]))
    if sample_ratio < 1:
        interp_win = sample_ratio * interp_win
    interp_delta = np.diff(interp_win, append=interp_win[-1])
    return interp_win, interp_delta, num_table, min(1.0, sample_ratio), sample_ratio


def resample(x, sr_orig, sr_new, filt=None, out_range=None, time_dtype=np.float64):
    """x: (..., n) float array -> (..., int(n * sr_new / sr_orig)), same dtype (vectorised over the output instants).

    out_range=(t0, t1) computes only the output samples [t0, t1) of that result, with the same arithmetic: a window of
    a long signal costs memory in proportion to the window, not to the signal.  time_dtype is the type the output
    instants are rounded to: resampy's float64, or float32 to see what a single-precision time register computes."""
    x = np.asarray(x)
    interp_win, interp_delta, num_table, scale, ratio = prepare(sr_orig, sr_new, filt)
    n_in = x.shape[-1]
    n_out = int(n_in * ratio)
    if n_out < 1:
        raise ValueError('Input signal length=%d is too small to resample from %s->%s' % (n_in, sr_orig, sr_new))
    t0, t1 = (0, n_out) if out_range is None else (int(out_range[0]), int(out_range[1]))
    if not 0 <= t0 <= t1 <= n_out:
        raise ValueError('out_range [%d, %d) is outside the %d output samples' % (t0, t1, n_out))
    xf = x.reshape(-1, n_in).astype(np.float64)
    y = np.zeros((xf.shape[0], t1 - t0), np.float64)
    t_out = (np.arange(t0, t1) * (1.0 / ratio)).astype(time_dtype).astype(np.float64)
    n = t_out.astype(np.int64)
    nwin = interp_win.shape[0]
    index_step = int(scale * num_table)
    for wing in (0, 1):
        frac = scale * (t_out - n)
        if wing:
            frac = scale - frac
        index_frac = frac * num_table
        offset = index_frac.astype(np.int64)
        eta = index_frac - offset
        limit = (n + 1) if wing == 0 else (n_in - n - 1)
        taps = np.minimum(limit, (nwin - offset) // index_step)
        for i in range(int(taps.max()) if taps.size else 0):
            live = i < taps
            idx = np.where(live, offset + i * index_step, 0)
            w = np.where(live, interp_win[idx] + eta * interp_delta[idx], 0.0)
            src = np.where(live, (n - i) if wing == 0 else (n + i + 1), 0)
            y += w[None, :] * xf[:, src]
    return y.reshape(x.shape[:-1] + (t1 - t0,)).astype(x.dtype)


def resample_literal(x, sr_orig, sr_new, filt=None):
    """The loop of resampy.interpn._resample_loop as written there, one output sample at a time (small inputs only)."""
    x = np.asarray(x, np.float64)
    assert x.ndim == 1
    interp_win, interp_delta, num_table, scale, ratio = prepare(sr_orig, sr_new, filt)
    n_orig = x.shape[0]
    n_out = int(n_orig * ratio)
    t_out = np.arange(n_out) * (1.0 / ratio)
    y = np.zeros(n_out)
    index_step = int(scale * num_table)
    nwin = interp_win.shape[0]
    for t in range(n_out):
        time_register = t_out[t]
        n = int(time_register)
        frac = scale * (time_register - n)
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        i_max = min(n + 1, (nwin - offset) // index_step)
        for i in range(i_max):
            weight = interp_win[offset + i * index_step] + eta * interp_delta[offset + i * index_step]
            y[t] += weight * x[n - i]
        frac = scale - frac
        index_frac = frac * num_table
        offset = int(index_frac)
        eta = index_frac - offset
        k_max = min(n_orig - n - 1, (nwin - offset) // index_step)
        for k in range(k_max):
            weight = interp_win[offset + k * index_step] + eta * interp_delta[offset + k * index_step]
            y[t] += weight * x[n + k + 1]
    return y
