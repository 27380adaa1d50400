"""Times the oracle separations of evaluate.py --oracle (DESIGN.md §12) on a 4-minute synthetic stereo pair.

Input: instruments ``0.4 * synth.sine_mix(240)`` and vocals ``0.4 * synth.sine_mix(120, sr=88200)`` (T = 10336 frames,
1025 bins at n_fft 2048, hop 1024), mixed.  Reported, as the median of --runs CUDA-event timings after warm-up:
- ``vr_oracle_mask`` per kind on the pair's spectrograms, with its bytes over the time: it reads the mixture and the
  instruments (16 B each per bin and frame, both channels) and writes the mask (8 B), 40 B per bin and frame, against
  the H100 SXM's 3.35 TB/s;
- each oracle's whole stem computation from the device waves (``spec_utils.oracle_separate_wave``: two STFTs, the mask
  or the filter, and the inverse STFTs).
The card's name and power limit are read in the same run (read-only ``nvidia-smi --query-gpu``).

Usage: python profiles/oracle.py [--seconds 240] [--runs 20] [--out oracle.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'vocal-remover_b200')
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

BYTES_PER_BIN_FRAME = 40
PEAK_TBPS = 3.35


def _gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # the numbers stay valid; the card is then named by torch only
        return dict(gpu=None, nvidia_smi_error=str(e))


def _median_ms(fn, runs, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--seconds', type=float, default=240.0)
    p.add_argument('--runs', type=int, default=20)
    p.add_argument('--out', type=str, default=None)
    args = p.parse_args()

    import torch
    from lib import _native, spec_utils, synth
    assert torch.cuda.is_available(), 'profiles/oracle.py needs a GPU'
    dev = torch.device('cuda:0')
    inst = 0.4 * synth.sine_mix(args.seconds)
    voc = 0.4 * synth.sine_mix(args.seconds / 2, sr=88200, seed=1)[:, :inst.shape[1]]
    X = torch.from_numpy((inst + voc).astype(np.float32)).to(dev)
    y = torch.from_numpy(inst.astype(np.float32)).to(dev)
    L = X.shape[1]
    T = 1 + L // 1024
    ctx = spec_utils._spectral_ctx(2048, 1024)
    Xs, Ys = (torch.empty((2, 1025, T), dtype=torch.complex64, device=dev) for _ in range(2))
    for w, s in ((X, Xs), (y, Ys)):
        ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(w), L, _native.ptr(s), T, None, _native.stream_ptr()),
                  'vr_stft')
    mask = torch.empty((2, 1025, T), dtype=torch.float32, device=dev)

    out = dict(_gpu_info(), torch_device=torch.cuda.get_device_name(dev), seconds=args.seconds, bins=1025, frames=T,
               runs=args.runs, mask_bytes=BYTES_PER_BIN_FRAME * 1025 * T, peak_TBps=PEAK_TBPS)
    out['mask_floor_ms'] = out['mask_bytes'] / (PEAK_TBPS * 1e12) * 1e3
    for k, kind in enumerate(spec_utils.MASK_ORACLES):
        def run(k=k):
            ctx.check(ctx.lib.vr_oracle_mask(ctx.handle, _native.ptr(Xs), _native.ptr(Ys), T, k, _native.ptr(mask),
                                             _native.stream_ptr()), 'vr_oracle_mask')
        ms = _median_ms(run, args.runs)
        out['mask_%s_ms' % kind] = ms
        out['mask_%s_TBps' % kind] = out['mask_bytes'] / (ms * 1e-3) / 1e12
    for kind in spec_utils.ORACLES:
        out['stems_%s_ms' % kind] = _median_ms(lambda: spec_utils.oracle_separate_wave(X, y, kind, 2048, 1024),
                                               args.runs)
    out['stems_iam_wiener1_ms'] = _median_ms(
        lambda: spec_utils.oracle_separate_wave(X, y, 'iam', 2048, 1024, wiener_iterations=1), args.runs)
    print(json.dumps(out))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
