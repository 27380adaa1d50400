"""Times the multichannel Wiener filter (vr_wiener, csrc/wiener.cu) on a 4-minute stereo track, next to separating it.

Input: ``synth.sine_mix(240)`` (T = 10336 frames, 1025 bins), separated with the seeded checkpoint
(synth.make_state_dict): its STFT, mask and masked spectrograms are the filter's input.  Reported, as the median of
--runs CUDA-event timings after warm-up: ``vr_wiener`` at 1 and 3 iterations (each run restores the initial estimates
first, outside the timed window), and ``Separator.separate_wave`` of the same track on the device.  The bytes per
iteration are the unfused minimum, 112 per bin and frame: the statistics pass reads both estimates (32), the apply pass
reads the mixture (16) and both estimates (32) and writes both estimates (32); TB/s is those bytes over the time.  The
card's name and power limit are read in the same run (read-only ``nvidia-smi --query-gpu``).

Usage: python profiles/wiener.py [--seconds 240] [--runs 20] [--out wiener.json]
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

BYTES_PER_BIN_FRAME = 112


def _gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # the numbers stay valid; the card is then named by torch only
        return dict(gpu=None, nvidia_smi_error=str(e))


def _median_ms(fn, runs, prepare=None):
    import torch
    times = []
    for _ in range(runs):
        if prepare:
            prepare()
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
    import inference
    from lib import _native, nets, synth
    assert torch.cuda.is_available(), 'profiles/wiener.py needs a GPU'
    dev = torch.device('cuda:0')
    model = nets.CascadedNet(2048, 1024, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    model.to(dev)
    sp = inference.Separator(model, dev, 4, 256, False)
    ctx = sp._ctx()
    wave = torch.from_numpy(synth.sine_mix(args.seconds)).to(dev)
    L = wave.shape[1]
    T = 1 + L // 1024
    spec = torch.empty((2, 1025, T), dtype=torch.complex64, device=dev)
    ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(wave), L, _native.ptr(spec), T, None, _native.stream_ptr()),
              'vr_stft')
    mask = sp._mask_device(spec, False)
    y0, v0 = torch.empty_like(spec), torch.empty_like(spec)
    ctx.check(ctx.lib.vr_apply_mask(ctx.handle, _native.ptr(spec), _native.ptr(mask), T, _native.ptr(y0),
                                    _native.ptr(v0), _native.stream_ptr()), 'vr_apply_mask')
    y, v = y0.clone(), v0.clone()

    def restore():
        y.copy_(y0)
        v.copy_(v0)

    out = dict(_gpu_info(), torch_device=torch.cuda.get_device_name(dev), seconds=args.seconds, bins=1025, frames=T,
               runs=args.runs, bytes_per_iteration=BYTES_PER_BIN_FRAME * 1025 * T)
    for it in (1, 3):
        def run(it=it):
            ctx.check(ctx.lib.vr_wiener(ctx.handle, _native.ptr(spec), _native.ptr(y), _native.ptr(v), T, it,
                                        _native.stream_ptr()), 'vr_wiener')
        for _ in range(3):
            restore()
            run()
        ms = _median_ms(run, args.runs, restore)
        out['wiener_%d_ms' % it] = ms
        out['wiener_%d_TBps' % it] = it * out['bytes_per_iteration'] / (ms * 1e-3) / 1e12
    for _ in range(2):
        sp.separate_wave(wave)
    out['separate_wave_ms'] = _median_ms(lambda: sp.separate_wave(wave), args.runs)
    print(json.dumps(out))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
