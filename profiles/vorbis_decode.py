"""Times the GPU Vorbis decoder (csrc/vorbis.cu through lib/vorbis.py) on 4-minute stereo 44.1 kHz Ogg Vorbis files at
two bitrates and on a 40-minute one at the lower, and ``separate_wave`` on the 4-minute track in the same run.

Each file is a 10-second ``synth.sine_mix`` encoded by the oracle (oracle/vorbis_oracle.py; long blocks of 2048,
residue type 2, the floor fitted ``gain`` below the spectral envelope: a higher gain spends more bits) with its
packets repeated in Ogg pages: a valid file whose decode cost is that of a real one of the same length and bitrate
(the oracle encoder is too slow for 40 minutes). Reported per file, as medians over --runs calls after warm-up: bytes
and packets; each kernel's time (torch.profiler) and their sum; the H2D and D2H copies per call; one whole
``vorbis.decode`` call (CUDA events around it, and host wall time); the host Ogg and setup parse (``vorbis.parse``
timed on its own). ``separate_wave`` runs the default CLI settings with a synthetic checkpoint (the cost does not
depend on the weights). The card's name and power limit are read in the same run (read-only
``nvidia-smi --query-gpu``).

Usage: python profiles/vorbis_decode.py [--runs 20] [--out vorbis_decode.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'vocal-remover_b200')):
    if p not in sys.path:
        sys.path.insert(0, p)


def _gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:
        return dict(gpu=None, nvidia_smi_error=str(e))


_TILES = {}


def _stream(gain, seconds):
    from lib import synth
    from oracle import vorbis_oracle as vo
    if gain not in _TILES:
        cfg = dict(bs=(8, 11), schedule=[1], rtype=2, mult=2, seed=int(gain), gain=gain)
        _TILES[gain] = vo.encode(synth.sine_mix(10.0).astype(np.float64), 44100, cfg)[:3]
    h, p, b = _TILES[gain]
    reps = int(np.ceil(seconds / 10.0))
    return vo.ogg(h, p * reps, b * reps)[0]


def _host_parse_ms(data, runs):
    from lib import vorbis
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        vorbis.parse(data)
        times.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(times))


KERNELS = ('parse', 'synth', 'overlap')


def _measure(data, runs):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from lib import vorbis
    for _ in range(3):
        vorbis.decode(data)
    torch.cuda.synchronize()
    call_ms, wall_ms = [], []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        a.record()
        vorbis.decode(data)
        b.record()
        b.synchronize()
        wall_ms.append(1e3 * (time.perf_counter() - w0))
        call_ms.append(a.elapsed_time(b))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            vorbis.decode(data)
        torch.cuda.synchronize()
    per = {}   # key -> [(start, ms)] in launch order
    for ev in prof.events():
        if ev.device_type.name != 'CUDA':
            continue
        name = ev.name
        key = next((k for k in KERNELS if 'vorbis_%s_kernel' % k in name), None)
        if key is None:
            key = 'memcpy HtoD' if 'HtoD' in name else ('memcpy DtoH' if 'DtoH' in name else None)
        if key is None:
            continue
        ms = (ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total) / 1e3
        per.setdefault(key, []).append((ev.time_range.start, ms))
    # every kernel runs once per call: the median over the calls; the copies run several times per call: their sum
    # per call (in launch order), then the median
    device = {}
    for k, v in per.items():
        ms = np.asarray([m for _, m in sorted(v)])
        if len(ms) % runs == 0:
            device[k] = float(np.median(ms.reshape(runs, -1).sum(axis=1)))
    kernel_sum = sum(v for k, v in device.items() if k in KERNELS)
    return dict(bytes=len(data), ms_per_call_median=float(np.median(call_ms)),
                wall_ms_median=float(np.median(wall_ms)), host_parse_ms_median=_host_parse_ms(data, runs),
                device_ms_per_call_median=device, decode_kernels_ms=kernel_sum)


def _separate_ms(x, runs):
    """Median CUDA-event time of Separator.separate_wave on x (channels, n) with the CLI's default settings."""
    import torch
    sys.path.insert(0, os.path.join(ROOT, 'vocal-remover_b200'))
    import inference
    from lib import nets, spec_utils, synth
    args = inference.build_parser().parse_args(['-P', 'unused', '-i', 'unused'])
    device = torch.device('cuda:0')
    model = nets.CascadedNet(args.n_fft, args.hop_length, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    model.to(device)
    spec_utils.set_device(0)
    sp = inference.Separator(model=model, device=device, batchsize=args.batchsize, cropsize=args.cropsize,
                             postprocess=args.postprocess, wiener_iterations=args.wiener_iterations)
    sp.separate_wave(x)
    times = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        sp.separate_wave(x)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from lib import vorbis
    assert torch.cuda.is_available(), 'profiles/vorbis_decode.py measures on the GPU'
    res = dict(_gpu_info(), torch_device=torch.cuda.get_device_name(0), runs=args.runs)
    for label, gain, seconds in (('4 min gain 4', 4.0, 240), ('4 min gain 32', 32.0, 240),
                                 ('40 min gain 4', 4.0, 2400)):
        data = _stream(gain, seconds)
        y, _, info = vorbis.decode(data)
        r = _measure(data, args.runs)
        r['packets'] = info['packets']
        r['kbit_per_s'] = 8.0 * len(data) / seconds / 1000.0
        if label == '4 min gain 4':
            r['separate_wave_ms_median'] = _separate_ms(y.cpu().numpy(), max(3, args.runs // 4))
        res[label] = r
        print(label, json.dumps(r), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict((k, v) for k, v in res.items() if not isinstance(v, dict))))


if __name__ == '__main__':
    main()
