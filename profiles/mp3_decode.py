"""Times the GPU MP3 decoder (csrc/mp3.cu through lib/mp3.py) on 4-minute stereo 44.1 kHz streams at 128 and 320 kbit/s
and on a 40-minute stream at 128 kbit/s.

Each stream is a 10-second ``synth.sine_mix`` encoded by the oracle (oracle/mp3_oracle.py, joint stereo, CBR) and
repeated: a valid stream whose decode cost is that of a real one of the same length and bitrate (the oracle encoder is
too slow for 40 minutes).  Reported per stream, as medians over --runs calls after warm-up: bytes and frames; each
kernel's time (torch.profiler) and their sum; the H2D and D2H copies per call; one whole ``mp3.decode`` call (CUDA
events around it, and host wall time); the host chain walk (``build_chain`` timed on its own).  The card's
name and power limit are read in the same run (read-only ``nvidia-smi --query-gpu``).

Usage: python profiles/mp3_decode.py [--runs 20] [--out mp3_decode.json]
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


def _stream(kbps, seconds):
    from lib import synth
    from oracle import mp3_oracle as mo
    tile = mo.encode(synth.sine_mix(10.0).astype(np.float64), 44100, kbps, mode='joint', seed=kbps)
    return tile * int(np.ceil(seconds / 10.0))


def _host_chain_ms(data, runs):
    """Median time of lib.mp3.build_chain (the host chain walk) on the stream's sync candidates in byte order, as
    vr_mp3_scan and the device sort hand them over (found here with numpy)."""
    from lib import codec, mp3
    start = codec.id3v2_size(data)
    end = mp3.audio_end(data, start)
    d = np.frombuffer(data, np.uint8)
    i = np.flatnonzero((d[:-1] == 0xFF) & ((d[1:] & 0xE0) == 0xE0))
    i = i[(i >= start) & (i + 4 <= end)]
    w = (d[i].astype(np.int64) << 24) | (d[i + 1].astype(np.int64) << 16) | (d[i + 2].astype(np.int64) << 8) | d[i + 3]
    cands = np.stack([i, w], axis=1)
    times = []
    for _ in range(runs):
        t0 = time.perf_counter()
        mp3.build_chain(cands, start, end)
        times.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(times)), len(cands)


KERNELS = ('scan', 'side_info', 'gather', 'pow43', 'huffman', 'stereo', 'hybrid', 'window', 'status')


def _measure(data, runs):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from lib import mp3
    for _ in range(3):
        mp3.decode(data)
    torch.cuda.synchronize()
    call_ms, wall_ms = [], []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        a.record()
        mp3.decode(data)
        b.record()
        b.synchronize()
        wall_ms.append(1e3 * (time.perf_counter() - w0))
        call_ms.append(a.elapsed_time(b))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            mp3.decode(data)
        torch.cuda.synchronize()
    per = {}   # key -> [(start, ms)] in launch order
    for ev in prof.events():
        if ev.device_type.name != 'CUDA':
            continue
        name = ev.name
        key = next((k for k in KERNELS if 'mp3_%s_kernel' % k in name), None)
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
    chain_ms, n_cands = _host_chain_ms(data, runs)
    return dict(bytes=len(data), sync_candidates=n_cands, ms_per_call_median=float(np.median(call_ms)),
                wall_ms_median=float(np.median(wall_ms)), chain_walk_ms_median=chain_ms,
                device_ms_per_call_median=device, decode_kernels_ms=kernel_sum)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from lib import mp3
    assert torch.cuda.is_available(), 'profiles/mp3_decode.py measures on the GPU'
    res = dict(_gpu_info(), torch_device=torch.cuda.get_device_name(0), runs=args.runs)
    for label, kbps, seconds in (('4 min 128 kbit/s', 128, 240), ('4 min 320 kbit/s', 320, 240),
                                 ('40 min 128 kbit/s', 128, 2400)):
        data = _stream(kbps, seconds)
        _, _, info = mp3.decode(data)
        r = _measure(data, args.runs)
        r['frames'] = info['frames']
        res[label] = r
        print(label, json.dumps(r))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict((k, v) for k, v in res.items() if not isinstance(v, dict))))


if __name__ == '__main__':
    main()
