"""Times the GPU FLAC decoder (csrc/flac.cu through lib/flac.py) on a 4-minute stereo 16-bit stream.

The stream is ``synth.sine_mix(240)`` quantised to 16 bits and written by the oracle's long-track encoder (FIXED or LPC
chosen per frame, block size 4096).  Reported: the stream's bytes and frames, the H2D copy of the compressed bytes
(pageable and pinned), the scan and decode kernel times (CUDA events, warm-up, median of --runs), the host chain step,
one whole ``flac.decode`` call, and whether the output equals ``int / 2^15`` exactly.  The card's name and power limit
are read in the same run (read-only ``nvidia-smi --query-gpu``).

Usage: python profiles/flac_decode.py [--runs 20] [--out flac_decode.json]
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
    return float(np.median(times)), float(np.min(times)), float(np.max(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from lib import _native, flac, synth
    from oracle import flac_oracle as fo
    assert torch.cuda.is_available(), 'profiles/flac_decode.py measures on the GPU'
    dev = torch.device('cuda:0')
    x = np.clip(np.round(synth.sine_mix(240.0).astype(np.float64) * 32768), -32768, 32767).astype(np.int64)
    t0 = time.perf_counter()
    data, info = fo.encode_long(x)
    encode_s = time.perf_counter() - t0

    lib = _native.load_library()
    start, si = flac.parse_metadata(data)
    end = flac.audio_end(data, start)
    host = torch.frombuffer(bytearray(data[:end]), dtype=torch.uint8)
    pinned = host.pin_memory()
    d_data = torch.empty(end, dtype=torch.uint8, device=dev)
    cap = 256 + end // 256
    cands = torch.empty((cap, 4), dtype=torch.int64, device=dev)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    stream = _native.stream_ptr()

    h2d_pageable = _median_ms(lambda: d_data.copy_(host), args.runs)
    h2d_pinned = _median_ms(lambda: d_data.copy_(pinned, non_blocking=True), args.runs)

    def scan():
        assert lib.vr_flac_scan(None, _native.ptr(d_data), end, start, _native.ptr(cands), cap, _native.ptr(count),
                                stream) == 0
    scan_ms = _median_ms(scan, args.runs)
    found = int(count.item())
    rows = cands[:found].cpu().numpy()
    t0 = time.perf_counter()
    frames, total = flac.build_chain(rows, start, end, si)
    chain_ms = (time.perf_counter() - t0) * 1e3
    out = torch.empty((si['channels'], total), dtype=torch.float32, device=dev)
    status = torch.empty(frames.shape[0], dtype=torch.int64, device=dev)
    d_frames = torch.from_numpy(frames).to(dev)

    def dec():
        assert lib.vr_flac_decode(None, _native.ptr(d_data), end, _native.ptr(d_frames), frames.shape[0],
                                  si['channels'], total, _native.ptr(out), _native.ptr(status), stream) == 0
    decode_ms = _median_ms(dec, args.runs)
    exact = bool(not status.cpu().numpy().any() and
                 np.array_equal(out.cpu().numpy(), x.astype(np.float32) / np.float32(32768)))

    walls = []
    for i in range(args.runs + 2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        y, _, _ = flac.decode(data)
        torch.cuda.synchronize()
        if i >= 2:
            walls.append((time.perf_counter() - t0) * 1e3)
    exact_api = bool(np.array_equal(y.cpu().numpy(), x.astype(np.float32) / np.float32(32768)))

    res = dict(_gpu_info(), torch_device=torch.cuda.get_device_name(0), stream_bytes=len(data),
               frames=int(frames.shape[0]), samples_per_channel=int(total), channels=si['channels'],
               candidates=found, encode_s=round(encode_s, 2),
               subframe_kinds=sorted('%s%d' % k for k in info['stats']['kinds']),
               h2d_pageable_ms=h2d_pageable, h2d_pinned_ms=h2d_pinned, scan_kernel_ms=scan_ms,
               decode_kernel_ms=decode_ms, chain_host_ms=round(chain_ms, 3),
               flac_decode_call_ms=[float(np.median(walls)), float(np.min(walls)), float(np.max(walls))],
               timing_note='kernel and copy entries: [median, min, max] over %d runs after 3 warm-up runs' % args.runs,
               exact=exact, exact_through_flac_decode=exact_api)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(json.dumps(res, indent=1) + '\n')


if __name__ == '__main__':
    main()
