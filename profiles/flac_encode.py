"""Times the GPU FLAC encoder (csrc/flac_encode.cu through lib/flac.py) on 4-minute stereo input.

Inputs: ``synth.sine_mix(240)`` and the two stems of separating it with the seeded checkpoint (synth.make_state_dict).
Reported per input: the analyse and pack kernel times (CUDA events, warm-up, median of --runs), one whole
``flac.encode`` call with and without the host MD5 (CUDA events around the call, which ends in copies to the host),
bytes in (float32) and out, the ratio to a 16-bit WAV, and the separation of the same track for comparison.  With
--cli, also the wall time of ``inference.py`` with ``--output_format wav`` and ``flac``, alternating.  The card's name
and power limit are read in the same run (read-only ``nvidia-smi --query-gpu``).

Usage: python profiles/flac_encode.py [--runs 20] [--cli 2] [--out flac_encode.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'vocal-remover_b200')
for p in (ROOT, PKG):
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
    return [float(np.median(times)), float(np.min(times)), float(np.max(times))]


def _kernels(x, runs):
    """analyse and pack kernel times of one input, as lib/flac.encode_frames launches them"""
    import torch
    from lib import _native, flac
    lib = _native.load_library()
    C, n = x.shape
    F = (n + flac.BLOCK - 1) // flac.BLOCK
    code, value = flac.rate_code(44100)
    pcm = torch.empty((n, C), dtype=torch.int16, device=x.device)
    plan = torch.empty((F, flac.PLAN_INTS), dtype=torch.int32, device=x.device)
    st = _native.stream_ptr()

    def analyse():
        assert lib.vr_flac_encode_analyse(None, _native.ptr(x), C, n, code, _native.ptr(pcm), _native.ptr(plan), st) == 0
    analyse_ms = _median_ms(analyse, runs)
    sizes = plan[:, 0].cpu().numpy().astype(np.int64)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)[:-1]])).to(x.device)
    out = torch.empty(int(sizes.sum()), dtype=torch.uint8, device=x.device)
    status = torch.empty(F, dtype=torch.int32, device=x.device)

    def pack():
        assert lib.vr_flac_encode_pack(None, _native.ptr(pcm), C, n, _native.ptr(plan), _native.ptr(offsets), code,
                                       value, _native.ptr(out), _native.ptr(status), st) == 0
    pack_ms = _median_ms(pack, runs)
    assert not status.cpu().numpy().any()
    return F, analyse_ms, pack_ms


def _cli(runs):
    """wall time of inference.py on a 4-minute 16-bit WAV, --output_format wav and flac alternating"""
    import torch
    from lib import synth
    walls = dict(wav=[], flac=[])
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, 'mix.wav')
        x = np.clip(np.round(synth.sine_mix(240.0) * np.float32(32767)), -32768, 32767).astype('<i2')
        with wave.open(src, 'wb') as f:
            f.setnchannels(2)
            f.setsampwidth(2)
            f.setframerate(44100)
            f.writeframes(np.ascontiguousarray(x.T).tobytes())
        ckpt = os.path.join(tmp, 'synthetic.pth')
        torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
        sizes = {}
        for i in range(runs):
            for fmt in ('wav', 'flac'):
                out = os.path.join(tmp, '%s%d' % (fmt, i))
                t0 = time.perf_counter()
                r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt, '-i', src,
                                    '-o', out, '--output_format', fmt], capture_output=True, text=True, cwd=PKG)
                walls[fmt].append(round(time.perf_counter() - t0, 2))
                assert r.returncode == 0, r.stderr
                sizes[fmt] = sum(os.path.getsize(os.path.join(out, f)) for f in os.listdir(out))
    return dict(cli_wall_s=walls, cli_output_bytes=sizes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--cli', type=int, default=0, help='CLI runs per format (0: skip)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    import inference
    from lib import flac, nets, synth
    assert torch.cuda.is_available(), 'profiles/flac_encode.py measures on the GPU'
    dev = torch.device('cuda:0')
    mix = torch.from_numpy(synth.sine_mix(240.0)).to(dev)
    model = nets.CascadedNet(2048, 1024, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    model.to(dev)
    sp = inference.Separator(model, dev, 4, 256, False)
    separate_ms = _median_ms(lambda: sp.separate_wave(mix), max(3, args.runs // 4), warmup=2)
    inst, voc = sp.separate_wave(mix)
    res = dict(_gpu_info(), torch_device=torch.cuda.get_device_name(0), separate_wave_4min_ms=separate_ms, inputs={})
    for name, x in (('sine_mix', mix), ('instruments', inst), ('vocals', voc)):
        frames, analyse_ms, pack_ms = _kernels(x, args.runs)
        call_ms = _median_ms(lambda: flac.encode(x, 44100), args.runs)
        call_nomd5_ms = _median_ms(lambda: flac.encode(x, 44100, md5=False), args.runs)
        data = flac.encode(x, 44100)
        wav = 44 + x.numel() * 2
        res['inputs'][name] = dict(frames=frames, samples_per_channel=int(x.shape[1]), bytes_in_float32=x.numel() * 4,
                                   bytes_out=len(data), wav16_bytes=wav, ratio_to_wav16=round(len(data) / wav, 4),
                                   analyse_kernel_ms=analyse_ms, pack_kernel_ms=pack_ms, encode_call_ms=call_ms,
                                   encode_call_no_md5_ms=call_nomd5_ms)
    stems = res['inputs']
    res['both_stems_kernels_ms'] = round(sum(stems[s]['analyse_kernel_ms'][0] + stems[s]['pack_kernel_ms'][0]
                                             for s in ('instruments', 'vocals')), 3)
    res['timing_note'] = ('[median, min, max] over %d runs after 3 warm-up runs; separate_wave over %d runs'
                          % (args.runs, max(3, args.runs // 4)))
    if args.cli:
        res.update(_cli(args.cli))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(json.dumps(res, indent=1) + '\n')


if __name__ == '__main__':
    main()
