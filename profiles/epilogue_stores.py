"""Per-layer time of the benchmark's workload under both epilogue stores of the wgmma convolutions (vr_debug_set key 9:
0 = 16-byte stores of 8 channels where the output allows them, 1 = epilogue_pair's 4-byte channel-pair stores;
csrc/tc_common.cuh, DESIGN 5.2, 5.3, 5.7).

The workload is bench.py's: CascadedNet(2048, 1024, 32, 128), the 240 s synthetic track, windows in batches of 27.
Each round runs one profiled step (vr_profile_enable: a CUDA event pair around every launch, band streams serialised)
under each key, alternating, after --warmup unprofiled steps; a layer's time is its summed launch time in a step, and
the table gives its median over --rounds rounds under each key, with the bytes of its output (N H W Cout, hi + lo bf16).
The card's name, power limit and SM clocks are read in the same run (read-only ``nvidia-smi --query-gpu``).

Usage: python profiles/epilogue_stores.py [--rounds 3] [--warmup 2] [--out epilogue_stores.json]
"""
import argparse
import collections
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'vocal-remover_b200')
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def _gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        name, power, max_clock, clock = [s.strip() for s in r.stdout.splitlines()[0].split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=max_clock, sm_clock=clock)
    except Exception as e:   # the numbers stay valid; the card is then named by torch only
        return dict(gpu=None, nvidia_smi_error=str(e))


def _profiled_step(ctx, step):
    """{(layer, N, H, W): summed ms} of the convolution launches of one profiled step"""
    ctx.check(ctx.lib.vr_profile_enable(ctx.handle, 1), 'vr_profile_enable')
    step()
    need = ctypes.c_int64(0)
    ctx.check(ctx.lib.vr_profile_dump(ctx.handle, None, 0, ctypes.byref(need)), 'vr_profile_dump')
    buf = ctypes.create_string_buffer(need.value)
    ctx.check(ctx.lib.vr_profile_dump(ctx.handle, buf, need.value, None), 'vr_profile_dump')
    ctx.check(ctx.lib.vr_profile_enable(ctx.handle, 0), 'vr_profile_enable')
    out = collections.OrderedDict()
    for ln in buf.value.decode().splitlines():
        name, n, h, w, tc, ms, _ = ln.split()
        if int(tc) != 1:   # not a convolution
            continue
        key = (name, int(h), int(w))
        a = out.setdefault(key, [0, 0.0])
        a[0] += int(n)
        a[1] += float(ms)
    return out


def _out_channels(state_dict):
    """{parameter path: output channels} of every convolution weight of the net"""
    return {name: t.shape[0] for name, t in state_dict.items() if name.endswith('weight') and t.dim() == 4}


def _cout(couts, layer):
    """output channels of a profiled layer (its name without the '+up' / '+mask' of fused work): the first
    convolution weight below its module path"""
    layer = layer.split('+')[0]
    for name, c in couts.items():
        if name.startswith(layer + '.'):
            return c
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--seconds', type=float, default=240.0)
    ap.add_argument('--batch', type=int, default=27)
    ap.add_argument('--out', type=str, default='')
    args = ap.parse_args()
    import torch
    import inference
    from lib import _native, nets, synth
    assert torch.cuda.is_available(), 'this profile needs a GPU'
    dev = torch.device('cuda:0')
    info = _gpu_info()
    model = nets.CascadedNet(2048, 1024, 32, 128)
    state = synth.to_torch_state_dict(synth.make_state_dict())
    model.load_state_dict(state)
    model.to(dev)
    sp = inference.Separator(model, dev, args.batch, 256, False)
    wave = torch.from_numpy(synth.sine_mix(args.seconds)).to(dev)
    ctx = sp._ctx()
    lib = _native.load_library()
    couts = _out_channels(state)

    def step():
        sp.separate_wave(wave)
        torch.cuda.synchronize()

    times = {0: collections.defaultdict(list), 1: collections.defaultdict(list)}
    counts = {}
    try:
        for key in (0, 1):
            assert lib.vr_debug_set(9, key) == 0
            for _ in range(args.warmup):
                step()
        for _ in range(args.rounds):
            for key in (0, 1):
                assert lib.vr_debug_set(9, key) == 0
                for k, (n, ms) in _profiled_step(ctx, step).items():
                    times[key][k].append(ms)
                    counts[k] = n
    finally:
        lib.vr_debug_set(9, 0)
    info_end = _gpu_info()
    rows = []
    for k in times[0]:
        name, h, w = k
        c = _cout(couts, name)
        rows.append(dict(layer=name, H=h, W=w, images=counts[k], cout=c,
                         out_bytes=counts[k] * h * w * c * 4 if c else None,
                         ms_16byte=statistics.median(times[0][k]), ms_pairs=statistics.median(times[1][k])))
    print('%s, power limit %s, max SM clock %s, SM clock at start %s / end %s' % (
        info.get('gpu'), info.get('power_limit'), info.get('max_sm_clock'), info.get('sm_clock'),
        info_end.get('sm_clock')))
    print('%-34s %5s %5s %6s %9s %9s %9s %6s' % ('layer', 'H', 'W', 'Cout', 'out MB', 'ms 16B', 'ms pairs', 'gain'))
    for r in rows:
        print('%-34s %5d %5d %6s %9s %9.3f %9.3f %5.1f%%' % (
            r['layer'], r['H'], r['W'], r['cout'] or '-', '%.1f' % (r['out_bytes'] / 1e6) if r['out_bytes'] else '-',
            r['ms_16byte'], r['ms_pairs'], 100.0 * (1.0 - r['ms_16byte'] / r['ms_pairs']) if r['ms_pairs'] else 0.0))
    t0, t1 = sum(r['ms_16byte'] for r in rows), sum(r['ms_pairs'] for r in rows)
    print('all convolutions: %.2f ms with 16-byte stores, %.2f ms with channel-pair stores' % (t0, t1))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(gpu=info, sm_clock_end=info_end.get('sm_clock'), rounds=args.rounds, rows=rows), f,
                      indent=1)


if __name__ == '__main__':
    main()
