"""Times every generic-kernel layer geometry of the benchmark's net (CascadedNet(2048, 1024, 32, 128), cropsize 256) at
batch 27 with each pairing of the generic wgmma convolution (vr_debug_set key 8: 1 = two warpgroups, 2 = PAIR_M,
3 = PAIR_N where the layer has two N tiles, 0 = the automatic choice; csrc/conv_tc.cu, DESIGN 5.3).

The geometries are the stride-2 enc*.conv1, the ASPP branches and bottleneck of the five BaseNets, and the two stage
bridges.  Each is run through vr_debug_conv with the library's per-launch CUDA events on (vr_profile_enable), and the
convolution launch's time is the median over --runs launches after --warmup.  Reported per geometry and key: ms per
launch, algorithmic TFLOP/s (2 N Ho Wo Cout Cin k^2 over the time), and the L2 -> SM operand bytes per FLOP the tiling
fetches (computed from the shapes: A boxes of 128 pixels and B boxes of BN rows, hi + lo bf16, per tap and channel).
The card's name, power limit and SM clocks are read in the same run (read-only ``nvidia-smi --query-gpu``).

Usage: python profiles/generic_conv.py [--batch 27] [--runs 10] [--warmup 3] [--out generic_conv.json]
"""
import argparse
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

NETS = [('stg1_low', 16, 512), ('stg1_high', 8, 512), ('stg2_low', 32, 512), ('stg2_high', 16, 512),
        ('stg3_full', 32, 1024)]
W = 256
NOUT = 32


def generic_layers():
    """{(Cin, H, W, Cout, k, stride, dh, dw, act): [layer names]} of the generic-kernel layers (input H x W)"""
    out = {}
    mult = [1, 2, 4, 6, 8]
    for net, n, H in NETS:
        for i in range(4):
            key = (n * mult[i], H >> i, W >> i, n * mult[i + 1], 3, 2, 1, 1, 2)
            out.setdefault(key, []).append('%s.enc%d.conv1' % (net, i + 2))
        c8, h16, w16 = 8 * n, H // 16, W // 16
        out.setdefault((c8, 1, w16, c8, 1, 1, 1, 1, 1), []).append(net + '.aspp.conv1.1')
        out.setdefault((c8, h16, w16, c8, 1, 1, 1, 1, 1), []).append(net + '.aspp.conv2')
        for j, (dh, dw) in enumerate([(4, 2), (8, 4), (12, 6)]):
            out.setdefault((c8, h16, w16, c8, 3, 1, dh, dw, 1), []).append('%s.aspp.conv%d' % (net, j + 3))
        out.setdefault((5 * c8, h16, w16, c8, 1, 1, 1, 1, 1), []).append(net + '.aspp.bottleneck')
    out.setdefault((NOUT // 2, 512, W, NOUT // 4, 1, 1, 1, 1, 1), []).append('stg1_low_band_net.1')
    out.setdefault((NOUT, 512, W, NOUT // 2, 1, 1, 1, 1, 1), []).append('stg2_low_band_net.1')
    return out


def _ceil(a, b):
    return -(-a // b)


def tiling(N, g):
    """the generic kernel's tiling of geometry g at batch N (tile_geom, n_tiling and tc_prepare in conv_tc.cu)"""
    Cin, H, Wi, Cout, k, s = g[:6]
    Ho, Wo = (H - 1) // s + 1, (Wi - 1) // s + 1
    cout16 = _ceil(Cout, 16) * 16
    n_tiles = _ceil(cout16, 128)
    BN = _ceil(_ceil(cout16, n_tiles), 16) * 16
    cin16 = _ceil(Cin, 16) * 16
    if Wo >= 128:
        Wt, Ht, Nt = 128, 1, 1
    else:
        Wt, Ht = Wo, min(128 // Wo, Ho)
        Nt = 128 // (Wt * Ht)
    m_tiles = (Wo // Wt) * (Ho // Ht) * _ceil(N, Nt)
    KB = 64 if cin16 % 64 == 0 else 32 if cin16 % 32 == 0 else 16
    return dict(Ho=Ho, Wo=Wo, BN=BN, n_tiles=n_tiles, m_tiles=m_tiles, CinPad=cin16, KB=KB,
                flops=2.0 * N * Ho * Wo * Cout * Cin * k * k)


def operand_bytes(t, k, mode):
    """L2 -> SM bytes of one launch: hi + lo bf16 (4 B) per pixel or weight row, per tap and padded input channel"""
    per = k * k * t['CinPad'] * 4
    m, nt, BN = t['m_tiles'], t['n_tiles'], t['BN']
    if mode == 'PAIR_M':
        return per * nt * (128 * m + BN * _ceil(m, 2))
    if mode == 'PAIR_N':
        return per * m * (128 + 2 * BN)
    return per * m * nt * (128 + BN)


def auto_mode(t, num_sms):
    """launch_pairing (conv_tc.cu) at key 8 = 0"""
    if t['KB'] > 32 or t['BN'] > 32:
        return 'NONE'
    pair = 'PAIR_N' if t['n_tiles'] == 2 and t['KB'] >= 32 else 'PAIR_M'
    units = t['m_tiles'] if pair == 'PAIR_N' else _ceil(t['m_tiles'], 2) * t['n_tiles']
    w1, w2 = _ceil(t['m_tiles'] * t['n_tiles'], num_sms), _ceil(units, num_sms)
    return pair if 19 * w2 <= 10 * w1 else 'NONE'


def _gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        name, power, max_clock, clock = [s.strip() for s in r.stdout.splitlines()[0].split(',')]
        return dict(gpu=name, power_limit=power, max_sm_clock=max_clock, sm_clock=clock)
    except Exception as e:   # the numbers stay valid; the card is then named by torch only
        return dict(gpu=None, nvidia_smi_error=str(e))


def _run_conv(ctx, x, w, b, g):
    """one vr_debug_conv of geometry g"""
    import torch
    from lib import _native
    Cin, H, Wi, Cout, k, s, dh, dw, act = g
    N = x.shape[0]
    Ho, Wo = (H - 1) // s + 1, (Wi - 1) // s + 1
    y = torch.empty((N, Cout, Ho, Wo), dtype=torch.float32, device='cuda')
    ctx.check(ctx.lib.vr_debug_conv(ctx.handle, _native.ptr(x), N, Cin, H, Wi, _native.ptr(w), _native.ptr(b), Cout,
                                    k, s, dh, dw, act, 1, _native.ptr(y), _native.stream_ptr()), 'vr_debug_conv')


def _profiled_ms(ctx):
    """CUDA-event ms of every convolution launch of vr_debug_conv since profiling was enabled"""
    need = ctypes.c_int64(0)
    ctx.check(ctx.lib.vr_profile_dump(ctx.handle, None, 0, ctypes.byref(need)), 'vr_profile_dump')
    buf = ctypes.create_string_buffer(need.value)
    ctx.check(ctx.lib.vr_profile_dump(ctx.handle, buf, need.value, None), 'vr_profile_dump')
    return [float(ln.split()[5]) for ln in buf.value.decode().splitlines() if ln.split()[0] == 'debug_conv']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=27)
    ap.add_argument('--runs', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', type=str, default='')
    args = ap.parse_args()
    import torch
    from lib import _native
    assert torch.cuda.is_available(), 'generic_conv.py times the GPU kernels: it needs a CUDA device'
    info = _gpu_info()
    info['torch_device'] = torch.cuda.get_device_name(0)
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = _native.Context(0, 2048, 1024, NOUT, 128, 256, 1, 0)
    modes = [(1, 'NONE'), (2, 'PAIR_M'), (3, 'PAIR_N'), (0, 'auto')]
    rows = []
    N = args.batch
    print('# %s, power limit %s, max SM clock %s (SM clock %s at start); batch %d, median of %d launches'
          % (info.get('gpu') or info['torch_device'], info.get('power_limit'), info.get('max_sm_clock'),
             info.get('sm_clock'), N, args.runs))
    print('%-28s %-38s %5s %5s %6s  %-8s %8s %7s %8s' % ('layers', 'Cin,H,W,Cout,k,s,dh,dw', 'BN', 'nt', 'mt', 'key',
                                                         'ms', 'TFLOP/s', 'B/FLOP'))
    try:
        for gi, (g, names) in enumerate(generic_layers().items()):
            Cin, H, Wi, Cout, k = g[:5]
            t = tiling(N, g)
            gen = torch.Generator().manual_seed(gi)
            x = torch.randn(N, Cin, H, Wi, generator=gen).cuda()
            w = (torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5).cuda()
            b = (torch.randn(Cout, generator=gen) * 0.1).cuda()
            auto = auto_mode(t, num_sms)
            for key, mode in modes:
                if mode == 'PAIR_N' and not (t['n_tiles'] == 2 and t['KB'] >= 32):
                    continue
                ctx.lib.vr_debug_set(8, key)
                for _ in range(args.warmup):
                    _run_conv(ctx, x, w, b, g)
                ctx.check(ctx.lib.vr_profile_enable(ctx.handle, 1), 'vr_profile_enable')
                for _ in range(args.runs):
                    _run_conv(ctx, x, w, b, g)
                ms = statistics.median(_profiled_ms(ctx))
                ctx.check(ctx.lib.vr_profile_enable(ctx.handle, 0), 'vr_profile_enable')
                ran = auto if mode == 'auto' else mode
                bpf = operand_bytes(t, k, ran) / t['flops']
                row = dict(layers=names, geometry=list(g), batch=N, key=key, mode=ran, ms=ms,
                           tflops=t['flops'] / ms * 1e-9, operand_bytes_per_flop=bpf, **t)
                rows.append(row)
                print('%-28s %-38s %5d %5d %6d  %-8s %8.4f %7.1f %8.4f' % (
                    names[0] + ('' if len(names) == 1 else ' +%d' % (len(names) - 1)), ','.join(map(str, g[:8])),
                    t['BN'], t['n_tiles'], t['m_tiles'], '%d %s' % (key, ran if key == 0 else ''), ms,
                    row['tflops'], bpf))
    finally:
        ctx.lib.vr_debug_set(8, 0)
        ctx.close()
    info_end = _gpu_info()
    print('# SM clock at end: %s' % info_end.get('sm_clock'))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(gpu=info, sm_clock_end=info_end.get('sm_clock'), rows=rows), f, indent=1)


if __name__ == '__main__':
    main()
