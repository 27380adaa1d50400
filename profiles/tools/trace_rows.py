"""Timeline of CTA 0 of the row-streaming convolution (vr_debug_set(0, 1) + vr_debug_trace): how long the TMA producer
and the interpolation warps wait for operand slots (role 0, the consumers, is not recorded).  Runs one layer through the debug entry points.

Needs a library built with the timeline compiled in:
    VR_BUILD_TAG=trace VR_BUILD_FLAGS=-DVR_TRACE python vocal-remover_b200/build.py
    VR_LIB_PATH=vocal-remover_b200/libvr_b200_trace.so python profiles/tools/trace_rows.py ...

    python profiles/tools/trace_rows.py conv    N Cin H W Cout        (3x3 stride-1 convolution, TMA rows only)
    python profiles/tools/trace_rows.py decoder N Cl h w Cs Cout      (fused bilinear x2 of the low tensor + skip)
"""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'vocal-remover_b200'))
from lib import _native  # noqa: E402


def main():
    kind = sys.argv[1]
    a = [int(x) for x in sys.argv[2:]]
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    lib = ctx.lib
    g = torch.Generator().manual_seed(0)
    for rep in range(2):
        lib.vr_debug_set(0, rep)   # first pass warms up, second is traced
        if kind == 'conv':
            N, Cin, H, W, Cout = a
            x = torch.randn(N, Cin, H, W, generator=g).cuda()
            w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5).cuda()
            b = torch.zeros(Cout).cuda()
            y = torch.empty((N, Cout, H, W), device='cuda')
            ctx.check(lib.vr_debug_conv(ctx.handle, _native.ptr(x), N, Cin, H, W, _native.ptr(w), _native.ptr(b), Cout, 3, 1,
                                        1, 1, 1, 1, _native.ptr(y), _native.stream_ptr()), 'vr_debug_conv')
        else:
            N, Cl, h, w_, Cs, Cout = a
            low = torch.randn(N, Cl, h, w_, generator=g).cuda()
            skip = torch.randn(N, Cs, 2 * h, 2 * w_, generator=g).cuda()
            wgt = (torch.randn(Cout, Cl + Cs, 3, 3, generator=g) / ((Cl + Cs) * 9) ** 0.5).cuda()
            b = torch.zeros(Cout).cuda()
            y = torch.empty((N, Cout, 2 * h, 2 * w_), device='cuda')
            ctx.check(lib.vr_debug_decoder(ctx.handle, _native.ptr(low), N, Cl, h, w_, _native.ptr(skip), Cs,
                                           _native.ptr(wgt), _native.ptr(b), Cout, 1, 1, _native.ptr(y),
                                           _native.stream_ptr()), 'vr_debug_decoder')
        torch.cuda.synchronize()
    lib.vr_debug_set(0, 0)
    n = 3 * 2048 * 3
    buf = (ctypes.c_uint64 * n)()
    got = lib.vr_debug_trace(ctypes.cast(buf, ctypes.c_void_p), n)
    assert got == n, got
    t = np.frombuffer(buf, dtype=np.uint64).reshape(3, 2048, 3).astype(np.int64)
    mma, tma, itp = t[0], t[1], t[2]
    nm = int((mma[:, 2] > 0).sum())
    mma = mma[:nm]
    if nm > 20:
        print('consumers: %d rows' % nm)
        per_row = np.diff(mma[:, 2])
        wait = mma[:, 1] - mma[:, 0]
        print('  cycles between consecutive rows (issue end to issue end): median %d  mean %.0f  p10 %d  p90 %d' % (
            np.median(per_row), per_row.mean(), np.percentile(per_row, 10), np.percentile(per_row, 90)))
        print('  operand wait per row: median %d  mean %.0f  p90 %d  share of time %.2f' % (
            np.median(wait), wait.mean(), np.percentile(wait, 90), wait[1:].sum() / max(1, per_row.sum())))
        k = min(nm, 60)
        print('  first rows: per-row cycles', per_row[:k].tolist())
        print('  first rows: operand wait  ', wait[:k].tolist())
    nt = int((tma[:, 1] > 0).sum())
    if nt > 20:
        tma = tma[:nt]
        w_t = tma[:, 1] - tma[:, 0]
        print('TMA producer: %d rows; slot wait per row: median %d mean %.0f; cycles between issues median %d' % (
            nt, np.median(w_t), w_t.mean(), np.median(np.diff(tma[:, 1]))))
    ni = int((itp[:, 2] > 0).sum())
    if ni > 20:
        itp = itp[:ni]
        fill = itp[:, 2] - itp[:, 0]
        print('interpolation warp 0: %d rows; row start to arrive: median %d mean %.0f; of which slot wait: median %d mean %.0f; '
              'cycles between arrives median %d' % (ni, np.median(fill), fill.mean(), np.median(itp[:, 1]), itp[:, 1].mean(),
                                                   np.median(np.diff(itp[:, 2]))))


if __name__ == '__main__':
    main()
