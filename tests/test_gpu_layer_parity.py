"""Per-layer parity of the forward pass (run on an H100).

After one synchronised forward, every tensor the forward wrote is read back through vr_debug_tensor and compared with
its op applied in float64 to the GPU's own inputs of that op (oracle/layer_oracle.py).  Errors do not accumulate
through the net, so each gate is set from one kernel's arithmetic, and a failure names the layer.  The convolution gate
sees a single layer losing one of its two correction products, which the 1e-3 mask gate of test_gpu_parity.py cannot
(DESIGN §3); every convolution also proves that on its own inputs (the two-product emulations must fail the gate).

Besides the values, the wiring: the channel slices of the stage-input buffer in3 each stage reads, the permuted dec1
reduction order, the zero pad channels (VR_KSKIP relies on them), and the two-stream schedule (a consumer that ran
before its producer finished fails against the producer's final output).
"""
import ctypes
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import record_parity
from oracle import layer_oracle as lo
from oracle import net_oracle

pytestmark = pytest.mark.gpu

DEFAULT = (2048, 1024, 32, 128)
# name: (n_fft, hop, nout, nout_lstm), conv_mode, cropsize, max_batch, images checked
CONFIGS = {
    'A': (DEFAULT, 0, 256, 2, (0, 1)),               # the benchmark's net: row, halo, generic kernels; fusions
    'B': (DEFAULT, 1, 256, 2, (0, 1)),               # the CUDA-core kernel at every layer shape of the net
    'C': (DEFAULT, 0, 256, 27, (0, 13, 26)),         # the benchmark's batch
    'D512': (DEFAULT, 0, 512, 1, (0,)),              # user cropsizes; LSTM T = 256 / 512
    'D1024': (DEFAULT, 0, 1024, 1, (0,)),
    'E': ((512, 256, 16, 32), 0, 192, 2, (0, 1)),    # generic kernel, staged decoders, LSTM HID 16 / 8
    'F': ((2048, 1024, 64, 128), 0, 256, 2, (0, 1)),  # dec1 with two N tiles: mask_out_kernel runs
    'G1024': ((1024, 256, 32, 128), 0, 256, 2, (0, 1)),    # band height 256
    'G4096': ((4096, 1024, 32, 128), 0, 256, 2, (0, 1)),   # band height 1024
    'H144': (DEFAULT, 0, 144, 2, (0, 1)),   # the smallest cropsize: maps 144/72/36/18/9 wide tile for no wgmma kernel
    'H320': (DEFAULT, 0, 320, 2, (0, 1)),   # maps 320/160/80/40/20 wide: no tiling either, no crop-mask fusion
}
OFFSET = 64
DILATIONS = ((4, 2), (8, 4), (12, 6))   # lib/nets.py:10
FAMILY_MAX = {}                          # kernel family -> (largest ratio to its gate, tensor)


def _round_up(a, b):
    return (a + b - 1) // b * b


def _on_tensor_cores(w, H, W, stride):
    """whether the layer of weights w (Cout, Cin, k, k), stride `stride` and H x W output maps runs on a tensor-core
    kernel.  Mirrors every TC_NONE exit of tc_choose (conv_tc.cu), which must be kept in step with it: a kernel size
    other than 1 or 3, a stride other than 1 or 2, fewer than 4 output channels, maps that tile_geom does not split
    into 128-pixel tiles, a tile taller or wider than 256 input pixels, and more output-channel tiles than the 256
    bias floats every tensor-core kernel stages.  Any other layer runs on the CUDA-core kernel."""
    cout, k = w.shape[0], w.shape[-1]
    if k not in (1, 3) or stride not in (1, 2) or cout < 4:
        return False
    # tile_geom
    if W >= 128:
        if W % 128:
            return False
        Wt, Ht = 128, 1
    else:
        if 128 % W:
            return False
        Wt, Ht = W, min(128 // W, H)
        if H % Ht or (128 // W) % Ht:
            return False
    if Wt * stride > 256 or Ht * stride > 256:
        return False
    # n_tiling of the generic and halo kernels (the row kernel's tiles fit exactly when these do)
    cout16 = _round_up(cout, 16)
    n_tiles = -(-cout16 // 128)
    return n_tiles * _round_up(-(-cout16 // n_tiles), 16) <= 256


class Checks:
    """Collects every ratio of one configuration; the test fails at the end with all the tensors out of their gates."""

    def __init__(self, tag, sd, conv_mode):
        self.tag, self.sd, self.conv_mode = tag, sd, conv_mode
        self.failed = []

    def ratio(self, name, r, gate, family):
        record_parity('layer_%s_%s' % (self.tag, name), r, gate)
        if r / gate > FAMILY_MAX.get(family, (-1.0, ''))[0]:
            FAMILY_MAX[family] = (r / gate, '%s %s' % (self.tag, name))
        if not r <= gate:
            self.failed.append('%s: %.4g > gate %.4g' % (name, r, gate))

    def rejects(self, name, r_wrong, need):
        """a wrong variant of the op must land at least `need` from its reference, in the gate's metric"""
        if not r_wrong >= need:
            self.failed.append('%s: wrong variant only %.4g (needs >= %.4g)' % (name, r_wrong, need))

    def exact(self, name, ok):
        if not ok:
            self.failed.append('%s: not exact' % name)

    def family(self, w, y, stride, dil):
        if self.conv_mode == 1 or not _on_tensor_cores(w, y.shape[-2], y.shape[-1], stride):
            return 'cuda-core'
        k, W = w.shape[-1], y.shape[-1]
        if k == 3 and stride == 1 and dil == 1:
            if W % 128 == 0:
                return 'row'
            if W in (16, 32, 64):
                return 'halo'
        return 'generic'

    def conv(self, p, x, y, stride=1, pad=1, dil=1, act='relu'):
        r, r_wlo, r_xlo, ref, den = lo.conv_ratios(self.sd, p, x, y, stride=stride, pad=pad, dil=dil, act=act)
        need = lo.nonvacuous_factor(self.sd, p) * lo.CONV_GATE
        self.rejects(p + ' no_wlo', r_wlo, need)
        self.rejects(p + ' no_xlo', r_xlo, need)
        if y is not None:
            w = net_oracle._t(self.sd, p + '.conv.0.weight')
            self.ratio(p, r, lo.CONV_GATE, self.family(w, y, stride, dil if isinstance(dil, int) else 2))
        return ref, den

    def up(self, name, low, y):
        r, r_wrong = lo.upsample_ratios(low, y)
        self.ratio(name, r, lo.UPSAMPLE_GATE, 'upsample')
        self.rejects(name + ' align_corners=False', r_wrong, lo.NONVACUOUS * lo.UPSAMPLE_GATE)


def _reader(ctx, images):
    """name -> float64 tensor of the checked images, as the last forward left it"""
    from lib import _native
    cache = {}

    def read(name):
        if name not in cache:
            parts = []
            for i in images:
                shape = (ctypes.c_int64 * 4)()
                ctx.check(ctx.lib.vr_debug_tensor(ctx.handle, name.encode(), i, 1, None, shape, _native.stream_ptr()),
                          'vr_debug_tensor(%s)' % name)
                out = torch.empty(tuple(shape), dtype=torch.float32, device='cuda')
                ctx.check(ctx.lib.vr_debug_tensor(ctx.handle, name.encode(), i, 1, _native.ptr(out), shape,
                                                  _native.stream_ptr()), 'vr_debug_tensor(%s)' % name)
                parts.append(out[..., 0] if '.lstm.' in name else out)
            cache[name] = torch.cat(parts).double()
        return cache[name]

    return read


def _dec1_inputs(read, p):
    """dec1's reduction channels in the reference's order [up(h) 2n | up(lstm) 1 | e1 n] (lib/nets.py:38-39) and the
    layout facts of the plan, from the buffers' shapes (DESIGN §4)"""
    cat1, t2, d2 = read(p + '.cat1'), read(p + '.t2'), read(p + '.d2')
    n = t2.shape[1] // 2
    Up = _round_up(2 * n, 32)
    Lp = _round_up(Up + n, 16)
    C1 = cat1.shape[1]
    assert C1 in (Lp + 16, Lp + 16 - Up, Lp - Up), (p, C1)
    staged = C1 == Lp + 16
    own = C1 == Lp - Up
    first = 0 if staged else Up       # the first of dec1's reduction channels cat1 holds
    h = d2[:, :2 * n]
    grp = read(p + '.lstm_up') if own else cat1[:, Lp - first:Lp - first + 16]
    e1 = cat1[:, Up - first:Up - first + n]
    up_h = cat1[:, :2 * n] if staged else lo.up2x(h)
    return dict(n=n, Up=Up, Lp=Lp, staged=staged, own=own, first=first, cat1=cat1, d2=d2, h=h, grp=grp, e1=e1,
                x=torch.cat([up_h, grp[:, :1], e1], dim=1))


def _basenet(chk, read, ctx, p, x, y1):
    """every tensor of BaseNet p (lib/nets.py:26-41) on the GPU's input x; y1: where dec1 wrote, or None.
    Returns dec1's inputs and its reference output and metric denominator."""
    sd = chk.sd
    D = _dec1_inputs(read, p)
    n, Up, Lp, first, cat1 = D['n'], D['Up'], D['Lp'], D['first'], D['cat1']
    t2, t3, t4, t5, e5 = (read(p + '.' + b) for b in ('t2', 't3', 't4', 't5', 'e5'))
    cat2, cat3, cat4 = read(p + '.cat2'), read(p + '.cat3'), read(p + '.cat4')
    fused2 = cat2.shape[1] == 2 * n
    e1, e2, e3, e4 = D['e1'], cat2[:, (0 if fused2 else 4 * n):][:, :2 * n], cat3[:, 6 * n:], cat4[:, 8 * n:]
    # encoders (lib/nets.py:27-31)
    chk.conv(p + '.enc1', x, e1)
    for i, (a, t, b) in enumerate(((e1, t2, e2), (e2, t3, e3), (e3, t4, e4), (e4, t5, e5))):
        chk.conv('%s.enc%d.conv1' % (p, i + 2), a, t, stride=2, act='leaky')
        chk.conv('%s.enc%d.conv2' % (p, i + 2), t, b, act='leaky')
    # ASPP (lib/layers.py:92-105): pool_freq_mean, the 1x1 branch, broadcast_rows, the other branches, bottleneck
    pool, f1, acat, ao = (read(p + '.' + b) for b in ('pool', 'f1', 'acat', 'ao'))
    chk.ratio(p + '.pool', lo.max_ratio(pool - e5.mean(dim=2, keepdim=True), e5.abs().mean(dim=2, keepdim=True)),
              lo.FP32_SUM_GATE, 'aspp')
    chk.conv(p + '.aspp.conv1.1', pool, f1, pad=0)
    chk.exact(p + '.acat[0:8n] = broadcast f1', torch.equal(acat[:, :8 * n], f1.expand(-1, -1, e5.shape[2], -1)))
    chk.conv(p + '.aspp.conv2', e5, acat[:, 8 * n:16 * n], pad=0)
    for i, d in enumerate(DILATIONS):
        chk.conv('%s.aspp.conv%d' % (p, i + 3), e5, acat[:, (16 + 8 * i) * n:(24 + 8 * i) * n], pad=d, dil=d)
    chk.conv(p + '.aspp.bottleneck', acat, ao, pad=0)
    # decoders (lib/nets.py:35-37)
    d4, d3, d2, h = read(p + '.d4'), read(p + '.d3'), D['d2'], D['h']
    chk.up(p + '.cat4[0:8n]', ao, cat4[:, :8 * n])
    chk.conv(p + '.dec4.conv1', cat4, d4)
    chk.up(p + '.cat3[0:6n]', d4, cat3[:, :6 * n])
    chk.conv(p + '.dec3.conv1', cat3, d3)
    if fused2:
        in2 = torch.cat([lo.up2x(d3), e2], dim=1)
    else:
        chk.up(p + '.cat2[0:4n]', d3, cat2[:, :4 * n])
        in2 = cat2
    chk.conv(p + '.dec2.conv1', in2, h)
    chk.exact(p + '.d2[2n:Up] zero', bool((d2[:, 2 * n:] == 0).all()))
    # LSTM branch (lib/layers.py:124-133), then its up-sampled group of dec1's input
    r = lo.lstm_ratios(sd, p, h, *(read('%s.lstm.%s' % (p, k)) for k in ('l0', 'xp', 'hs', 'y')))
    for k in ('l0', 'xp', 'y'):
        chk.ratio('%s.lstm.%s' % (p, k), r[k], lo.FP32_SUM_GATE, 'lstm')
    chk.ratio(p + '.lstm.hs', r['hs'], lo.LSTM_H_GATE, 'lstm')
    chk.rejects(p + '.lstm.hs reverse run forwards', r['hs_reverse_forwards'], lo.NONVACUOUS * lo.LSTM_H_GATE)
    grp = D['grp']
    chk.up(p + '.up(lstm)', read(p + '.lstm.y')[:, None], grp[:, :1])
    chk.exact(p + '.up(lstm) group channels 1.. zero', bool((grp[:, 1:] == 0).all()))
    if not D['own']:
        shape = (ctypes.c_int64 * 4)()
        chk.exact(p + '.lstm_up rejected', ctx.lib.vr_debug_tensor(ctx.handle, (p + '.lstm_up').encode(), 0, 1, None,
                                                                   shape, None) != 0)
    if D['staged']:
        chk.up(p + '.cat1[0:2n]', h, cat1[:, :2 * n])
        chk.exact(p + '.cat1 zero groups', bool((cat1[:, 2 * n:Up] == 0).all() and (cat1[:, Up + n:Lp] == 0).all()))
    else:
        chk.exact(p + '.cat1 zero groups', bool((cat1[:, n:Lp - first] == 0).all()))
    ref, den = chk.conv(p + '.dec1.conv1', D['x'], y1)
    return D, ref, den


def _mask_checks(chk, name, mask, f3, den, w_out, max_bin, crop):
    """mask (N, 2, bins, frames) = sigmoid(out . f3) over the frames [crop, W - crop), the Nyquist row replicated.
    den: None when f3 is what the GPU stored, else the dec1 metric's denominator of the reference f3."""
    z = F.conv2d(f3, w_out)
    ez = 2.0 ** -16 * F.conv2d(f3.abs(), w_out.abs())
    if den is not None:   # the logit error that dec1's gate allows on top
        ez = ez + lo.CONV_GATE * F.conv2d(den, w_out.abs())
    W = z.shape[3]
    r = lo.mask_ratio(mask[:, :, :max_bin], z[..., crop:W - crop], ez[..., crop:W - crop])
    chk.ratio(name, r, 1.0, 'mask')
    chk.exact(name + ' Nyquist row', torch.equal(mask[:, :, max_bin], mask[:, :, max_bin - 1]))


def _run(tag):
    from lib import _native, synth
    (n_fft, hop, nout, nout_lstm), conv_mode, crop, batch, images = CONFIGS[tag]
    t0 = time.time()
    dev = torch.device('cuda:0')
    ctx = _native.Context(0, n_fft, hop, nout, nout_lstm, crop, batch, conv_mode)
    try:
        sd = synth.make_state_dict(n_fft, nout, nout_lstm)
        ctx.load_state_dict(sd)
        sd64 = lo.state_dict64(synth.to_torch_state_dict(sd), dev)
        chk = Checks(tag, sd64, conv_mode)
        bins, max_bin = n_fft // 2 + 1, n_fft // 2
        g = torch.Generator(device='cuda').manual_seed(11)
        mag = torch.rand((batch, 2, bins, crop), dtype=torch.float32, device='cuda', generator=g)
        idx = torch.tensor(images, device='cuda')
        st = _native.stream_ptr()

        # pass 1: stage 3's dec1 over every frame into f3, then mask_out_kernel
        full = torch.empty_like(mag)
        assert ctx.lib.vr_debug_set(7, 0) == 0
        try:
            ctx.check(ctx.lib.vr_forward(ctx.handle, _native.ptr(mag), batch, _native.ptr(full), st), 'vr_forward')
        finally:
            ctx.lib.vr_debug_set(7, 1)
        torch.cuda.synchronize()
        read = _reader(ctx, images)
        Hb, a1, a2 = max_bin // 2, nout // 4, nout // 2
        pos_aux1, pos_x = a2, a2 + a1
        in3 = read('in3')
        x, aux1, aux2 = in3[:, pos_x:pos_x + 2], in3[:, pos_aux1:pos_aux1 + a1], in3[:, :a2]
        m = mag[idx, :, :max_bin]
        hi = m.to(torch.bfloat16).float()
        chk.exact('in3 x = split-bf16 of the input', torch.equal(x, (hi + (m - hi).to(torch.bfloat16).float()).double()))
        chk.exact('in3 pad channels zero', bool((in3[:, pos_x + 2:] == 0).all()))
        lo_, hi_ = slice(0, Hb), slice(Hb, 2 * Hb)
        o1, o2, f3 = read('o1'), read('o2'), read('f3')
        _basenet(chk, read, ctx, 'stg1_low_band_net.0', x[:, :, lo_], o1)
        _basenet(chk, read, ctx, 'stg1_high_band_net', x[:, :, hi_], aux1[:, :, hi_])
        chk.conv('stg1_low_band_net.1', o1, aux1[:, :, lo_], pad=0)
        x2 = torch.cat([x, aux1], dim=1)
        _basenet(chk, read, ctx, 'stg2_low_band_net.0', x2[:, :, lo_], o2)
        _basenet(chk, read, ctx, 'stg2_high_band_net', x2[:, :, hi_], aux2[:, :, hi_])
        chk.conv('stg2_low_band_net.1', o2, aux2[:, :, lo_], pad=0)
        D3, f3_ref, den3 = _basenet(chk, read, ctx, 'stg3_full_band_net', torch.cat([x, aux1, aux2], dim=1), f3)
        w_out = net_oracle._t(sd64, 'out.weight')
        _mask_checks(chk, 'mask (from f3)', full[idx].double(), f3, None, w_out, max_bin, 0)

        # pass 2: the default path (stage 3's dec1 writes the mask of the kept frames where its plan can); the mask is
        # checked from dec1's inputs, which must be the same as in pass 1
        crop_mask = torch.empty((batch, 2, bins, crop - 2 * OFFSET), dtype=torch.float32, device='cuda')
        ctx.check(ctx.lib.vr_predict_mask(ctx.handle, _native.ptr(mag), batch, _native.ptr(crop_mask), st),
                  'vr_predict_mask')
        torch.cuda.synchronize()
        D3b = _dec1_inputs(_reader(ctx, images), 'stg3_full_band_net')
        chk.exact('stg3 dec1 inputs repeat', torch.equal(D3b['x'], D3['x']))
        _mask_checks(chk, 'mask (from dec1 inputs, offset crop)', crop_mask[idx].double(), f3_ref, den3, w_out,
                     max_bin, OFFSET)
        torch.cuda.synchronize()
        print('layer parity %s: %.1f s' % (tag, time.time() - t0))
        return ctx, chk
    except BaseException:
        ctx.close()
        raise


@pytest.mark.parametrize('tag', list(CONFIGS))
def test_every_tensor_of_the_forward(tag):
    ctx, chk = _run(tag)
    try:
        if tag == 'A':
            _hook_rejects_bad_requests(ctx, chk)
        if tag == 'C':
            _pack_from_spec(ctx, chk)
    finally:
        ctx.close()
    for fam, (r, name) in sorted(FAMILY_MAX.items()):
        print('largest ratio to gate so far, %-9s %.3g  (%s)' % (fam, r, name))
    assert not chk.failed, '\n'.join(chk.failed)


def _hook_rejects_bad_requests(ctx, chk):
    shape = (ctypes.c_int64 * 4)()
    for name, n0, n in (('no_such_tensor', 0, 1), ('stg3_full_band_net.nope', 0, 1), ('in3', -1, 1), ('in3', 1, 2)):
        rc = ctx.lib.vr_debug_tensor(ctx.handle, name.encode(), n0, n, None, shape, None)
        chk.exact('vr_debug_tensor rejects %s [%d, %d)' % (name, n0, n0 + n), rc != 0 and ctx.lib.vr_last_error(ctx.handle))


def _pack_from_spec(ctx, chk):
    """pack_mag_from_spec: after vr_separate of a 300-frame track (three windows of 128 kept frames, one batch), the
    x channels of in3 hold |X window| / max|X|, zero outside the track, for the first and the last window"""
    from lib import _native
    T, r, bins, max_bin = 300, 128, 1025, 1024
    g = torch.Generator(device='cuda').manual_seed(12)
    spec = torch.randn((2, bins, T), dtype=torch.complex64, device='cuda', generator=g)
    mask = torch.empty((2, bins, T), dtype=torch.float32, device='cuda')
    ctx.check(ctx.lib.vr_separate(ctx.handle, _native.ptr(spec), T, 0, _native.ptr(mask), _native.stream_ptr()),
              'vr_separate')
    torch.cuda.synchronize()
    mag = spec.abs().double()
    mag = mag / mag.max()
    pos_x = 16 + 8
    for w in (0, 2):
        got = _reader(ctx, (w,))('in3')[0, pos_x:pos_x + 2]
        t = torch.arange(256, device='cuda') + w * r - OFFSET
        inside = (t >= 0) & (t < T)
        ref = torch.zeros_like(got)
        ref[:, :, inside] = mag[:, :max_bin, t[inside]]
        chk.exact('pack window %d zero frames' % w, bool((got[:, :, ~inside] == 0).all()))
        chk.ratio('pack_mag_from_spec window %d' % w, lo.max_ratio((got - ref)[:, :, inside], ref[:, :, inside]),
                  lo.PACK_GATE, 'pack')
