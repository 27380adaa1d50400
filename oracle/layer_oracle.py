"""Per-layer references and gates for the tensors one forward writes.  TEST INFRASTRUCTURE.

Each check applies ONE op of the oracle (``net_oracle``'s functions, on a float64 copy of the state dict) to the
inputs the GPU itself gave that op, and compares the result with what the GPU wrote.  Errors then do not accumulate
through the net, so the gate can be set from the arithmetic of the one kernel: tight enough to see a convolution lose
one of its two correction products (DESIGN §3), which the end-to-end mask gate cannot.

Convolution gate.  r = max |y - ref| / (B + 2^-4 |ref|), B = sqrt(conv(x^2, w'^2)) with the BatchNorm-folded weights
w': B is the size of the error per-product rounding can cause, the |ref| term covers the split-bf16 rounding of the
stored output.  The three-product scheme must give r <= CONV_GATE; the same metric of the two-product emulations
(``no_wlo``: x * w'_hi, ``no_xlo``: x_hi * w', products exact in float64) must be >= NONVACUOUS * CONV_GATE, which
proves layer by layer that the gate would see the loss of either product.

fp32 ops.  r = max |y - ref| / mag, mag = the op applied to |inputs| (the bound of its rounding errors), against a
gate set from the fp32 arithmetic of the kernel.  The upsamples and the recurrence also have a named wrong variant
(bilinear with align_corners=False, the reverse direction run forwards in time) that the gate must reject by
NONVACUOUS.
"""
import torch
import torch.nn.functional as F

from oracle import net_oracle
from oracle.precision_oracle import activation, bf16, fold_bn, folded_conv

CONV_GATE = 2.0 ** -12
NONVACUOUS = 8.0
# bilinear x2 with the kernel's (ATen's) fp32 weights: two fp32 lerps, then a split-bf16 store (2^-18)
UPSAMPLE_GATE = 2.0 ** -14
# sums of at most a few hundred fp32 terms (pool over rows, the 1x1 input convolution, the two LSTM GEMMs), then at
# worst a split-bf16 store (2^-18)
FP32_SUM_GATE = 2.0 ** -14
LSTM_H_GATE = 1e-5            # absolute, h in (-1, 1): fp32 gates with accurate expf / tanhf over T steps
PACK_GATE = 2.0 ** -16        # |X| / norm: hypotf, a reciprocal and a product in fp32, stored split-bf16 (2^-18)


def nonvacuous_factor_fan_in(fan_in):
    """How far above CONV_GATE both two-product emulations of a convolution summing ``fan_in`` products per output
    (Cin * kh * kw) must land.  A dropped correction product errs by at most 2^-9 = 8 * CONV_GATE per product, so a
    layer summing fewer than 16 products per output (the 1x1 bridge over 8 channels of the nout = 16 net: 6.9x on the
    CPU emulation) can only be held to 4x."""
    return NONVACUOUS if fan_in >= 16 else NONVACUOUS / 2


def nonvacuous_factor(sd, p):
    """nonvacuous_factor_fan_in of Conv2DBNActiv ``p``"""
    return nonvacuous_factor_fan_in(net_oracle._t(sd, p + '.conv.0.weight')[0].numel())


def state_dict64(sd, device):
    """float64 copy of the state dict on ``device`` (integer entries kept as they are)."""
    out = {}
    for k, v in sd.items():
        t = v if torch.is_tensor(v) else torch.from_numpy(v)
        out[k] = t.to(device=device, dtype=torch.float64) if t.is_floating_point() else t.to(device)
    return out


def max_ratio(err, den):
    """max of |err| / den, where 0 / 0 counts as 0"""
    num = err.abs()
    r = torch.where(num == 0, torch.zeros_like(num), num / den)
    return float(r.max()) if r.numel() else 0.0


def conv_ratios_of(x, w, b, y, stride=1, pad=1, dil=1, act='relu', ref=None):
    """The convolution gate of act(conv2d(x, w) + b) on the GPU's input x against its output y (x, w, b, y float64,
    NCHW; y may be None; act 'relu', 'leaky' or None for none): (r of y, r of the no_wlo emulation, r of the no_xlo
    emulation, ref, den) with den the metric's denominator.  ref: the float64 reference when the caller has it."""
    def act_of(v):
        return v if act is None else activation(v, act)

    kw = dict(stride=stride, padding=pad, dilation=dil)
    if ref is None:
        ref = act_of(F.conv2d(x, w, b, **kw))
    den = F.conv2d(x * x, w * w, None, **kw).sqrt() + 2.0 ** -4 * ref.abs()
    no_wlo = act_of(F.conv2d(x, bf16(w), b, **kw))
    no_xlo = act_of(F.conv2d(bf16(x), w, b, **kw))
    r = None if y is None else max_ratio(y - ref, den)
    return r, max_ratio(no_wlo - ref, den), max_ratio(no_xlo - ref, den), ref, den


def conv_ratios(sd, p, x, y, stride=1, pad=1, dil=1, act='relu'):
    """Conv2DBNActiv ``p`` on the GPU's input x against its output y (both float64, NCHW; y may be None):
    conv_ratios_of with the BatchNorm-folded weights, against the unfolded layer of the oracle."""
    ref = net_oracle.conv_bn_act(sd, p, x, stride=stride, pad=pad, dil=dil, act=act)
    w, b = folded_conv(sd, p)
    return conv_ratios_of(x, w, b, y, stride=stride, pad=pad, dil=dil, act=act, ref=ref)


def mask_ratio(m, z, ez):
    """The network's mask m = sigmoid(z) against the float64 logits z, where 1e-6 < sigmoid(z) < 1 - 1e-6: the error
    in logit units, |dm| / sigmoid'(z), over ez, the bound of the logit error, with the fp32 rounding of m itself
    (2^-20 of m) allowed on top.  The gate is 1."""
    ref = torch.sigmoid(z)
    keep = (ref > 1e-6) & (ref < 1 - 1e-6)
    den = ref * (1 - ref) * ez + 2.0 ** -20 * ref
    return max_ratio((m - ref)[keep], den[keep])


def _source_index(n_in, n_out, device):
    """ATen's align_corners=True source index of upsample_bilinear2d for float input: scale = (in-1)/(out-1) and
    src = scale * dst in fp32, so the interpolation weights carry an error of up to 2^-24 * in (enough to move a
    result near an input row by 2^-9 of the local magnitude at 512 rows).  Returns i0, i1 and the fp32 weights of
    each, as float64."""
    s = torch.tensor((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0, dtype=torch.float32, device=device)
    f = s * torch.arange(n_out, dtype=torch.float32, device=device)
    i0 = f.long()
    i1 = torch.clamp(i0 + 1, max=n_in - 1)
    lam = f - i0.float()
    return i0, i1, (1 - lam).double(), lam.double()


def up2x(x, align_corners=True):
    """lib/layers.py:52, F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=True) on float input, in
    float64 arithmetic with the fp32 weights of ATen's kernel (align_corners=False: F.interpolate itself, the wrong
    variant the upsample gate must reject)"""
    if not align_corners:
        return F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False)
    h0, h1, hy, ly = _source_index(x.shape[2], 2 * x.shape[2], x.device)
    w0, w1, hx, lx = _source_index(x.shape[3], 2 * x.shape[3], x.device)
    r0, r1 = x[:, :, h0], x[:, :, h1]
    top = hx * r0[..., w0] + lx * r0[..., w1]
    bot = hx * r1[..., w0] + lx * r1[..., w1]
    return hy[:, None] * top + ly[:, None] * bot


def upsample_ratios(low, y):
    """bilinear x2 of the GPU's low against its output y: (r, r of the align_corners=False variant)."""
    mag = up2x(low.abs())
    return max_ratio(y - up2x(low), mag), max_ratio(up2x(low, False) - up2x(low), mag)


def _lstm(xp, w_hh, bidirectional):
    """the fused nn.LSTM call of net_oracle.lstm_module, driven by the gate pre-activations xp (T, N, dirs * 4 hid)
    through identity input weights: xp already holds x . W_ih^T + b_ih + b_hh"""
    T, N, G = xp.shape
    four = w_hh[0].shape[0]
    hid = four // 4
    flat = []
    for d, whh in enumerate(w_hh):
        sel = torch.zeros(four, G, dtype=xp.dtype, device=xp.device)
        sel[:, d * four:(d + 1) * four] = torch.eye(four, dtype=xp.dtype, device=xp.device)
        z = torch.zeros(four, dtype=xp.dtype, device=xp.device)
        flat += [sel, whh, z, z]
    h0 = torch.zeros(len(w_hh), N, hid, dtype=xp.dtype, device=xp.device)
    with torch.backends.cudnn.flags(enabled=False):   # ATen's own float64 recurrence on any device
        out, _, _ = torch._VF.lstm(xp, (h0, h0), flat, True, 1, 0.0, False, bidirectional, False)
    return out


def bilstm(sd, p, xp):
    """the BiLSTM of LSTMModule ``p`` from the GPU's gate pre-activations xp (n, T, 8 hid) -> hs (n, T, 2 hid)"""
    w = [net_oracle._t(sd, f'{p}.lstm.weight_hh_l0{s}').to(xp.dtype) for s in ('', '_reverse')]
    return _lstm(xp.permute(1, 0, 2).contiguous(), w, True).permute(1, 0, 2)


def reverse_run_forwards(sd, p, xp):
    """wrong variant: the reverse direction's gates and weights stepped forwards in time -> (n, T, hid)"""
    four = xp.shape[2] // 2
    w = net_oracle._t(sd, f'{p}.lstm.weight_hh_l0_reverse').to(xp.dtype)
    return _lstm(xp[:, :, four:].permute(1, 0, 2).contiguous(), [w], False).permute(1, 0, 2)


def lstm_ratios(sd, p, h, l0, xp, hs, y):
    """The LSTM branch of BaseNet ``p`` (its state_dict prefix), each plane from the GPU's previous one (float64):
    h (n, 2n, bins, T) dec2's output, l0 / y (n, bins, T), xp (n, T, 8 hid), hs (n, T, 2 hid).
    Returns {plane: r} plus 'hs_reverse_forwards', the r of the wrong recurrence."""
    q = p + '.lstm_dec2'
    scale, shift = fold_bn(sd, q + '.conv.conv.1')
    w = net_oracle._t(sd, q + '.conv.conv.0.weight').double()[0, :, 0, 0] * scale[0]
    r = {'l0': max_ratio(l0 - torch.einsum('nchw,c->nhw', h, w), torch.einsum('nchw,c->nhw', h.abs(), w.abs()))}
    a = F.relu(l0 + shift[0]).permute(0, 2, 1)                       # (n, T, bins)
    wih = torch.cat([net_oracle._t(sd, f'{q}.lstm.weight_ih_l0{s}').double() for s in ('', '_reverse')])
    b = torch.cat([(net_oracle._t(sd, f'{q}.lstm.bias_ih_l0{s}') + net_oracle._t(sd, f'{q}.lstm.bias_hh_l0{s}'))
                   .double() for s in ('', '_reverse')])
    r['xp'] = max_ratio(xp - (a @ wih.t() + b), a @ wih.abs().t() + b.abs())
    ref_hs = bilstm(sd, q, xp)
    r['hs'] = max_ratio(hs - ref_hs, torch.ones_like(hs))
    hid = hs.shape[2] // 2
    r['hs_reverse_forwards'] = max_ratio(reverse_run_forwards(sd, q, xp) - ref_hs[:, :, hid:],
                                         torch.ones_like(ref_hs[:, :, hid:]))
    n, T, K = hs.shape
    ref_y = net_oracle.lstm_dense(sd, q, hs.reshape(n * T, K)).reshape(n, T, -1).permute(0, 2, 1)
    dscale, dshift = fold_bn(sd, q + '.dense.1', net_oracle._t(sd, q + '.dense.0.bias'))
    wd = net_oracle._t(sd, q + '.dense.0.weight').double()
    mag = (dscale.abs()[None, :, None] * (wd.abs() @ hs.abs().reshape(n * T, K).t()).reshape(-1, n, T).permute(1, 0, 2)
           + dshift.abs()[None, :, None])
    r['y'] = max_ratio(y - ref_y, mag)
    return r
