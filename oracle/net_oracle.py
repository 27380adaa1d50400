"""CPU fp32 oracle for ``CascadedNet.forward`` / ``predict_mask``.  TEST INFRASTRUCTURE.

A functional restatement (plain ``torch.nn.functional`` calls on CPU float32, driven by the
checkpoint's ``state_dict`` keys) of the reference model:

* Conv2DBNActiv  lib/layers.py:8-26    conv(bias=False) -> BatchNorm2d(eval) -> ReLU | LeakyReLU(0.01)
* Encoder        lib/layers.py:29-40   conv(stride 2) -> conv(stride 1), LeakyReLU
* Decoder        lib/layers.py:43-64   bilinear x2 (align_corners=True) -> crop_center -> cat -> conv, ReLU
* ASPPModule     lib/layers.py:67-105  freq-mean-pool branch + 1x1 + 3 dilated 3x3 -> cat -> 1x1 bottleneck
* LSTMModule     lib/layers.py:108-133 1x1 conv -> BiLSTM over time -> Linear + BatchNorm1d + ReLU
* BaseNet        lib/nets.py:8-41
* CascadedNet    lib/nets.py:44-141    (real-mask branch only; ``is_complex`` is never enabled by a caller)

The oracle is pinned in tests/test_oracle_net.py against golden tensors produced by the
UNMODIFIED reference modules (oracle/make_golden.py, run in the build container where
a reference checkout is given) and, when the reference is importable, against it directly.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5  # nn.BatchNorm2d / BatchNorm1d default


def _t(sd, key):
    v = sd[key]
    if not torch.is_tensor(v):
        v = torch.from_numpy(v)
    return v


def to_device(sd, device):
    """Copy of the state_dict on ``device`` (float tensors only are moved; used by the cuDNN baseline leg of bench.py,
    which runs this same functional restatement on cuda:0 with PyTorch's default TF32 convolutions)."""
    return {k: (v if not torch.is_tensor(v) else v.to(device)) for k, v in
            ((k, _t(sd, k)) for k in sd)}


def conv_bn_act(sd, p, x, stride=1, pad=1, dil=1, act='relu'):
    """lib/layers.py:8-26 at state_dict prefix ``p``."""
    w = _t(sd, p + '.conv.0.weight')
    h = F.conv2d(x, w, None, stride=stride, padding=pad, dilation=dil)
    h = F.batch_norm(h, _t(sd, p + '.conv.1.running_mean'), _t(sd, p + '.conv.1.running_var'),
                     _t(sd, p + '.conv.1.weight'), _t(sd, p + '.conv.1.bias'), False, 0.0, BN_EPS)
    if act == 'relu':
        return F.relu(h)
    if act == 'leaky':
        return F.leaky_relu(h, 0.01)
    raise ValueError(act)


def encoder(sd, p, x, conv=conv_bn_act):
    """lib/layers.py:29-40 (ksize 3, stride 2, pad 1, LeakyReLU)."""
    h = conv(sd, p + '.conv1', x, stride=2, pad=1, act='leaky')
    return conv(sd, p + '.conv2', h, stride=1, pad=1, act='leaky')


def crop_center(h1, h2):
    """lib/spec_utils.py:8-23: crop ``h1`` on the time axis to ``h2``'s width."""
    if h1.shape[3] == h2.shape[3]:
        return h1
    if h1.shape[3] < h2.shape[3]:
        raise ValueError('h1_shape[3] must be greater than h2_shape[3]')
    s = (h1.shape[3] - h2.shape[3]) // 2
    return h1[:, :, :, s:s + h2.shape[3]]


def decoder(sd, p, x, skip, conv=conv_bn_act):
    """lib/layers.py:51-64."""
    x = F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=True)
    skip = crop_center(skip, x)
    x = torch.cat([x, skip], dim=1)
    return conv(sd, p + '.conv1', x, stride=1, pad=1, act='relu')


def aspp(sd, p, x, dilations=((4, 2), (8, 4), (12, 6)), conv=conv_bn_act):
    """lib/layers.py:92-105 (dropout is identity in eval)."""
    _, _, h, w = x.shape
    pooled = x.mean(dim=2, keepdim=True)  # AdaptiveAvgPool2d((1, None))
    f1 = conv(sd, p + '.conv1.1', pooled, pad=0)
    f1 = F.interpolate(f1, size=(h, w), mode='bilinear', align_corners=True)
    f2 = conv(sd, p + '.conv2', x, pad=0)
    feats = [f1, f2]
    for i, d in zip((3, 4, 5), dilations):
        feats.append(conv(sd, f'{p}.conv{i}', x, pad=d, dil=d))
    return conv(sd, p + '.bottleneck', torch.cat(feats, dim=1), pad=0)


def lstm_dense(sd, p, h):
    """lib/layers.py:119-122,131: Linear + BatchNorm1d + ReLU of the BiLSTM output h (M, 2*hid) -> (M, nbins)."""
    h = F.linear(h, _t(sd, p + '.dense.0.weight'), _t(sd, p + '.dense.0.bias'))
    h = F.batch_norm(h, _t(sd, p + '.dense.1.running_mean'), _t(sd, p + '.dense.1.running_var'),
                     _t(sd, p + '.dense.1.weight'), _t(sd, p + '.dense.1.bias'), False, 0.0, BN_EPS)
    return F.relu(h)


def lstm_module(sd, p, x, conv=conv_bn_act):
    """lib/layers.py:124-133: returns (N, 1, nbins, nframes)."""
    N, _, nbins, nframes = x.shape
    h = conv(sd, p + '.conv', x, pad=0)[:, 0]                 # N, nbins, nframes
    h = h.permute(2, 0, 1).contiguous()                       # nframes, N, nbins
    hid = _t(sd, p + '.lstm.weight_hh_l0').shape[1]
    if x.is_cuda:
        # the reference module is nn.LSTM (cuDNN on a GPU): same fused call, not a Python time loop
        flat = [_t(sd, f'{p}.lstm.{n}_l0{sfx}') for sfx in ('', '_reverse')
                for n in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')]
        zeros = torch.zeros(2, N, hid, device=x.device, dtype=x.dtype)
        out, _, _ = torch._VF.lstm(h, (zeros, zeros), flat, True, 1, 0.0, False, True, False)
        h2 = lstm_dense(sd, p, out.reshape(nframes * N, 2 * hid))
        return h2.reshape(nframes, N, 1, nbins).permute(1, 2, 3, 0)
    outs = []
    for sfx, rev in (('', False), ('_reverse', True)):
        w_ih = _t(sd, f'{p}.lstm.weight_ih_l0{sfx}')
        w_hh = _t(sd, f'{p}.lstm.weight_hh_l0{sfx}')
        b = _t(sd, f'{p}.lstm.bias_ih_l0{sfx}') + _t(sd, f'{p}.lstm.bias_hh_l0{sfx}')
        xp = h @ w_ih.t() + b                                  # nframes, N, 4*hid
        hs = torch.zeros(N, hid)
        cs = torch.zeros(N, hid)
        out = torch.empty(nframes, N, hid)
        steps = range(nframes - 1, -1, -1) if rev else range(nframes)
        for t in steps:
            g = xp[t] + hs @ w_hh.t()
            i, f, gg, o = g.split(hid, dim=1)                  # torch gate order i, f, g, o
            cs = torch.sigmoid(f) * cs + torch.sigmoid(i) * torch.tanh(gg)
            hs = torch.sigmoid(o) * torch.tanh(cs)
            out[t] = hs
        outs.append(out)
    h = lstm_dense(sd, p, torch.cat(outs, dim=2).reshape(nframes * N, 2 * hid))
    return h.reshape(nframes, N, 1, nbins).permute(1, 2, 3, 0)


def basenet(sd, p, x, conv=conv_bn_act):
    """lib/nets.py:26-41."""
    e1 = conv(sd, p + '.enc1', x)
    e2 = encoder(sd, p + '.enc2', e1, conv)
    e3 = encoder(sd, p + '.enc3', e2, conv)
    e4 = encoder(sd, p + '.enc4', e3, conv)
    e5 = encoder(sd, p + '.enc5', e4, conv)
    h = aspp(sd, p + '.aspp', e5, conv=conv)
    h = decoder(sd, p + '.dec4', h, e4, conv)
    h = decoder(sd, p + '.dec3', h, e3, conv)
    h = decoder(sd, p + '.dec2', h, e2, conv)
    h = torch.cat([h, lstm_module(sd, p + '.lstm_dec2', h, conv)], dim=1)
    return decoder(sd, p + '.dec1', h, e1, conv)


def forward(sd, x, n_fft=2048, return_stages=False, conv=conv_bn_act):
    """lib/nets.py:82-117 (real mask).  x: float32 (N, 2, n_fft//2+1, W) -> mask same shape.  ``conv`` runs every
    Conv2DBNActiv, with conv_bn_act's signature (oracle/precision_oracle.py emulates the product's arithmetic)."""
    with torch.no_grad():
        if not torch.is_tensor(x):
            x = torch.from_numpy(x)
        max_bin = n_fft // 2
        output_bin = n_fft // 2 + 1
        x = x[:, :, :max_bin]
        bandw = x.shape[2] // 2
        l1_in, h1_in = x[:, :, :bandw], x[:, :, bandw:]
        l1 = conv(sd, 'stg1_low_band_net.1', basenet(sd, 'stg1_low_band_net.0', l1_in, conv), pad=0)
        h1 = basenet(sd, 'stg1_high_band_net', h1_in, conv)
        aux1 = torch.cat([l1, h1], dim=2)
        l2 = conv(sd, 'stg2_low_band_net.1',
                  basenet(sd, 'stg2_low_band_net.0', torch.cat([l1_in, l1], dim=1), conv), pad=0)
        h2 = basenet(sd, 'stg2_high_band_net', torch.cat([h1_in, h1], dim=1), conv)
        aux2 = torch.cat([l2, h2], dim=2)
        f3 = basenet(sd, 'stg3_full_band_net', torch.cat([x, aux1, aux2], dim=1), conv)
        logit = F.conv2d(f3, _t(sd, 'out.weight'))
        mask = torch.sigmoid(logit)
        mask = F.pad(mask, (0, 0, 0, output_bin - mask.shape[2]), mode='replicate')
        if return_stages:
            return mask, dict(l1=l1, h1=h1, l2=l2, h2=h2, f3=f3, logit=logit)
        return mask


def predict_mask(sd, x, n_fft=2048, offset=64):
    """lib/nets.py:124-131."""
    mask = forward(sd, x, n_fft)
    if offset > 0:
        mask = mask[:, :, :, offset:-offset]
        assert mask.shape[3] > 0
    return mask
