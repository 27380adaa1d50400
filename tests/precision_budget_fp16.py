"""fp16 instead of bf16 operand pairs (CPU emulation; not a pytest module; companion of precision_budget.py).

x = hi + lo with both parts rounded to IEEE half (11-bit significands) instead of bf16 (8-bit): mask error of the whole net
for the three-product scheme and for the cheaper ones.  Emulated: 3pass 9.9e-6
(bf16: 1.2e-4), two products 4.7e-3 / 6.0e-3, one product 8.3e-3 - with halves too every layer needs all three products
at the 1e-3 gate; the three-product error itself is 12x lower than with bf16 at the same tensor-core rate.
Usage: python tests/precision_budget_fp16.py"""
import os, sys, numpy as np, torch, torch.nn.functional as F
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import precision_budget as pb
from precision_budget import net_oracle, separator_oracle, stft_oracle, synth
def h16(x): return x.to(torch.float16).to(torch.float32)
def split16(x):
    hi = h16(x); return hi, h16(x - hi)
MODE = {'m': '3pass'}
def conv(sd, p, x, stride=1, pad=1, dil=1, act='relu'):
    w = net_oracle._t(sd, p + '.conv.0.weight').double()
    g, b = net_oracle._t(sd, p + '.conv.1.weight').double(), net_oracle._t(sd, p + '.conv.1.bias').double()
    m, v = net_oracle._t(sd, p + '.conv.1.running_mean').double(), net_oracle._t(sd, p + '.conv.1.running_var').double()
    scale = g / torch.sqrt(v + net_oracle.BN_EPS)
    wf = (w * scale[:, None, None, None]).float(); bias = (b - m * scale).float()
    xh, xl = split16(x); wh, wl = split16(wf)
    kw = dict(stride=stride, padding=pad, dilation=dil)
    md = MODE['m']
    if md == '3pass': y = F.conv2d(xh, wh, None, **kw) + F.conv2d(xl, wh, None, **kw) + F.conv2d(xh, wl, None, **kw)
    elif md == 'no_wlo': y = F.conv2d(xh, wh, None, **kw) + F.conv2d(xl, wh, None, **kw)
    elif md == 'no_xlo': y = F.conv2d(xh, wh, None, **kw) + F.conv2d(xh, wl, None, **kw)
    else: y = F.conv2d(xh, wh, None, **kw)
    y = y + bias[None, :, None, None]
    y = F.relu(y) if act == 'relu' else F.leaky_relu(y, 0.01)
    h, l = split16(y)
    return h + l
torch.set_num_threads(8)
sd = synth.to_torch_state_dict(synth.make_state_dict())
wave = synth.sine_mix(10.0)
X = stft_oracle.wave_to_spectrogram(wave, 1024, 2048)
pad_l, pad_r, roi = separator_oracle.make_padding(X.shape[2], 256, 64)
Xp = np.pad(X, ((0, 0), (0, 0), (pad_l, pad_r))); Xp /= np.abs(X).max()
x = torch.from_numpy(np.abs(Xp[None, :, :, 128:384]).astype(np.float32))
ref = net_oracle.forward(sd, x)
net_oracle.conv_bn_act = conv
for md in ('3pass', 'no_wlo', 'no_xlo', '1pass'):
    MODE['m'] = md
    print('fp16 all layers %s\t%.3e' % (md, (net_oracle.forward(sd, x) - ref).abs().max().item()), flush=True)
