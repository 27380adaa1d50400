"""A two-unit scheme that passes the gate (CPU emulation; not a pytest module; companion of precision_budget*.py).

Main product in IEEE half (x_hi16 * w_hi16, fp32 accumulate) and the two correction products with BOTH operands in fp8
(per-tensor power-of-two scale): x_lo * w_hi + x_hi * w_lo.  With a half hi part the lo part is 2^-12 of the value instead
of bf16's 2^-9, so the fp8 rounding of the corrections weighs 8x less than in precision_budget_fp8.py.  With wgmma the
half product runs at the bf16 rate and the two fp8 products at twice that rate: 1 + 1/2 + 1/2 = 2 units of tensor
time per product instead of 3, i.e. the roofline bound moves from 0.33 to 0.50, and an activation still costs 4 bytes
(half hi + fp8 lo + fp8 copy of hi).  Emulated, every layer at once: corrections in half 9.9e-6, in e4m3 2.7e-4
(gate 1e-3), in e5m2 5.5e-4, in block-scaled fp4 1.4e-3 - too coarse (and the H100 has no fp4 tensor-core path).
Usage: python tests/precision_budget_mixed.py"""
import os, sys, numpy as np, torch, torch.nn.functional as F
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import precision_budget as pb
from precision_budget import net_oracle, separator_oracle, stft_oracle, synth
def h16(x): return x.to(torch.float16).to(torch.float32)
def split16(x):
    hi = h16(x); return hi, x - hi          # lo kept exact here; it is rounded by the correction format below
def q(x, dt, top):
    m = x.abs().max().item()
    if m == 0.0: return x
    s = 2.0 ** np.floor(np.log2(top / m))
    return (x * s).to(dt).to(torch.float32) / s
GRID4 = torch.tensor([0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0])


def q4_blocks(x, dim=1, blk=32):
    """block-scaled fp4 (e2m1 magnitudes, one power-of-two scale per 32 channels: mxfp4-like) along the reduction dim"""
    x = x.movedim(dim, -1).contiguous()
    shp = x.shape
    c = shp[-1]
    pad = (-c) % blk
    xp = F.pad(x, (0, pad)).reshape(*shp[:-1], (c + pad) // blk, blk)
    m = xp.abs().amax(dim=-1, keepdim=True).clamp(min=1e-30)
    s = torch.exp2(torch.floor(torch.log2(6.0 / m)))
    a = (xp * s).abs().clamp(max=6.0).contiguous()
    y = torch.sign(xp) * GRID4[torch.bucketize(a, (GRID4[1:] + GRID4[:-1]) / 2)] / s
    return y.reshape(*shp[:-1], c + pad)[..., :c].movedim(-1, dim)


MODE = {'m': None}
TOP = {'t': 256.0}
def conv(sd, p, x, stride=1, pad=1, dil=1, act='relu'):
    w = net_oracle._t(sd, p + '.conv.0.weight').double()
    g, b = net_oracle._t(sd, p + '.conv.1.weight').double(), net_oracle._t(sd, p + '.conv.1.bias').double()
    m, v = net_oracle._t(sd, p + '.conv.1.running_mean').double(), net_oracle._t(sd, p + '.conv.1.running_var').double()
    scale = g / torch.sqrt(v + net_oracle.BN_EPS)
    wf = (w * scale[:, None, None, None]).float(); bias = (b - m * scale).float()
    xh, xl = split16(x); wh, wl = split16(wf)
    kw = dict(stride=stride, padding=pad, dilation=dil)
    md = MODE['m']
    if md == 'e4m3':
        f = lambda t: q(t, torch.float8_e4m3fn, TOP['t'])
    elif md == 'e5m2':
        f = lambda t: q(t, torch.float8_e5m2, 16384.0)
    elif md == 'mxfp4':
        f = q4_blocks
    else:
        f = h16
    y = F.conv2d(xh, wh, None, **kw) + F.conv2d(f(xl), f(wh), None, **kw) + F.conv2d(f(xh), f(wl), None, **kw)
    y = y + bias[None, :, None, None]
    y = F.relu(y) if act == 'relu' else F.leaky_relu(y, 0.01)
    hi = h16(y)
    return hi + h16(y - hi)                  # activations stored as a half pair
torch.set_num_threads(8)
sd = synth.to_torch_state_dict(synth.make_state_dict())
wave = synth.sine_mix(10.0)
X = stft_oracle.wave_to_spectrogram(wave, 1024, 2048)
pad_l, pad_r, roi = separator_oracle.make_padding(X.shape[2], 256, 64)
Xp = np.pad(X, ((0, 0), (0, 0), (pad_l, pad_r))); Xp /= np.abs(X).max()
wins = [torch.from_numpy(np.abs(Xp[None, :, :, i * roi:i * roi + 256]).astype(np.float32)) for i in range(4)]
refs = [net_oracle.forward(sd, w) for w in wins]
net_oracle.conv_bn_act = conv
for md in ('half', 'e4m3', 'e5m2', 'mxfp4'):
    MODE['m'] = md
    print('half hi*hi + corrections in %s\t%.3e' % (md, (net_oracle.forward(sd, wins[1]) - refs[1]).abs().max().item()), flush=True)
# all four windows of the 10 s input, and per-tensor scales 8x / 64x smaller than the tightest one: a static, calibrated
# scale per layer is enough (e4m3 keeps its relative precision over that range)
MODE['m'] = 'e4m3'
for top in (256.0, 32.0, 4.0):
    TOP['t'] = top
    errs = [(net_oracle.forward(sd, w) - r).abs().max().item() for w, r in zip(wins, refs)]
    print('e4m3 corrections, max|x| scaled to %3.0f of 448, windows 0-3\t%s' % (top, ' '.join('%.2e' % e for e in errs)), flush=True)
