"""CPU emulation of the tensor-core convolution's arithmetic.  TEST INFRASTRUCTURE.

The product computes every Conv2DBNActiv as the sum of products of operand pairs (x = hi + lo, w' = hi + lo, with the
BatchNorm folded into w' at weight load) with fp32 accumulation, and stores its output as such a pair (DESIGN §3).
A ``Scheme`` states one variant of that arithmetic as data: the pair format, which products are issued, and how the
operands of the correction products are quantised.  ``Scheme.conv_bn_act`` runs it in place of
``net_oracle.conv_bn_act``, and an ``Assignment`` gives every layer of a forward its scheme:

    net_oracle.forward(sd, x, conv=Assignment(Scheme(products=('hh', 'lh'))))
"""
import dataclasses
import functools
import operator

import numpy as np
import torch
import torch.nn.functional as F

from oracle import net_oracle


def bf16(x):
    return x.to(torch.bfloat16).to(x.dtype)


def half(x):
    return x.to(torch.float16).to(x.dtype)


ROUND = {'bf16': bf16, 'half': half}
FP8 = {'e4m3': torch.float8_e4m3fn, 'e5m2': torch.float8_e5m2}


def split(x, fmt, round_lo=True):
    """(hi, lo) with hi = x rounded to ``fmt`` ('bf16' or 'half') and lo = x - hi, itself rounded to ``fmt`` unless
    ``round_lo`` is false."""
    hi = ROUND[fmt](x)
    return hi, ROUND[fmt](x - hi) if round_lo else x - hi


def fold_bn(sd, bn, pre_bias=None):
    """eval BatchNorm at ``bn`` as y = scale * x + shift per channel, in float64 (engine.cu fold_bn)."""
    g, b = net_oracle._t(sd, bn + '.weight').double(), net_oracle._t(sd, bn + '.bias').double()
    m, v = net_oracle._t(sd, bn + '.running_mean').double(), net_oracle._t(sd, bn + '.running_var').double()
    scale = g / torch.sqrt(v + net_oracle.BN_EPS)
    shift = scale * ((0.0 if pre_bias is None else pre_bias.double()) - m) + b
    return scale, shift


def folded_conv(sd, p):
    """(w', b') of Conv2DBNActiv ``p``: its weights and bias with the BatchNorm folded in, float64."""
    scale, shift = fold_bn(sd, p + '.conv.1')
    return net_oracle._t(sd, p + '.conv.0.weight').double() * scale[:, None, None, None], shift


def activation(y, act):
    return F.relu(y) if act == 'relu' else F.leaky_relu(y, 0.01)


def scaled_fp8(x, dt, top):
    """``dt`` rounding with a per-tensor power-of-two scale that puts max|x| just under ``top``."""
    m = x.abs().max().item()
    if m == 0.0:
        return x
    s = 2.0 ** np.floor(np.log2(top / m))
    return (x * s).to(dt).to(torch.float32) / s


GRID4 = torch.tensor([0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0])


def mxfp4(x, dim=1, blk=32):
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


@dataclasses.dataclass(frozen=True)
class Scheme:
    """One emulated convolution arithmetic.  The default is the product's: bf16 pairs, three products, bf16 output.

    pair      format of the operand pairs, 'bf16' or 'half'
    round_lo  lo rounded to the pair format; False keeps lo = x - hi exact and leaves its rounding to ``corr``
    products  which of hi*hi ('hh'), lo*hi ('lh', x_lo * w_hi) and hi*lo ('hl', x_hi * w_lo) are issued
    corr      quantiser of both operands of the correction products: None, 'e4m3' or 'e5m2' (per-tensor power-of-two
              scale that puts max|x| just under ``top``), or 'mxfp4' (blocks of 32 input channels)
    out       format of the stored output pair
    """
    pair: str = 'bf16'
    round_lo: bool = True
    products: tuple = ('hh', 'lh', 'hl')
    corr: str = None
    top: float = 256.0
    out: str = 'bf16'

    def quantise(self, t):
        if self.corr is None:
            return t
        if self.corr == 'mxfp4':
            return mxfp4(t)
        return scaled_fp8(t, FP8[self.corr], self.top)

    def conv_bn_act(self, sd, p, x, stride=1, pad=1, dil=1, act='relu'):
        """net_oracle.conv_bn_act at prefix ``p`` in this arithmetic: the issued products of the split operands
        summed in fp32 as hh + lh + hl, then the folded bias, the activation, and the output rounded to a pair."""
        w, b = folded_conv(sd, p)
        xh, xl = split(x, self.pair, self.round_lo)
        wh, wl = split(w.float(), self.pair, self.round_lo)
        q = self.quantise
        kw = dict(stride=stride, padding=pad, dilation=dil)
        terms = []
        if 'hh' in self.products:
            terms.append(F.conv2d(xh, wh, None, **kw))
        if 'lh' in self.products:
            terms.append(F.conv2d(q(xl), q(wh), None, **kw))
        if 'hl' in self.products:
            terms.append(F.conv2d(q(xh), q(wl), None, **kw))
        y = functools.reduce(operator.add, terms) + b.float()[None, :, None, None]
        hi, lo = split(activation(y, act), self.out)
        return hi + lo


class Assignment:
    """The ``conv`` of net_oracle.forward that runs layer prefix p with ``schemes[p]``, every other layer with
    ``default``.  ``layers`` lists the prefixes in the order they first ran."""

    def __init__(self, default=Scheme(), schemes=None):
        self.default = default
        self.schemes = dict(schemes or {})
        self.layers = []

    def __call__(self, sd, p, x, stride=1, pad=1, dil=1, act='relu'):
        if p not in self.layers:
            self.layers.append(p)
        return self.schemes.get(p, self.default).conv_bn_act(sd, p, x, stride, pad, dil, act)
