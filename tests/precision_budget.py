"""Precision budget of the tensor-core convolution (CPU emulation; not a pytest module).

The product computes every convolution as hi*hi + lo*hi + hi*lo of bf16 pairs (x = hi + lo, 16-bit significand) with fp32
accumulation, and stores every activation as such a pair.  Each subcommand runs the oracle's functional CascadedNet
(oracle/net_oracle.py) with variants of that arithmetic (oracle/precision_oracle.py) and prints the mask max-abs error
against the fp32 oracle (seeded synthetic checkpoint, lib/synth.py; window 1 of the 10 s input unless stated):

layers [out.tsv]  ONE layer at a time, then every layer, drops one of the two correction products:
                      3pass   hi*hi + lo*hi + hi*lo          (the product path)
                      no_wlo  (hi + lo) * w_hi               two MMAs per k-step: weights rounded to bf16
                      no_xlo  x_hi * (w_hi + w_lo)           two MMAs per k-step: activations rounded to bf16
                      1pass   x_hi * w_hi
fp8 [out.tsv]     both operands of the two correction products in fp8 e4m3 (per-tensor power-of-two scale, max|x| just
                  under 256 of 448), which could run as fp8 MMAs at twice the bf16 rate: every layer at once, then one
                  layer at a time.
fp16              IEEE half pairs (11-bit significands) instead of bf16 pairs, for the four product sets of `layers`.
mixed             main product in half (x_hi16 * w_hi16) and the two corrections with both operands in half, e4m3,
                  e5m2 or block-scaled fp4, lo = x - hi kept exact before that rounding.  With a half hi part the lo
                  part is 2^-12 of the value instead of bf16's 2^-9, so the fp8 rounding of the corrections weighs 8x
                  less than in `fp8`: 1 + 1/2 + 1/2 = 2 units of tensor time per product instead of 3, and an
                  activation still costs 4 bytes (half hi + fp8 lo + fp8 copy of hi).  Then e4m3 on all four windows
                  with per-tensor scales 8x / 64x smaller than the tightest one: a static, calibrated scale per layer
                  is enough if the error holds (e4m3 keeps its relative precision over that range).

Usage: python tests/precision_budget.py layers|fp8 [out.tsv] | fp16 | mixed
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'vocal-remover_b200'))
from lib import synth  # noqa: E402
from oracle import net_oracle, separator_oracle, stft_oracle  # noqa: E402
from oracle.precision_oracle import Assignment, Scheme  # noqa: E402

PRODUCTS = {'3pass': ('hh', 'lh', 'hl'), 'no_wlo': ('hh', 'lh'), 'no_xlo': ('hh', 'hl'), '1pass': ('hh',)}
BF16 = {k: Scheme(products=v) for k, v in PRODUCTS.items()}
HALF = {k: Scheme(pair='half', products=v, out='half') for k, v in PRODUCTS.items()}


def setup(windows):
    """The synthetic checkpoint and (x, fp32 oracle mask) of the given 256-frame windows of the 10 s input."""
    sd = synth.to_torch_state_dict(synth.make_state_dict())
    wave = synth.sine_mix(10.0)
    X = stft_oracle.wave_to_spectrogram(wave, 1024, 2048)
    pad_l, pad_r, roi = separator_oracle.make_padding(X.shape[2], 256, 64)
    Xp = np.pad(X, ((0, 0), (0, 0), (pad_l, pad_r)))
    Xp /= np.abs(X).max()
    out = []
    for i in windows:
        x = torch.from_numpy(np.abs(Xp[None, :, :, i * roi:i * roi + 256]).astype(np.float32))
        out.append((x, net_oracle.forward(sd, x)))
    return sd, out


def error(sd, window, conv):
    x, ref = window
    return (net_oracle.forward(sd, x, conv=conv) - ref).abs().max().item()


class Sweep:
    """Errors on one window, each printed with its run time and kept for out.tsv."""

    def __init__(self, sd, window):
        self.sd, self.window, self.lines = sd, window, []

    def run(self, tag, conv):
        t0 = time.time()
        err = error(self.sd, self.window, conv)
        self.lines.append('%s\t%.3e' % (tag, err))
        print(self.lines[-1], '(%.1f s)' % (time.time() - t0), flush=True)
        return err

    def save(self, path, base):
        with open(path, 'w') as f:
            f.write('# mask max-abs error vs the fp32 oracle, first window of the 10 s input; baseline (all 3pass) %.3e\n' % base)
            f.write('\n'.join(self.lines) + '\n')


def layers(out_path=None):
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    sd, (win,) = setup([1])
    sweep, first = Sweep(sd, win), Assignment()
    base = sweep.run('all layers 3pass', first)
    for name in ('no_wlo', 'no_xlo'):
        for p in first.layers:
            sweep.run('%s\t%s' % (name, p), Assignment(schemes={p: BF16[name]}))
    for name in ('no_wlo', 'no_xlo', '1pass'):
        sweep.run('all layers %s' % name, Assignment(BF16[name]))
    if out_path:
        sweep.save(out_path, base)


def fp8(out_path=None):
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    sd, (win,) = setup([1])
    sweep, first, fp8corr = Sweep(sd, win), Assignment(), Scheme(corr='e4m3')
    base = sweep.run('all layers 3pass', first)
    sweep.run('all layers fp8corr', Assignment(fp8corr))
    for p in first.layers:
        sweep.run('fp8corr\t%s' % p, Assignment(schemes={p: fp8corr}))
    if out_path:
        sweep.save(out_path, base)


def fp16():
    torch.set_num_threads(8)
    sd, (win,) = setup([1])
    for name, scheme in HALF.items():
        print('fp16 all layers %s\t%.3e' % (name, error(sd, win, Assignment(scheme))), flush=True)


def mixed():
    torch.set_num_threads(8)
    sd, wins = setup(range(4))
    exact_lo = dict(pair='half', round_lo=False, out='half')
    corrections = {'half': HALF['3pass'],   # exact lo rounded to half: the plain half-pair scheme
                   'e4m3': Scheme(corr='e4m3', **exact_lo),
                   'e5m2': Scheme(corr='e5m2', top=16384.0, **exact_lo),
                   'mxfp4': Scheme(corr='mxfp4', **exact_lo)}
    for name, scheme in corrections.items():
        print('half hi*hi + corrections in %s\t%.3e' % (name, error(sd, wins[1], Assignment(scheme))), flush=True)
    for top in (256.0, 32.0, 4.0):
        conv = Assignment(Scheme(corr='e4m3', top=top, **exact_lo))
        errs = [error(sd, w, conv) for w in wins]
        print('e4m3 corrections, max|x| scaled to %3.0f of 448, windows 0-3\t%s' % (top, ' '.join('%.2e' % e for e in errs)),
              flush=True)


if __name__ == '__main__':
    commands = {'layers': layers, 'fp8': fp8, 'fp16': fp16, 'mixed': mixed}
    if len(sys.argv) < 2 or sys.argv[1] not in commands:
        sys.exit(__doc__)
    commands[sys.argv[1]](*sys.argv[2:])
