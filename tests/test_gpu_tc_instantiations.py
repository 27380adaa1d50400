"""Every instantiation of the three wgmma convolution kernels against a float64 reference of the same layer.

The instantiations are read from the VR_TC_FOR_ALL (conv_tc.cu: KB x BN x pairing), VR_HALO_FOR_ALL (conv_tc_halo.cu:
BN x MB) and VR_ROWS_FOR_ALL (conv_tc_rows.cu: BN x fused upsample) macros, and the case table below must name each
of them and nothing else; that check needs no GPU.  On the GPU every case is one vr_debug_conv / vr_debug_decoder call,
and vr_debug_last_conv must report the instantiation the case names.  The geometry selects it: the kernel family from
k, stride, dilation and whether the maps tile, KB from Cin, BN and n_tiles from Cout, the pairing, MB and the row
kernel's 64-wide tile from vr_debug_set keys 8, 3 and 2, the fused upsample from vr_debug_decoder.

Each instantiation has a clean case and a ragged one: Cin % 16 != 0 (the last chunk is partly TMA zero fill), Cout not
a multiple of BN (down to 4 channels, or a second N tile with few real channels) and, on the generic kernel, a last
m-tile that is short: a batch that is not a whole number of the images a narrow tile stacks, an odd m-tile count under
PAIR_M.  Across the table: batch 27 with more tiles than one persistent wave in each family, stride 2 on odd input
sizes and dilation (12, 6) on maps shorter than the dilation (only the generic kernel takes those layers), and weights
with all-zero 8-channel groups and 32-channel chunks on the row and halo kernels, which skip them (vr_debug_set key 6).

Gate (oracle/layer_oracle.py): r = max |y - ref| / (sqrt(conv(x^2, w^2)) + 2^-4 |ref|) <= CONV_GATE, and on the same
inputs the two-product emulations that drop w_lo or x_lo must land at least nonvacuous_factor_fan_in times above it,
so every case would see a lost correction product.  Each case runs on randn inputs and on non-negative log-uniform
ones over [1e-6, 1] with 10 % exact zeros, as normalised magnitudes are.

Bitwise relations: PAIR_M and PAIR_N give the two-warpgroup kernel's outputs bit for bit; the halo kernel gives the
same bits at MB = 1, MB = 2 and its automatic choice; skipping all-zero weight groups changes no bit."""
import ctypes
import math
import os
import re
import zlib
from collections import namedtuple

import pytest
import torch

from conftest import ROOT, record_parity

Conv = namedtuple('Conv', 'inst n_tiles knobs N Cin H W Cout k stride dil act zero')
Dec = namedtuple('Dec', 'inst n_tiles knobs N Cl h w Cs Cout act zero')

CONV_CASES = [
    # instantiation, n_tiles, vr_debug_set knobs, N, Cin, H, W, Cout, k, stride, (dh, dw), act, zero weight channels
    Conv(('generic', 64, 16, 'PAIR_NONE'), 1, {8: 1}, 2, 64, 8, 32, 16, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 64, 16, 'PAIR_NONE'), 1, {8: 1}, 9, 56, 2, 16, 4, 3, 1, (1, 1), 1, ()),
    Conv(('generic', 64, 32, 'PAIR_NONE'), 1, {8: 1}, 1, 128, 16, 64, 32, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 64, 32, 'PAIR_NONE'), 1, {8: 1}, 5, 120, 7, 31, 27, 3, 2, (1, 1), 0, ()),
    Conv(('generic', 64, 48, 'PAIR_NONE'), 1, {8: 1}, 2, 64, 8, 16, 48, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 64, 48, 'PAIR_NONE'), 1, {8: 1}, 27, 56, 9, 128, 37, 1, 1, (1, 1), 2, ()),
    Conv(('generic', 64, 64, 'PAIR_NONE'), 1, {8: 1}, 2, 128, 8, 32, 64, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 64, 64, 'PAIR_NONE'), 1, {8: 1}, 19, 120, 1, 16, 57, 1, 1, (1, 1), 1, ()),
    Conv(('generic', 64, 80, 'PAIR_NONE'), 2, {8: 1}, 1, 64, 16, 64, 160, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 64, 80, 'PAIR_NONE'), 2, {8: 1}, 9, 56, 2, 16, 136, 3, 1, (1, 1), 0, ()),
    Conv(('generic', 64, 96, 'PAIR_NONE'), 1, {8: 1}, 2, 128, 8, 16, 96, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 64, 96, 'PAIR_NONE'), 1, {8: 1}, 5, 120, 7, 31, 84, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 64, 112, 'PAIR_NONE'), 1, {8: 1}, 2, 64, 8, 32, 112, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 64, 112, 'PAIR_NONE'), 2, {8: 1}, 3, 56, 4, 4, 200, 3, 1, (12, 6), 1, ()),
    Conv(('generic', 64, 128, 'PAIR_NONE'), 2, {8: 1}, 1, 128, 16, 64, 256, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 64, 128, 'PAIR_NONE'), 1, {8: 1}, 19, 120, 1, 16, 115, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 16, 'PAIR_NONE'), 1, {8: 1}, 2, 32, 8, 16, 16, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 32, 16, 'PAIR_NONE'), 1, {8: 1}, 9, 24, 2, 16, 4, 3, 1, (1, 1), 2, ()),
    Conv(('generic', 32, 32, 'PAIR_NONE'), 1, {8: 1}, 2, 96, 8, 32, 32, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 32, 'PAIR_NONE'), 1, {8: 1}, 5, 88, 7, 31, 27, 3, 2, (1, 1), 1, ()),
    Conv(('generic', 32, 48, 'PAIR_NONE'), 1, {8: 1}, 1, 32, 16, 64, 48, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 32, 48, 'PAIR_NONE'), 1, {8: 1}, 3, 24, 4, 4, 37, 3, 1, (12, 6), 0, ()),
    Conv(('generic', 32, 64, 'PAIR_NONE'), 1, {8: 1}, 2, 96, 8, 16, 64, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 32, 64, 'PAIR_NONE'), 1, {8: 1}, 19, 88, 1, 16, 57, 1, 1, (1, 1), 2, ()),
    Conv(('generic', 32, 80, 'PAIR_NONE'), 1, {8: 1}, 2, 32, 8, 32, 80, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 80, 'PAIR_NONE'), 2, {8: 1}, 9, 24, 2, 16, 136, 3, 1, (1, 1), 1, ()),
    Conv(('generic', 32, 96, 'PAIR_NONE'), 2, {8: 1}, 1, 96, 16, 64, 192, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 32, 96, 'PAIR_NONE'), 1, {8: 1}, 5, 88, 7, 31, 84, 3, 2, (1, 1), 0, ()),
    Conv(('generic', 32, 112, 'PAIR_NONE'), 1, {8: 1}, 2, 32, 8, 16, 112, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 32, 112, 'PAIR_NONE'), 2, {8: 1}, 3, 24, 4, 4, 200, 3, 1, (12, 6), 2, ()),
    Conv(('generic', 32, 128, 'PAIR_NONE'), 1, {8: 1}, 2, 96, 8, 32, 128, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 128, 'PAIR_NONE'), 1, {8: 1}, 19, 88, 1, 16, 115, 1, 1, (1, 1), 1, ()),
    Conv(('generic', 16, 16, 'PAIR_NONE'), 1, {8: 1}, 1, 16, 16, 64, 16, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 16, 16, 'PAIR_NONE'), 1, {8: 1}, 9, 40, 2, 16, 4, 3, 1, (1, 1), 0, ()),
    Conv(('generic', 16, 32, 'PAIR_NONE'), 1, {8: 1}, 2, 48, 8, 16, 32, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 16, 32, 'PAIR_NONE'), 1, {8: 1}, 5, 72, 7, 31, 27, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 16, 48, 'PAIR_NONE'), 1, {8: 1}, 2, 16, 8, 32, 48, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 16, 48, 'PAIR_NONE'), 1, {8: 1}, 3, 40, 4, 4, 37, 3, 1, (12, 6), 1, ()),
    Conv(('generic', 16, 64, 'PAIR_NONE'), 1, {8: 1}, 1, 48, 16, 64, 64, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 16, 64, 'PAIR_NONE'), 1, {8: 1}, 19, 72, 1, 16, 57, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 16, 80, 'PAIR_NONE'), 1, {8: 1}, 2, 16, 8, 16, 80, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 16, 80, 'PAIR_NONE'), 2, {8: 1}, 9, 40, 2, 16, 136, 3, 1, (1, 1), 2, ()),
    Conv(('generic', 16, 96, 'PAIR_NONE'), 1, {8: 1}, 2, 48, 8, 32, 96, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 16, 96, 'PAIR_NONE'), 1, {8: 1}, 5, 72, 7, 31, 84, 3, 2, (1, 1), 1, ()),
    Conv(('generic', 16, 112, 'PAIR_NONE'), 2, {8: 1}, 1, 16, 16, 64, 224, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 16, 112, 'PAIR_NONE'), 2, {8: 1}, 3, 40, 4, 4, 200, 3, 1, (12, 6), 0, ()),
    Conv(('generic', 16, 128, 'PAIR_NONE'), 1, {8: 1}, 2, 48, 8, 16, 128, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 16, 128, 'PAIR_NONE'), 1, {8: 1}, 19, 72, 1, 16, 115, 1, 1, (1, 1), 2, ()),
    Conv(('generic', 32, 16, 'PAIR_M'), 1, {8: 2}, 2, 32, 8, 32, 16, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 16, 'PAIR_M'), 1, {8: 2}, 9, 24, 2, 16, 4, 3, 1, (1, 1), 1, ()),
    Conv(('generic', 32, 32, 'PAIR_M'), 1, {8: 2}, 1, 128, 16, 64, 32, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 32, 32, 'PAIR_M'), 1, {8: 2}, 5, 120, 7, 31, 27, 3, 2, (1, 1), 0, ()),
    Conv(('generic', 32, 48, 'PAIR_M'), 1, {8: 2}, 2, 32, 8, 16, 48, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 32, 48, 'PAIR_M'), 1, {8: 2}, 3, 24, 4, 4, 37, 3, 1, (12, 6), 2, ()),
    Conv(('generic', 32, 64, 'PAIR_M'), 1, {8: 2}, 2, 128, 8, 32, 64, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 64, 'PAIR_M'), 1, {8: 2}, 19, 120, 1, 16, 57, 1, 1, (1, 1), 1, ()),
    Conv(('generic', 32, 80, 'PAIR_M'), 2, {8: 2}, 1, 32, 16, 64, 160, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 32, 80, 'PAIR_M'), 2, {8: 2}, 9, 24, 2, 16, 136, 3, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 96, 'PAIR_M'), 1, {8: 2}, 2, 128, 8, 16, 96, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 32, 96, 'PAIR_M'), 1, {8: 2}, 5, 120, 7, 31, 84, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 32, 112, 'PAIR_M'), 1, {8: 2}, 2, 32, 8, 32, 112, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 112, 'PAIR_M'), 2, {8: 2}, 27, 24, 9, 128, 200, 1, 1, (1, 1), 1, ()),
    Conv(('generic', 32, 128, 'PAIR_M'), 2, {8: 2}, 1, 128, 16, 64, 256, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 32, 128, 'PAIR_M'), 1, {8: 2}, 19, 120, 1, 16, 115, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 16, 16, 'PAIR_M'), 1, {8: 2}, 2, 16, 8, 16, 16, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 16, 16, 'PAIR_M'), 1, {8: 2}, 9, 40, 2, 16, 4, 3, 1, (1, 1), 2, ()),
    Conv(('generic', 16, 32, 'PAIR_M'), 1, {8: 2}, 2, 48, 8, 32, 32, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 16, 32, 'PAIR_M'), 1, {8: 2}, 5, 72, 7, 31, 27, 3, 2, (1, 1), 1, ()),
    Conv(('generic', 16, 48, 'PAIR_M'), 1, {8: 2}, 1, 16, 16, 64, 48, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 16, 48, 'PAIR_M'), 1, {8: 2}, 3, 40, 4, 4, 37, 3, 1, (12, 6), 0, ()),
    Conv(('generic', 16, 64, 'PAIR_M'), 1, {8: 2}, 2, 48, 8, 16, 64, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 16, 64, 'PAIR_M'), 1, {8: 2}, 19, 72, 1, 16, 57, 1, 1, (1, 1), 2, ()),
    Conv(('generic', 16, 80, 'PAIR_M'), 1, {8: 2}, 2, 16, 8, 32, 80, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 16, 80, 'PAIR_M'), 2, {8: 2}, 9, 40, 2, 16, 136, 3, 1, (1, 1), 1, ()),
    Conv(('generic', 16, 96, 'PAIR_M'), 2, {8: 2}, 1, 48, 16, 64, 192, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 16, 96, 'PAIR_M'), 1, {8: 2}, 5, 72, 7, 31, 84, 3, 2, (1, 1), 0, ()),
    Conv(('generic', 16, 112, 'PAIR_M'), 1, {8: 2}, 2, 16, 8, 16, 112, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 16, 112, 'PAIR_M'), 2, {8: 2}, 3, 40, 4, 4, 200, 3, 1, (12, 6), 2, ()),
    Conv(('generic', 16, 128, 'PAIR_M'), 1, {8: 2}, 2, 48, 8, 32, 128, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 16, 128, 'PAIR_M'), 1, {8: 2}, 19, 72, 1, 16, 115, 1, 1, (1, 1), 1, ()),
    Conv(('generic', 32, 80, 'PAIR_N'), 2, {8: 3}, 1, 32, 16, 64, 160, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 32, 80, 'PAIR_N'), 2, {8: 3}, 9, 24, 2, 16, 136, 3, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 96, 'PAIR_N'), 2, {8: 3}, 2, 128, 8, 16, 192, 3, 1, (4, 2), 1, ()),
    Conv(('generic', 32, 96, 'PAIR_N'), 2, {8: 3}, 27, 120, 9, 128, 170, 1, 1, (1, 1), 2, ()),
    Conv(('generic', 32, 112, 'PAIR_N'), 2, {8: 3}, 2, 32, 8, 32, 224, 1, 1, (1, 1), 0, ()),
    Conv(('generic', 32, 112, 'PAIR_N'), 2, {8: 3}, 3, 24, 4, 4, 200, 3, 1, (12, 6), 1, ()),
    Conv(('generic', 32, 128, 'PAIR_N'), 2, {8: 3}, 1, 128, 16, 64, 256, 3, 2, (1, 1), 2, ()),
    Conv(('generic', 32, 128, 'PAIR_N'), 2, {8: 3}, 19, 120, 1, 16, 230, 1, 1, (1, 1), 0, ()),
    Conv(('halo', 16, 1), 1, {3: 2}, 2, 64, 8, 32, 16, 3, 1, (1, 1), 1, ()),
    Conv(('halo', 16, 1), 1, {3: 2}, 3, 40, 16, 16, 4, 3, 1, (1, 1), 2, ()),
    Conv(('halo', 16, 2), 1, {3: 3}, 2, 96, 8, 32, 16, 3, 1, (1, 1), 0, ()),
    Conv(('halo', 16, 2), 1, {3: 3}, 1, 88, 4, 64, 4, 3, 1, (1, 1), 1, ()),
    Conv(('halo', 32, 1), 1, {3: 2}, 2, 64, 8, 32, 32, 3, 1, (1, 1), 2, ()),
    Conv(('halo', 32, 1), 1, {3: 2}, 2, 120, 8, 64, 27, 3, 1, (1, 1), 0, ()),
    Conv(('halo', 32, 2), 1, {3: 3}, 2, 96, 8, 32, 32, 3, 1, (1, 1), 1, ()),
    Conv(('halo', 32, 2), 1, {3: 3}, 3, 40, 16, 16, 27, 3, 1, (1, 1), 2, ()),
    Conv(('halo', 48, 1), 1, {3: 2}, 2, 64, 8, 32, 48, 3, 1, (1, 1), 0, ()),
    Conv(('halo', 48, 1), 1, {3: 2}, 27, 88, 16, 64, 37, 3, 1, (1, 1), 1, ()),
    Conv(('halo', 48, 2), 1, {3: 3}, 2, 96, 8, 32, 48, 3, 1, (1, 1), 2, ()),
    Conv(('halo', 48, 2), 1, {3: 3}, 2, 120, 8, 64, 37, 3, 1, (1, 1), 0, ()),
    Conv(('halo', 64, 1), 1, {3: 2}, 2, 64, 8, 32, 64, 3, 1, (1, 1), 1, ()),
    Conv(('halo', 64, 1), 1, {3: 2}, 3, 40, 16, 16, 57, 3, 1, (1, 1), 2, ()),
    Conv(('halo', 64, 2), 1, {3: 3}, 2, 96, 8, 32, 64, 3, 1, (1, 1), 0, ()),
    Conv(('halo', 64, 2), 1, {3: 3}, 1, 88, 4, 64, 57, 3, 1, (1, 1), 1, ()),
    Conv(('halo', 96, 1), 1, {3: 2}, 2, 64, 8, 32, 96, 3, 1, (1, 1), 2, ()),
    Conv(('halo', 96, 1), 2, {3: 2}, 2, 88, 8, 64, 170, 3, 1, (1, 1), 0, ((8, 16), (32, 64))),
    Conv(('halo', 96, 2), 2, {3: 3}, 2, 96, 8, 32, 192, 3, 1, (1, 1), 1, ()),
    Conv(('halo', 96, 2), 1, {3: 3}, 3, 40, 16, 16, 84, 3, 1, (1, 1), 2, ()),
    Conv(('halo', 128, 1), 1, {3: 2}, 2, 64, 8, 32, 128, 3, 1, (1, 1), 0, ()),
    Conv(('halo', 128, 1), 2, {3: 2}, 1, 88, 4, 64, 230, 3, 1, (1, 1), 1, ()),
    Conv(('halo', 128, 2), 2, {3: 3}, 2, 96, 8, 32, 256, 3, 1, (1, 1), 2, ()),
    Conv(('halo', 128, 2), 1, {3: 3}, 2, 120, 8, 64, 115, 3, 1, (1, 1), 0, ()),
    Conv(('rows', 16, False), 1, {2: 0}, 1, 64, 8, 128, 16, 3, 1, (1, 1), 1, ()),
    Conv(('rows', 16, False), 1, {2: 0}, 2, 40, 16, 256, 4, 3, 1, (1, 1), 2, ((8, 16),)),
    Conv(('rows', 32, False), 1, {2: 0}, 1, 64, 8, 128, 32, 3, 1, (1, 1), 0, ()),
    Conv(('rows', 32, False), 2, {2: 0}, 27, 24, 16, 128, 40, 3, 1, (1, 1), 1, ()),
    Conv(('rows', 64, False), 1, {2: 1}, 1, 64, 8, 128, 64, 3, 1, (1, 1), 2, ((16, 24), (32, 64))),
    Conv(('rows', 64, False), 2, {2: 1}, 3, 88, 8, 128, 120, 3, 1, (1, 1), 0, ()),
]

DEC_CASES = [
    # instantiation, n_tiles, knobs, N, Cl (low-res channels), h, w, Cs (skip channels), Cout, act, zero weight channels
    Dec(('rows', 16, True), 1, {}, 1, 32, 4, 64, 32, 16, 1, ()),
    Dec(('rows', 16, True), 1, {}, 2, 40, 8, 64, 13, 4, 2, ()),
    Dec(('rows', 32, True), 1, {}, 1, 64, 4, 64, 32, 32, 0, ((32, 64),)),
    Dec(('rows', 32, True), 2, {}, 2, 40, 8, 64, 13, 40, 1, ()),
    Dec(('rows', 64, True), 1, {}, 1, 32, 4, 64, 32, 64, 2, ()),
    Dec(('rows', 64, True), 2, {}, 2, 40, 8, 64, 13, 120, 0, ()),
]

CASES = CONV_CASES + DEC_CASES
CSRC = os.path.join(ROOT, 'vocal-remover_b200', 'csrc')
FOR_ALL = {'generic': ('conv_tc.cu', 'VR_TC_FOR_ALL'), 'halo': ('conv_tc_halo.cu', 'VR_HALO_FOR_ALL'),
           'rows': ('conv_tc_rows.cu', 'VR_ROWS_FOR_ALL')}
KIND = {'generic': 1, 'rows': 2, 'halo': 3}
PAIR = {'PAIR_NONE': 0, 'PAIR_M': 1, 'PAIR_N': 2}
ACT = {0: None, 1: 'relu', 2: 'leaky'}
DEFAULT_KNOBS = {2: 0, 3: 0, 6: 1, 8: 0}


def _value(tok):
    return int(tok) if tok.isdigit() else {'true': True, 'false': False}.get(tok, tok)


def _expand(macros, name, args, emit):
    """expands macro `name`(args); calls of the parameter bound to '<emit>' are the instantiations"""
    params, body = macros[name]
    env = dict(zip(params, args))
    for m in re.finditer(r'(\w+)\(([^()]*)\)', body):
        callee = env.get(m.group(1), m.group(1))
        cargs = [env.get(a.strip(), a.strip()) for a in m.group(2).split(',')]
        if callee == '<emit>':
            emit(tuple(_value(a) for a in cargs))
        else:
            _expand(macros, callee, cargs, emit)


def instantiations():
    """{('generic', KB, BN, pairing), ('halo', BN, MB), ('rows', BN, up)} as the FOR_ALL macros list them"""
    out = set()
    for family, (src, top) in FOR_ALL.items():
        with open(os.path.join(CSRC, src)) as f:
            text = f.read().replace('\\\n', ' ')
        macros = {m.group(1): ([a.strip() for a in m.group(2).split(',')], m.group(3))
                  for m in re.finditer(r'^#define\s+(\w+)\(([^)]*)\)(.*)$', text, re.M)}
        found = []
        _expand(macros, top, ['<emit>'], found.append)
        assert found, 'no instantiations parsed from %s in %s' % (top, src)
        out |= {(family,) + args for args in found}
    return out


def _cin(c):
    return c.Cl + c.Cs if isinstance(c, Dec) else c.Cin


def test_case_table_covers_every_instantiation():
    built = instantiations()
    named = {c.inst for c in CASES}
    missing, extra = sorted(built - named, key=str), sorted(named - built, key=str)
    assert not missing, 'instantiations without a case: %s' % missing
    assert not extra, 'cases of instantiations no FOR_ALL macro lists: %s' % extra
    for inst in built:
        bn = inst[2] if inst[0] == 'generic' else inst[1]
        assert any(_cin(c) % 16 and c.Cout % bn for c in CASES if c.inst == inst), \
            'no ragged case (Cin % 16 != 0, Cout % BN != 0) for %s' % (inst,)


def _case_id(c):
    geo = ('dec%d_%dx%dx%d+%d' % (c.N, c.Cl, c.h, c.w, c.Cs) if isinstance(c, Dec) else
           'n%d_%dx%dx%d_k%ds%dd%dx%d' % (c.N, c.Cin, c.H, c.W, c.k, c.stride, c.dil[0], c.dil[1]))
    return '%s_%s_co%d%s' % ('_'.join(str(v) for v in c.inst), geo, c.Cout, '_zero' if c.zero else '')


def _input(shape, dist, g):
    if dist == 'randn':
        return torch.randn(shape, generator=g)
    # log-uniform over [1e-6, 1], with about 10 % exact zeros
    x = torch.exp(torch.rand(shape, generator=g, dtype=torch.float64) * math.log(1e-6)).float()
    x[torch.rand(shape, generator=g) < 0.1] = 0.0
    return x


def _operands(c, dist):
    g = torch.Generator().manual_seed(zlib.crc32(repr((c, dist)).encode()))
    k = 3 if isinstance(c, Dec) else c.k
    cin = _cin(c)
    if isinstance(c, Dec):
        xs = (_input((c.N, c.Cl, c.h, c.w), dist, g), _input((c.N, c.Cs, 2 * c.h, 2 * c.w), dist, g))
    else:
        xs = (_input((c.N, c.Cin, c.H, c.W), dist, g),)
    w = torch.randn(c.Cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    for c0, c1 in c.zero:
        w[:, c0:c1] = 0.0
    b = torch.randn(c.Cout, generator=g) * 0.1
    return xs, w, b


def _run(ctx, c, xs, w, b, knobs):
    """one vr_debug_conv / vr_debug_decoder call under the vr_debug_set knobs -> (y, vr_debug_last_conv)"""
    from lib import _native
    lib = ctx.lib
    try:
        for key, val in knobs.items():
            assert lib.vr_debug_set(key, val) == 0
        dev = [t.cuda() for t in xs + (w, b)]
        if isinstance(c, Dec):
            y = torch.empty((c.N, c.Cout, 2 * c.h, 2 * c.w), dtype=torch.float32, device='cuda')
            ctx.check(lib.vr_debug_decoder(ctx.handle, _native.ptr(dev[0]), c.N, c.Cl, c.h, c.w, _native.ptr(dev[1]),
                                           c.Cs, _native.ptr(dev[2]), _native.ptr(dev[3]), c.Cout, c.act, 1,
                                           _native.ptr(y), _native.stream_ptr()), 'vr_debug_decoder')
        else:
            Ho, Wo = (c.H - 1) // c.stride + 1, (c.W - 1) // c.stride + 1
            y = torch.empty((c.N, c.Cout, Ho, Wo), dtype=torch.float32, device='cuda')
            ctx.check(lib.vr_debug_conv(ctx.handle, _native.ptr(dev[0]), c.N, c.Cin, c.H, c.W, _native.ptr(dev[1]),
                                        _native.ptr(dev[2]), c.Cout, c.k, c.stride, c.dil[0], c.dil[1], c.act, 1,
                                        _native.ptr(y), _native.stream_ptr()), 'vr_debug_conv')
        last = (ctypes.c_int32 * 8)()
        assert lib.vr_debug_last_conv(last) == 0
        return y.cpu(), tuple(last)
    finally:
        for key in knobs:
            lib.vr_debug_set(key, DEFAULT_KNOBS[key])


def _reported(c):
    """the first seven fields vr_debug_last_conv must report for the case's instantiation"""
    fam = c.inst[0]
    if fam == 'generic':
        _, kb, bn, mode = c.inst
        return (KIND[fam], kb, bn, c.n_tiles, PAIR[mode], 0, 0)
    if fam == 'halo':
        return (KIND[fam], 32, c.inst[1], c.n_tiles, 0, c.inst[2], 0)
    return (KIND[fam], 32, c.inst[1], c.n_tiles, 0, 0, int(c.inst[2]))


@pytest.fixture(scope='module')
def ctx():
    from lib import _native
    c = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    yield c
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize('dist', ['randn', 'logu'])
@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_instantiation_vs_float64(ctx, case, dist):
    from oracle import layer_oracle as lo
    c = case
    xs, w, b = _operands(c, dist)
    y, last = _run(ctx, c, xs, w, b, c.knobs)
    assert last[:7] == _reported(c), 'launched %s, the case names %s' % (last, _reported(c))

    # float64 reference of the same fp32 tensors, the gate and its non-vacuity
    if isinstance(c, Dec):
        x = torch.cat([lo.up2x(xs[0].double()), xs[1].double()], 1)
        kw = dict(stride=1, pad=1, dil=1)
        fan_in = 9 * (c.Cl + c.Cs)
    else:
        x = xs[0].double()
        kw = dict(stride=c.stride, pad=(c.dil[0] * (c.k // 2), c.dil[1] * (c.k // 2)), dil=c.dil)
        fan_in = c.Cin * c.k * c.k
    r, r_wlo, r_xlo, _, _ = lo.conv_ratios_of(x, w.double(), b.double(), y.double(), act=ACT[c.act], **kw)
    record_parity('tc_inst_%s_%s' % (_case_id(c), dist), r, lo.CONV_GATE)
    need = lo.nonvacuous_factor_fan_in(fan_in) * lo.CONV_GATE
    assert min(r_wlo, r_xlo) >= need, 'vacuous gate: no_wlo %.3g, no_xlo %.3g, need %.3g' % (r_wlo, r_xlo, need)
    assert r <= lo.CONV_GATE, r

    # bitwise relations
    fam = c.inst[0]
    if fam == 'generic' and c.inst[3] != 'PAIR_NONE':
        y1, last1 = _run(ctx, c, xs, w, b, {8: 1})
        assert last1[0] == KIND['generic'] and last1[4] == PAIR['PAIR_NONE'], last1
        assert torch.equal(y, y1), (y - y1).abs().max().item()
    if fam == 'halo':
        for knob in (2, 3, 0):   # MB = 1, MB = 2 (where the height tiles), automatic
            yk, lastk = _run(ctx, c, xs, w, b, {3: knob})
            assert lastk[0] == KIND['halo'] and lastk[2] == c.inst[1], lastk
            assert torch.equal(y, yk), (knob, lastk, (y - yk).abs().max().item())
    if c.zero:
        y0, last0 = _run(ctx, c, xs, w, b, {**c.knobs, 6: 0})
        assert last0[:7] == last[:7], last0
        assert torch.equal(y, y0), (y - y0).abs().max().item()
