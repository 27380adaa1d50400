"""Halo-tile convolution (csrc/conv_tc_halo.cu: 3x3, stride 1, W = 16 / 32 / 64) against the per-tap wgmma kernel it
replaces for these layers (vr_debug_set(3, 1) routes them back to it) and against a float64 torch reference, with
tiles of 128 and 256 pixels (MB = 1 / 2, pinned with vr_debug_set(3, 2) / (3, 3))."""
import pytest
import torch

from conftest import record_parity
from test_gpu_parity import _ref_conv, _run_debug_conv

pytestmark = pytest.mark.gpu

HALO_CASES = [
    # N, Cin, H, W, Cout, act
    (2, 320, 16, 64, 128, 1),   # dec3 class: ten chunks, BN = 128
    (2, 448, 8, 32, 192, 1),    # dec4 class: fourteen chunks, two N tiles of 96
    (1, 128, 8, 64, 128, 1),    # enc3.conv2 class
    (3, 192, 8, 32, 192, 2),    # enc4.conv2 class, three images
    (2, 256, 16, 16, 256, 1),   # enc5.conv2 class: eight rows per tile, two N tiles of 128
    (1, 80, 8, 32, 64, 1),      # Cin 80: a partial last chunk
    (2, 112, 16, 16, 48, 2),    # Cin 112, BN = 48
    (4, 16, 32, 64, 32, 0),     # one mostly zero-filled chunk, several tiles per image, no activation
    (33, 32, 64, 64, 32, 1),    # enough tiles for the automatic choice of MB = 2
]


def _case(case, seed):
    N, Cin, H, W, Cout, act = case
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    return x, w, b, act


@pytest.mark.parametrize('case', HALO_CASES)
def test_halo_conv_vs_per_tap_kernel_and_torch(case):
    from lib import _native
    x, w, b, act = _case(case, 11 + len(HALO_CASES) * case[1] + case[3])
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    ref = _ref_conv(x, w, b, 3, 1, (1, 1), act)
    scale = max(1.0, ref.abs().max().item())
    ys = {}
    try:
        for knob in (0, 1, 2, 3):   # automatic MB, per-tap kernel, MB = 1, MB = 2
            ctx.lib.vr_debug_set(3, knob)
            ys[knob] = _run_debug_conv(ctx, x, w, b, 3, 1, (1, 1), act, 1)
    finally:
        ctx.lib.vr_debug_set(3, 0)
    err = max((ys[k] - ref).abs().max().item() for k in (0, 2, 3))
    record_parity('conv_tc_halo_%s' % '_'.join(str(v) for v in case), err / scale, 2e-4)
    assert err < 2e-4 * scale, err
    assert (ys[1] - ref).abs().max().item() < 2e-4 * scale
    # same split-bf16 products, only the fp32 accumulation order differs from the per-tap kernel: the outputs agree to
    # about one step of their split-bf16 storage (16 significant bits); MB does not change the order at all
    assert (ys[2] - ys[1]).abs().max().item() < 2 ** -15 * scale
    assert torch.equal(ys[2], ys[3])
    assert torch.equal(ys[0], ys[2])


def test_halo_conv_shapes_that_do_not_tile_fall_back():
    """H = 2 at W = 32 (four rows per tile) and H = 4 at W = 16 (eight) go to the per-tap kernel."""
    from lib import _native
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    for case in [(3, 64, 2, 32, 32, 1), (2, 64, 4, 16, 64, 1)]:
        x, w, b, act = _case(case, 5)
        ref = _ref_conv(x, w, b, 3, 1, (1, 1), act)
        y = _run_debug_conv(ctx, x, w, b, 3, 1, (1, 1), act, 1)
        assert (y - ref).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())
