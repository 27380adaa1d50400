"""wgmma implicit-GEMM convolutions (csrc/conv_tc*.cu) against a float64 torch reference of the same op,
layer class by layer class (3x3, strided, dilated, 1x1, ragged batch, multi-N-tile), called through the C ABI.  Each
case runs on the kernel tc_choose picks for its geometry: the row kernel (3x3 stride 1, W % 128 == 0, H % 8 == 0), else
the halo kernel (3x3 stride 1, W = 16 / 32 / 64, whole tiles of 128 / W rows), else the generic one."""
import pytest
import torch

from conftest import record_parity
from test_gpu_parity import _ref_conv, _run_debug_conv

pytestmark = pytest.mark.gpu

TC_CASES = [
    # N, Cin, H, W, Cout, k, stride, (dh, dw), act
    (1, 64, 8, 128, 64, 3, 1, (1, 1), 1),      # row kernel, two N tiles of 32
    (1, 32, 16, 64, 32, 3, 1, (1, 1), 1),      # halo kernel, 2 rows per 128-pixel tile
    (2, 16, 16, 16, 16, 3, 1, (1, 1), 2),      # halo kernel, 8 rows per 128-pixel tile
    (1, 2, 8, 256, 16, 3, 1, (1, 1), 1),       # first layer shape class (row kernel): Cin=2 padded to 32, W=256
    (1, 64, 32, 32, 128, 3, 2, (1, 1), 2),     # generic, KB=64 (SW128): stride 2 (TMA element strides)
    (1, 32, 16, 256, 64, 3, 2, (1, 1), 2),     # stride 2, wide
    (1, 64, 32, 16, 64, 3, 1, (4, 2), 1),      # dilated ASPP
    (1, 64, 32, 16, 64, 3, 1, (12, 6), 1),
    (1, 320, 8, 16, 256, 1, 1, (1, 1), 1),     # 1x1 bottleneck, two N tiles of 128
    (3, 64, 2, 16, 32, 3, 1, (1, 1), 1),       # generic (H=2 is no halo tile): 4 images per tile, ragged batch
    (1, 128, 8, 32, 192, 3, 1, (1, 1), 1),     # halo kernel, BN=96 x 2
    (1, 97, 4, 128, 32, 3, 1, (1, 1), 1),      # generic (H=4 is no row tile): dec1 shape class, Cin=97 -> 112, KB=16
    (2, 448, 8, 32, 192, 3, 1, (1, 1), 1),     # halo kernel: dec4 shape class, deep K
    (5, 256, 1, 16, 256, 1, 1, (1, 1), 1),     # ASPP pooled branch: H=1, 8 images per tile, ragged
    (1, 16, 16, 64, 8, 3, 1, (1, 1), 0),       # halo kernel: Cout=8 -> N=16, no activation
    # row-streaming kernel (3x3, stride 1, W % 128 == 0, H % 8 == 0)
    (1, 64, 8, 128, 32, 3, 1, (1, 1), 1),
    (1, 16, 8, 128, 16, 3, 1, (1, 1), 1),      # one 32-channel chunk, half of it TMA zero fill
    (1, 32, 16, 256, 32, 3, 1, (1, 1), 2),     # two 128-pixel tiles per row
    (2, 97, 8, 128, 32, 3, 1, (1, 1), 1),      # dec1 class: 97 -> 112 channels, two chunks
    (1, 192, 16, 128, 64, 3, 1, (1, 1), 1),    # dec2 class: three chunks, two N tiles
    (3, 2, 24, 256, 8, 3, 1, (1, 1), 0),       # more tiles than one wave per CTA set, Cout 8
]


@pytest.mark.parametrize('case', TC_CASES)
def test_conv_tcgen05_vs_torch(case):
    from lib import _native
    N, Cin, H, W, Cout, k, stride, dil, act = case
    g = torch.Generator().manual_seed(abs(hash(case)) % (2 ** 31))
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    y = _run_debug_conv(ctx, x, w, b, k, stride, dil, act, 1)
    ref = _ref_conv(x, w, b, k, stride, dil, act)
    err = (y - ref).abs().max().item()
    record_parity('conv_tc_%s' % '_'.join(str(v) for v in case).replace(' ', ''), err / max(1.0, ref.abs().max().item()), 2e-4)
    assert err < 2e-4 * max(1.0, ref.abs().max().item()), err
    # and the CUDA-core kernel agrees with it even more closely (same split-bf16 storage)
    y2 = _run_debug_conv(ctx, x, w, b, k, stride, dil, act, 0)
    assert (y - y2).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item())


DEC_CASES = [
    # N, Cl (low-res channels), h, w, Cs (skip channels), Cout, act
    (1, 64, 4, 64, 32, 32, 1),        # dec1/dec2 class, W = 128
    (2, 32, 8, 128, 16, 16, 1),       # W = 256: two 128-pixel tiles per row, BN = 16
    (1, 128, 8, 64, 64, 64, 1),       # four up chunks, two N tiles
    (1, 80, 4, 64, 32, 32, 2),        # low-res channel count padded to a chunk (96)
]


@pytest.mark.parametrize('case', DEC_CASES)
def test_decoder_fused_upsample_vs_staged_and_torch(case):
    """Decoder (lib/layers.py:51-64): bilinear x2 upsample fused into the row-streaming kernel's operand producer."""
    import torch.nn.functional as F
    from lib import _native
    N, Cl, h, w, Cs, Cout, act = case
    g = torch.Generator().manual_seed(abs(hash(case)) % (2 ** 31))
    low = torch.randn(N, Cl, h, w, generator=g)
    skip = torch.randn(N, Cs, 2 * h, 2 * w, generator=g)
    wgt = torch.randn(Cout, Cl + Cs, 3, 3, generator=g) / ((Cl + Cs) * 9) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    outs = []
    for fused in (0, 1):
        y = torch.empty((N, Cout, 2 * h, 2 * w), dtype=torch.float32, device='cuda')
        dl, ds, dw, db = low.cuda(), skip.cuda(), wgt.cuda(), b.cuda()
        ctx.check(ctx.lib.vr_debug_decoder(ctx.handle, _native.ptr(dl), N, Cl, h, w, _native.ptr(ds), Cs,
                                           _native.ptr(dw), _native.ptr(db), Cout, act, fused, _native.ptr(y),
                                           _native.stream_ptr()), 'vr_debug_decoder')
        outs.append(y.cpu())
    x = torch.cat([F.interpolate(low.double(), scale_factor=2, mode='bilinear', align_corners=True), skip.double()], 1)
    ref = F.conv2d(x, wgt.double(), b.double(), padding=1)
    ref = F.relu(ref) if act == 1 else F.leaky_relu(ref, 0.01)
    tol = 2e-4 * max(1.0, ref.abs().max().item())
    assert (outs[0] - ref.float()).abs().max().item() < tol
    assert (outs[1] - ref.float()).abs().max().item() < tol
    # same interpolation arithmetic, same products: the two paths agree to accumulation-order noise
    assert (outs[0] - outs[1]).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())


def test_row_kernel_64_wide_tile_on_plain_convolution():
    """The 64-output-channel tile of the row kernel (single accumulator set, N = 192 MMAs) is used by the net only for
    the fused decoder layers; vr_debug_set(2, 1) selects it for a plain TMA-fed convolution as well."""
    from lib import _native
    case = (2, 64, 16, 128, 64, 3, 1, (1, 1), 2)
    N, Cin, H, W, Cout, k, stride, dil, act = case
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    ref = _ref_conv(x, w, b, k, stride, dil, act)
    ctx.lib.vr_debug_set(2, 1)
    try:
        y = _run_debug_conv(ctx, x, w, b, k, stride, dil, act, 1)
    finally:
        ctx.lib.vr_debug_set(2, 0)
    err = (y - ref).abs().max().item()
    record_parity('conv_tc_rows64_%s' % '_'.join(str(v) for v in case).replace(' ', ''), err / max(1.0, ref.abs().max().item()), 2e-4)
    assert err < 2e-4 * max(1.0, ref.abs().max().item()), err
