"""Four-warpgroup variants of the generic wgmma convolution (csrc/conv_tc.cu, DESIGN 5.3): two m-tiles per CTA sharing
the weights (PAIR_M, vr_debug_set(8, 2)) or both N tiles of a layer sharing the activations (PAIR_N, (8, 3)).  Every
accumulator receives its products in the order of the two-warpgroup kernel ((8, 1)), so the outputs must be bitwise
equal to it, for every generic-layer geometry of the default net, at batches 1, 2 and 27."""
import pytest
import torch

from test_gpu_parity import _ref_conv, _run_debug_conv

pytestmark = pytest.mark.gpu

GENERIC_CASES = [
    # Cin, H, W (input), Cout, k, stride, (dh, dw), act
    (32, 62, 256, 64, 3, 2, (1, 1), 2),      # enc2.conv1 class: W = 128 out, 31 rows (odd m-tile count at odd N)
    (16, 32, 256, 32, 3, 2, (1, 1), 2),      # stg1_low enc2.conv1: KB = 16
    (64, 32, 128, 128, 3, 2, (1, 1), 2),     # enc3.conv1 class: W = 64 out, two rows per tile, KB = 64
    (128, 16, 64, 192, 3, 2, (1, 1), 2),     # enc4.conv1 class: two N tiles of 96
    (192, 16, 32, 256, 3, 2, (1, 1), 2),     # enc5.conv1 class: W = 16 out, eight rows, two N tiles of 128
    (256, 64, 16, 256, 3, 1, (4, 2), 1),     # stage-3 ASPP conv3
    (128, 64, 16, 128, 3, 1, (8, 4), 1),     # stage-2 high / stage-1 low ASPP conv4
    (256, 64, 16, 256, 3, 1, (12, 6), 1),    # stage-3 ASPP conv5
    (256, 4, 16, 256, 3, 1, (4, 2), 1),      # four rows: two images stacked per 128-pixel tile (Nt = 2)
    (256, 64, 16, 256, 1, 1, (1, 1), 1),     # ASPP conv2 (1x1)
    (1280, 64, 16, 256, 1, 1, (1, 1), 1),    # ASPP bottleneck
    (256, 1, 16, 256, 1, 1, (1, 1), 1),      # ASPP conv1.1 on the pooled row: eight images per tile
    (16, 32, 256, 16, 1, 1, (1, 1), 1),      # stage bridge, BN = 16, KB = 16
]


def _case(case, N, seed):
    Cin, H, W, Cout, k, stride, dil, act = case
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    return x, w, b


@pytest.fixture(scope='module')
def ctx():
    from lib import _native
    c = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    yield c
    c.close()


@pytest.mark.parametrize('N', [1, 2, 27])
@pytest.mark.parametrize('case', GENERIC_CASES)
def test_paired_generic_kernel_is_bitwise_equal(ctx, case, N):
    Cin, H, W, Cout, k, stride, dil, act = case
    x, w, b = _case(case, N, 7 + Cin + 3 * H + W + N)
    ys = {}
    try:
        for key in (1, 2, 3, 0):   # two warpgroups, PAIR_M, PAIR_N (where Cout needs two N tiles), automatic
            assert ctx.lib.vr_debug_set(8, key) == 0
            ys[key] = _run_debug_conv(ctx, x, w, b, k, stride, dil, act, 1)
    finally:
        ctx.lib.vr_debug_set(8, 0)
    ref = _ref_conv(x, w, b, k, stride, dil, act)
    assert (ys[1] - ref).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())
    for key in (2, 3, 0):
        assert torch.equal(ys[key], ys[1]), (key, (ys[key] - ys[1]).abs().max().item())


def test_separate_10s_stems_identical_with_every_pairing():
    import inference
    from lib import _native, nets, synth
    m = nets.CascadedNet(2048, 1024, 32, 128)
    m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    m.to(torch.device('cuda:0'))
    wave = torch.from_numpy(synth.sine_mix(10.0)).cuda()
    sp = inference.Separator(m, torch.device('cuda:0'), 4, 256, False)
    lib = _native.load_library()
    stems = {}
    try:
        for key in (1, 0, 2, 3):
            assert lib.vr_debug_set(8, key) == 0
            inst, voc = sp.separate_wave(wave)
            stems[key] = (inst.cpu().numpy().tobytes(), voc.cpu().numpy().tobytes())
    finally:
        lib.vr_debug_set(8, 0)
    for key in (0, 2, 3):
        assert stems[key] == stems[1], key
