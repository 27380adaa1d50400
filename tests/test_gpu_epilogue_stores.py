"""16-byte epilogue stores of the three wgmma convolutions (epilogue_store, csrc/tc_common.cuh; DESIGN 5.2, 5.3, 5.7).

vr_debug_set(9, 1) makes every launch store channel pairs with epilogue_pair; the default (9, 0) stores 8 channels per
lane and plane where the output allows it.  Both write the same values, so the outputs must be bitwise equal: for the
row kernel at BN = 16 / 32 / 64, with and without the fused upsample, Cout = 8 on a BN = 16 tile and two N tiles; for
the halo kernel at every BN and MB = 1 / 2; for the generic kernel at BN = 16 and 48, paired and not; at batches 1 and
27.  The row kernel with the fused upsample and the halo kernel at BN = 128, MB = 2 store with epilogue_pixel8 (8-byte
stores) instead.  Cout values that are not a multiple of 8 exercise the sets that fall back to epilogue_pair."""
import pytest
import torch

from test_gpu_parity import _run_debug_conv

pytestmark = pytest.mark.gpu

# N is filled in by the batch parameter
ROW_CASES = [
    # Cin, H, W, Cout, act, rows_wide (vr_debug_set(2, .)): the row kernel's BN
    (32, 8, 128, 16, 1, 0),     # BN = 16 (R = 8)
    (16, 8, 128, 8, 0, 0),      # Cout = 8 on a BN = 16 tile: group 1 is not stored
    (64, 8, 256, 32, 2, 0),     # BN = 32 (R = 4), two column tiles
    (64, 8, 128, 64, 1, 0),     # BN = 32, two N tiles
    (32, 8, 128, 20, 1, 0),     # Cout = 20: the set of groups 0-3 straddles Cout
    (64, 8, 128, 64, 1, 1),     # BN = 64 (R = 2)
    (64, 8, 128, 128, 2, 1),    # BN = 64, two N tiles
]

DEC_CASES = [
    # Cl (low-res channels), h, w, Cs (skip channels), Cout, act
    (32, 4, 64, 16, 16, 1),     # BN = 16
    (32, 4, 64, 16, 8, 1),      # Cout = 8 on a BN = 16 tile
    (64, 4, 64, 32, 32, 1),     # BN = 32
    (64, 4, 64, 32, 64, 2),     # BN = 64 (the fused decoders' wide tile)
    (128, 4, 64, 64, 128, 1),   # BN = 64, two N tiles
    (32, 4, 64, 16, 20, 1),     # Cout = 20: the group pair 2-3 straddles Cout and takes epilogue_pair
    (64, 4, 64, 32, 40, 2),     # Cout = 40: the second N tile stores group 4 only
]

HALO_CASES = [
    # Cin, H, W, Cout, act: BN = round_up(Cout, 16) per N tile
    (32, 16, 64, 16, 1),
    (64, 16, 32, 32, 1),
    (64, 16, 16, 48, 2),
    (64, 16, 16, 36, 1),        # BN = 48, group 4 straddles Cout: the BN % 32 == 16 set falls back
    (64, 16, 64, 64, 1),
    (64, 16, 32, 192, 1),       # two N tiles of 96
    (96, 16, 16, 128, 0),
]

GENERIC_CASES = [
    # Cin, H, W (input), Cout, k, stride, (dh, dw), act
    (16, 32, 256, 16, 3, 2, (1, 1), 2),    # BN = 16
    (16, 64, 256, 8, 1, 1, (1, 1), 1),     # stage bridge class: BN = 16, Cout = 8
    (32, 32, 256, 48, 3, 2, (1, 1), 2),    # BN = 48
    (64, 16, 128, 40, 3, 2, (1, 1), 2),    # BN = 48, Cout = 40
]


def _tensors(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(*s, generator=g) for s in shapes]


def _conv(Cin, H, W, Cout, k, N, seed):
    x, w, b = _tensors([(N, Cin, H, W), (Cout, Cin, k, k), (Cout,)], seed)
    return x, w / (Cin * k * k) ** 0.5, b * 0.1


@pytest.fixture(scope='module')
def ctx():
    from lib import _native
    c = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 0)
    yield c
    c.close()


def _both(ctx, run):
    """run() under vr_debug_set(9, 1) and (9, 0)"""
    ys = {}
    try:
        for key in (1, 0):
            assert ctx.lib.vr_debug_set(9, key) == 0
            ys[key] = run()
    finally:
        ctx.lib.vr_debug_set(9, 0)
    return ys


def _assert_equal(ys):
    assert torch.isfinite(ys[1]).all()
    assert torch.equal(ys[0], ys[1]), (ys[0] - ys[1]).abs().max().item()


@pytest.mark.parametrize('N', [1, 27])
@pytest.mark.parametrize('case', ROW_CASES)
def test_row_kernel_stores(ctx, case, N):
    Cin, H, W, Cout, act, wide = case
    x, w, b = _conv(Cin, H, W, Cout, 3, N, 3 + Cin + Cout + N)
    ctx.lib.vr_debug_set(2, wide)
    try:
        ys = _both(ctx, lambda: _run_debug_conv(ctx, x, w, b, 3, 1, (1, 1), act, 1))
    finally:
        ctx.lib.vr_debug_set(2, 0)
    _assert_equal(ys)


@pytest.mark.parametrize('fused', [0, 1])
@pytest.mark.parametrize('N', [1, 27])
@pytest.mark.parametrize('case', DEC_CASES)
def test_row_kernel_stores_with_fused_upsample(ctx, case, N, fused):
    from lib import _native
    Cl, h, w, Cs, Cout, act = case
    low, skip, wgt, b = _tensors([(N, Cl, h, w), (N, Cs, 2 * h, 2 * w), (Cout, Cl + Cs, 3, 3), (Cout,)], 5 + Cl + Cout)
    wgt = wgt / ((Cl + Cs) * 9) ** 0.5
    dl, ds, dw, db = low.cuda(), skip.cuda(), wgt.cuda(), b.cuda()

    def run():
        y = torch.empty((N, Cout, 2 * h, 2 * w), dtype=torch.float32, device='cuda')
        ctx.check(ctx.lib.vr_debug_decoder(ctx.handle, _native.ptr(dl), N, Cl, h, w, _native.ptr(ds), Cs,
                                           _native.ptr(dw), _native.ptr(db), Cout, act, fused, _native.ptr(y),
                                           _native.stream_ptr()), 'vr_debug_decoder')
        return y.cpu()

    _assert_equal(_both(ctx, run))


@pytest.mark.parametrize('mb', [2, 3])   # vr_debug_set(3, 2 / 3): MB = 1 / 2
@pytest.mark.parametrize('N', [1, 27])
@pytest.mark.parametrize('case', HALO_CASES)
def test_halo_kernel_stores(ctx, case, N, mb):
    Cin, H, W, Cout, act = case
    x, w, b = _conv(Cin, H, W, Cout, 3, N, 7 + Cin + Cout + W + N)
    ctx.lib.vr_debug_set(3, mb)
    try:
        ys = _both(ctx, lambda: _run_debug_conv(ctx, x, w, b, 3, 1, (1, 1), act, 1))
    finally:
        ctx.lib.vr_debug_set(3, 0)
    _assert_equal(ys)


@pytest.mark.parametrize('pair', [1, 2])   # vr_debug_set(8, 1 / 2): two warpgroups / PAIR_M
@pytest.mark.parametrize('N', [1, 27])
@pytest.mark.parametrize('case', GENERIC_CASES)
def test_generic_kernel_stores(ctx, case, N, pair):
    Cin, H, W, Cout, k, stride, dil, act = case
    x, w, b = _conv(Cin, H, W, Cout, k, N, 9 + Cin + Cout + H + N)
    ctx.lib.vr_debug_set(8, pair)
    try:
        ys = _both(ctx, lambda: _run_debug_conv(ctx, x, w, b, k, stride, dil, act, 1))
    finally:
        ctx.lib.vr_debug_set(8, 0)
    _assert_equal(ys)


def test_separate_10s_stems_identical_with_either_store():
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
        for key in (1, 0):
            assert lib.vr_debug_set(9, key) == 0
            inst, voc = sp.separate_wave(wave)
            stems[key] = (inst.cpu().numpy().tobytes(), voc.cpu().numpy().tobytes())
    finally:
        lib.vr_debug_set(9, 0)
    assert stems[0] == stems[1]
