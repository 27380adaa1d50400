"""Stage 3's dec1 computes only the frames the mask keeps and applies the network's output layer in its epilogue
(vr_debug_set key 7 = 1, the default).  Every kept pixel receives the same products in the same order as in the
full-width layer, and the epilogue repeats mask_out_kernel's arithmetic on the values the layer would have stored, so
the mask must be bit-identical to the one of the old path (key 7 = 0: dec1 over every frame into f3_, then
mask_out_kernel)."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_FFT, HOP, BINS = 2048, 1024, 1025
FUSED = 'stg3_full_band_net.dec1.conv1+up+mask'


def _context(nout=32, cropsize=256, max_batch=4):
    from lib import _native, synth
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    c = _native.Context(0, N_FFT, HOP, nout, 128, cropsize, max_batch)
    c.load_state_dict(synth.make_state_dict(N_FFT, nout, 128))
    return c


@pytest.fixture(scope='module')
def ctx():
    c = _context(max_batch=27)   # the benchmark's batch: 27 windows per forward
    yield c
    c.close()


def _both(ctx, call):
    """call() -> device tensor, run on the cropped path and on the old path: the two results as numpy arrays."""
    out = []
    for key in (1, 0):
        assert ctx.lib.vr_debug_set(7, key) == 0
        try:
            res = call()
            torch.cuda.synchronize()
        finally:
            ctx.lib.vr_debug_set(7, 1)
        out.append(res.cpu().numpy().copy())
    return out


def _layers(ctx, call):
    """names of the launches profiled over one call() on the default path"""
    ctx.check(ctx.lib.vr_profile_enable(ctx.handle, 1), 'vr_profile_enable')
    try:
        call()
        torch.cuda.synchronize()
        need = ctypes.c_int64(0)
        ctx.check(ctx.lib.vr_profile_dump(ctx.handle, None, 0, ctypes.byref(need)), 'vr_profile_dump')
        buf = ctypes.create_string_buffer(need.value)
        ctx.check(ctx.lib.vr_profile_dump(ctx.handle, buf, need.value, None), 'vr_profile_dump')
    finally:
        ctx.check(ctx.lib.vr_profile_enable(ctx.handle, 0), 'vr_profile_enable')
    return [ln.split()[0] for ln in buf.value.decode().splitlines()]


def _mag(N, W, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.rand((N, 2, BINS, W), dtype=torch.float32, device='cuda', generator=g)


def _spec(T, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn((2, BINS, T), dtype=torch.complex64, device='cuda', generator=g)


def _predict(ctx, mag, roi, cropped=True):
    from lib import _native
    N = mag.shape[0]
    mask = torch.empty((N, 2, BINS, roi), dtype=torch.float32, device='cuda')
    fn = ctx.lib.vr_predict_mask if cropped else ctx.lib.vr_forward

    def call():
        ctx.check(fn(ctx.handle, _native.ptr(mag), N, _native.ptr(mask), _native.stream_ptr()), 'vr_predict_mask')
        return mask

    return call


@pytest.mark.parametrize('N', [1, 27, 30])
def test_predict_mask(ctx, N):
    new, old = _both(ctx, _predict(ctx, _mag(N, 256, N), 128))
    assert np.array_equal(new, old)


def test_predict_mask_runs_the_cropped_layer(ctx):
    names = _layers(ctx, _predict(ctx, _mag(2, 256, 0), 128))
    assert FUSED in names and 'mask_out' not in names, sorted(set(names))


def test_forward_all_columns(ctx):
    call = _predict(ctx, _mag(3, 256, 1), 256, cropped=False)
    new, old = _both(ctx, call)
    assert np.array_equal(new, old)
    names = _layers(ctx, call)
    assert FUSED in names and 'mask_out' not in names, sorted(set(names))


@pytest.mark.parametrize('tta', [0, 1])
def test_separate_with_a_partial_last_window(ctx, tta):
    from lib import _native
    T = 300   # 3 windows of 128 kept frames, the last one partial
    spec = _spec(T, 2)
    mask = torch.empty((2, BINS, T), dtype=torch.float32, device='cuda')

    def call():
        ctx.check(ctx.lib.vr_separate(ctx.handle, _native.ptr(spec), T, tta, _native.ptr(mask), _native.stream_ptr()),
                  'vr_separate')
        return mask

    new, old = _both(ctx, call)
    assert np.array_equal(new, old)


def test_separate_windows_shifted_frame_range(ctx):
    """The second (--tta) pass of a window range as the multi-GPU path runs it: frame_shift = roi / 2, so window 0
    starts at mask frame -64, and the frames it reaches are averaged into what the mask already holds."""
    from lib import _native
    T = 450
    spec = _spec(T, 3)
    norm = torch.tensor([float(spec.abs().max())], dtype=torch.float32, device='cuda')
    g = torch.Generator(device='cuda').manual_seed(4)
    prior = torch.rand((2, BINS, T), dtype=torch.float32, device='cuda', generator=g)
    mask = torch.empty_like(prior)

    def call():
        mask.copy_(prior)
        ctx.check(ctx.lib.vr_separate_windows(ctx.handle, _native.ptr(spec), T, _native.ptr(norm), 64 + 64, 0, 4,
                                              _native.ptr(mask), T, 64, 1, _native.stream_ptr()),
                  'vr_separate_windows')
        return mask

    new, old = _both(ctx, call)
    assert np.array_equal(new, old)
    assert not np.array_equal(new, prior.cpu().numpy())


def test_validation_loss(ctx):
    from lib import _native
    T = 300
    x, y = _spec(T, 5), _spec(T, 6)
    coef = torch.empty(1, dtype=torch.float32, device='cuda')
    sums = torch.empty(3, dtype=torch.float64, device='cuda')

    def call():
        ctx.check(ctx.lib.vr_validation_loss(ctx.handle, _native.ptr(x), _native.ptr(y), T, _native.ptr(coef),
                                             _native.ptr(sums), _native.stream_ptr()), 'vr_validation_loss')
        return sums

    new, old = _both(ctx, call)
    assert np.array_equal(new, old)


def test_cropsize_384_two_kept_tiles_per_row():
    c = _context(cropsize=384)
    try:
        call = _predict(c, _mag(5, 384, 7), 256)
        new, old = _both(c, call)
        assert np.array_equal(new, old)
        names = _layers(c, call)
        assert FUSED in names and 'mask_out' not in names, sorted(set(names))
    finally:
        c.close()


def test_two_channel_tiles_keep_the_old_path():
    """nout = 64: dec1 has two N tiles of 32 channels, so no quad of lanes holds a whole pixel - dec1 writes f3_ and
    mask_out_kernel runs, whatever key 7 says."""
    c = _context(nout=64)
    try:
        call = _predict(c, _mag(2, 256, 8), 128)
        new, old = _both(c, call)
        assert np.array_equal(new, old)
        names = _layers(c, call)
        assert 'mask_out' in names and FUSED not in names, sorted(set(names))
    finally:
        c.close()
