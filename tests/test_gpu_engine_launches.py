"""vr_launch_count is "the number of kernels launched by this context" (include/vr_b200.h): over one library call its
increase must equal the number of kernels the CUDA profiler records for the call (memsets and copies not counted)."""
import json

import pytest
import torch

pytestmark = pytest.mark.gpu

SECONDS = 6.0   # 259 frames: 3 windows, and 4 more in the second pass of --tta


@pytest.fixture(scope='module')
def ctx():
    from lib import _native, synth
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    c = _native.Context(0, 2048, 1024, 32, 128, 256, 4)
    c.load_state_dict(synth.make_state_dict())
    yield c
    c.close()


def _counted_and_profiled(ctx, call, tmp_path):
    """(vr_launch_count increase, kernels in the profiler trace) over one call, after a first call outside the trace."""
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    before = ctx.launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    counted = ctx.launch_count() - before
    path = tmp_path / 'trace.json'
    prof.export_chrome_trace(str(path))
    with open(path) as f:
        kernels = [e['name'] for e in json.load(f)['traceEvents'] if e.get('cat') == 'kernel']
    return counted, kernels


@pytest.mark.parametrize('tta', [0, 1])
def test_separate_wave_launch_count(ctx, tta, tmp_path):
    from lib import _native, synth
    wave = torch.from_numpy(synth.sine_mix(SECONDS)).cuda()
    L = wave.shape[1]
    inst = torch.empty((2, 1024 * (L // 1024)), dtype=torch.float32, device='cuda')
    voc = torch.empty_like(inst)

    def call():
        ctx.check(ctx.lib.vr_separate_wave(ctx.handle, _native.ptr(wave), L, tta, _native.ptr(inst), _native.ptr(voc),
                                           _native.stream_ptr()), 'vr_separate_wave')

    counted, kernels = _counted_and_profiled(ctx, call, tmp_path)
    assert kernels, 'the profiler recorded no kernel'
    assert counted == len(kernels), (counted, sorted(set(kernels)))


def test_validation_loss_launch_count(ctx, tmp_path):
    from lib import _native
    g = torch.Generator(device='cuda').manual_seed(0)
    T = 300   # 3 windows of 128 frames
    x = torch.randn((2, 1025, T), dtype=torch.complex64, device='cuda', generator=g)
    y = torch.randn((2, 1025, T), dtype=torch.complex64, device='cuda', generator=g)
    coef = torch.empty(1, dtype=torch.float32, device='cuda')
    sums = torch.empty(3, dtype=torch.float64, device='cuda')

    def call():
        ctx.check(ctx.lib.vr_validation_loss(ctx.handle, _native.ptr(x), _native.ptr(y), T, _native.ptr(coef),
                                             _native.ptr(sums), _native.stream_ptr()), 'vr_validation_loss')

    counted, kernels = _counted_and_profiled(ctx, call, tmp_path)
    assert kernels, 'the profiler recorded no kernel'
    assert counted == len(kernels), (counted, sorted(set(kernels)))
