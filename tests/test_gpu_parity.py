"""GPU parity tests (run on an H100): the CUDA path, called through the C ABI / the reference-shaped
Python surface, against the CPU oracle (oracle/) and the golden fixtures produced by the unmodified
reference (tests/golden, oracle/make_golden.py).

Tolerances (floating point path; BASELINE.json north_star): mask max-abs < 1e-3 vs the CPU fp32
reference; masked spectrogram compared in normalised units (|.| / max|X|) < 1e-3 (SURVEY 0.6).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import checksum, record_parity

pytestmark = pytest.mark.gpu

MASK_TOL = 1e-3


def _dev():
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def default_model():
    from lib import nets, synth
    m = nets.CascadedNet(2048, 1024, 32, 128)
    m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    m.to(_dev())
    return m


@pytest.fixture(scope='module')
def wave10():
    from lib import synth
    return synth.sine_mix(10.0)


def test_stft_matches_oracle_and_golden(wave10, golden_default):
    from lib import spec_utils
    from oracle import stft_oracle
    S = spec_utils.wave_to_spectrogram(wave10, 1024, 2048)
    R = stft_oracle.wave_to_spectrogram(wave10, 1024, 2048)
    assert S.shape == R.shape and S.dtype == np.complex64
    scale = np.abs(R).max()
    record_parity('stft_10s_relative_vs_oracle', np.abs(S - R).max() / scale, 5e-6)
    assert np.abs(S - R).max() / scale < 5e-6
    assert np.abs(S[:, ::16, :] - golden_default['X_sub']).max() / scale < 5e-6


def test_istft_matches_oracle_and_roundtrip(wave10):
    from lib import spec_utils
    from oracle import stft_oracle
    R = stft_oracle.wave_to_spectrogram(wave10, 1024, 2048)
    w = spec_utils.spectrogram_to_wave(R, 1024)
    wr = stft_oracle.spectrogram_to_wave(R, 1024)
    assert w.shape == wr.shape and w.dtype == np.float32
    record_parity('istft_10s_vs_oracle', np.abs(w - wr).max(), 5e-6)
    assert np.abs(w - wr).max() < 5e-6
    assert np.abs(w - wave10[:, :w.shape[1]]).max() < 5e-6
    w0 = spec_utils.spectrogram_to_wave(R[0], 1024)   # 2-D mono input (lib/spec_utils.py:158-159)
    assert w0.shape == (w.shape[1],) and np.abs(w0 - wr[0]).max() < 5e-6


def test_frame_ranges_match_the_whole_track_calls(wave10):
    """The shard-sized entry points of the multi-GPU path (vr_stft_range, vr_normaliser_range,
    vr_apply_mask_istft_range) on ONE GPU: frame ranges with odd starts and lengths that are not multiples of the four
    frames a CTA of the n_fft = 2048 kernels transforms, the last one ending at the track's end, must reproduce the
    whole-track calls exactly (the same kernels, other alignment / tail branches).  Every n_fft at hop n_fft / 2 (the
    radix-2 kernels and the n_fft = 2048 ones), and n_fft = 2048 at hop 512, where each output sample reads four
    frames and a range's first and last frames lie outside its own hops."""
    from lib import _native, spec_utils
    dev = _dev()
    L = wave10.shape[1]
    d_wave = torch.from_numpy(wave10).to(dev)
    st = _native.stream_ptr()
    g = torch.Generator(device=dev).manual_seed(5)
    for n_fft, hop in [(n, n // 2) for n in (64, 128, 256, 512, 1024, 2048, 4096)] + [(2048, 512)]:
        ctx = spec_utils._spectral_ctx(n_fft, hop)
        T = 1 + L // hop
        bins = n_fft // 2 + 1
        full = torch.empty((2, bins, T), dtype=torch.complex64, device=dev)
        ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(d_wave), L, _native.ptr(full), T, None, st), 'vr_stft')
        part = torch.zeros_like(full)
        ranges = ((0, 3), (3, 10), (10, 11), (11, T - 5), (T - 5, T))
        for a, b in ranges:
            ctx.check(ctx.lib.vr_stft_range(ctx.handle, _native.ptr(d_wave), L, _native.ptr(part), T, a, b, st),
                      'vr_stft_range')
        norm = torch.empty(1, device=dev)
        ctx.check(ctx.lib.vr_normaliser(ctx.handle, _native.ptr(full), T, 0, _native.ptr(norm), st), 'vr_normaliser')
        norms = torch.empty(len(ranges), device=dev)
        for i, (a, b) in enumerate(ranges):
            ctx.check(ctx.lib.vr_normaliser_range(ctx.handle, _native.ptr(full), T, a, b, _native.ptr(norms[i:]), st),
                      'vr_normaliser_range')
        mask = torch.rand((2, bins, T), device=dev, generator=g)
        Lo = hop * (T - 1)
        ia, va = torch.empty((2, Lo), device=dev), torch.empty((2, Lo), device=dev)
        ctx.check(ctx.lib.vr_apply_mask_istft(ctx.handle, _native.ptr(full), _native.ptr(mask), T, _native.ptr(ia),
                                              _native.ptr(va), st), 'vr_apply_mask_istft')
        ib, vb = torch.zeros_like(ia), torch.zeros_like(va)
        for k0, k1 in ((0, 1), (1, 6), (6, 7), (7, T - 4), (T - 4, T - 1)):
            ctx.check(ctx.lib.vr_apply_mask_istft_range(ctx.handle, _native.ptr(full), _native.ptr(mask), T, k0, k1,
                                                        _native.ptr(ib), _native.ptr(vb), st),
                      'vr_apply_mask_istft_range')
        torch.cuda.synchronize()
        diff = max((part - full).abs().max().item(), (norms.max() - norm[0]).abs().item(),
                   (ia - ib).abs().max().item(), (va - vb).abs().max().item())
        record_parity('frame_ranges_nfft%d_hop%d_vs_whole_track' % (n_fft, hop), diff, 0.0)
        assert torch.equal(torch.view_as_real(part), torch.view_as_real(full)), (n_fft, hop)
        # the whole-track normaliser is the largest of the ranges' (hypotf in both kernels, no rounding in a max)
        assert torch.equal(norms.max(), norm[0]), (n_fft, hop)
        assert torch.equal(ia, ib) and torch.equal(va, vb), (n_fft, hop)


def test_stft_ragged_and_small_fft():
    from lib import spec_utils
    from oracle import stft_oracle
    rng = np.random.default_rng(3)
    for n_fft, hop, L in ((512, 256, 5000), (2048, 1024, 1023), (2048, 1024, 2048), (1024, 256, 7777)):
        x = rng.standard_normal((2, L)).astype(np.float32)
        S = spec_utils.wave_to_spectrogram(x, hop, n_fft)
        R = stft_oracle.wave_to_spectrogram(x, hop, n_fft)
        assert S.shape == R.shape
        assert np.abs(S - R).max() / np.abs(R).max() < 5e-6
        if S.shape[2] > 1:
            w = spec_utils.spectrogram_to_wave(R, hop)
            wr = stft_oracle.spectrogram_to_wave(R, hop)
            assert np.abs(w - wr).max() < 1e-5


CONV_CASES = [
    # N, Cin, H, W, Cout, k, stride, (dh, dw), act
    (2, 2, 32, 32, 16, 3, 1, (1, 1), 1),
    (1, 10, 16, 48, 32, 3, 1, (1, 1), 1),
    (1, 16, 32, 32, 32, 3, 2, (1, 1), 2),
    (1, 64, 16, 16, 64, 3, 1, (4, 2), 1),
    (1, 64, 16, 16, 24, 3, 1, (12, 6), 1),
    (2, 48, 8, 16, 8, 1, 1, (1, 1), 1),
    (1, 25, 16, 32, 8, 3, 1, (1, 1), 0),
]


def _run_debug_conv(ctx, x, w, b, k, stride, dil, act, use_tc):
    from lib import _native
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    dx, dw, db = x.cuda(), w.cuda(), b.cuda()
    y = torch.empty((N, Cout, Ho, Wo), dtype=torch.float32, device='cuda')
    ctx.check(ctx.lib.vr_debug_conv(ctx.handle, _native.ptr(dx), N, Cin, H, W, _native.ptr(dw), _native.ptr(db), Cout,
                                    k, stride, dil[0], dil[1], act, use_tc, _native.ptr(y), _native.stream_ptr()),
              'vr_debug_conv')
    return y.cpu()


def _ref_conv(x, w, b, k, stride, dil, act):
    pad = (dil[0] * (k // 2), dil[1] * (k // 2))
    y = F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=pad, dilation=dil)
    if act == 1:
        y = F.relu(y)
    elif act == 2:
        y = F.leaky_relu(y, 0.01)
    return y.float()


@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_cuda_core_kernel_vs_torch(case):
    from lib import _native
    N, Cin, H, W, Cout, k, stride, dil, act = case
    g = torch.Generator().manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1, 1)
    y = _run_debug_conv(ctx, x, w, b, k, stride, dil, act, 0)
    ref = _ref_conv(x, w, b, k, stride, dil, act)
    # storage is split-bf16 (16-bit significand): ~1.5e-5 relative on inputs and outputs
    assert (y - ref).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())


def _first_window(wave10):
    from oracle import stft_oracle, separator_oracle
    X = stft_oracle.wave_to_spectrogram(wave10, 1024, 2048)
    pad_l, pad_r, roi = separator_oracle.make_padding(X.shape[2], 256, 64)
    Xp = np.pad(X, ((0, 0), (0, 0), (pad_l, pad_r)))
    Xp /= np.abs(X).max()
    return X, Xp


def test_predict_mask_and_forward_vs_oracle(default_model, wave10):
    from lib import synth
    from oracle import net_oracle
    _, Xp = _first_window(wave10)
    x = np.abs(np.stack([Xp[:, :, 128:384], Xp[:, :, 256:512]]))
    sd = synth.to_torch_state_dict(synth.make_state_dict())
    ref = net_oracle.forward(sd, torch.from_numpy(x))
    got = default_model.forward(torch.from_numpy(x).cuda()).cpu()
    assert got.shape == ref.shape == (2, 2, 1025, 256)
    record_parity('forward_2windows_mask_vs_oracle', (got - ref).abs().max().item(), MASK_TOL)
    assert (got - ref).abs().max().item() < MASK_TOL
    got_c = default_model.predict_mask(torch.from_numpy(x).cuda()).cpu()
    assert got_c.shape == (2, 2, 1025, 128)
    assert (got_c - ref[:, :, :, 64:-64]).abs().max().item() < MASK_TOL
    pred = default_model.predict(torch.from_numpy(x).cuda()).cpu()
    assert (pred - (torch.from_numpy(x) * ref)[:, :, :, 64:-64]).abs().max().item() < MASK_TOL


def test_separate_10s_vs_reference_golden(default_model, wave10, golden_default):
    import inference
    from oracle import stft_oracle
    g = golden_default
    X = stft_oracle.wave_to_spectrogram(wave10, 1024, 2048)
    sp = inference.Separator(default_model, _dev(), 4, 256, False)
    X_before = X.copy()
    y, v = sp.separate(X)
    assert np.array_equal(X, X_before)            # caller's array is not mutated (inference.py:73-74)
    assert y.dtype == np.complex64 and y.shape == X.shape and v.shape == X.shape
    absmax = float(g['absmax'])
    assert np.abs(y[:, ::16, :] - g['y_sub']).max() / absmax < MASK_TOL
    # mask recovered from y = mask * X where |X| is not tiny
    big = np.abs(X) > 1e-2 * absmax
    mask = np.real(y * np.conj(X)) / np.maximum(np.abs(X) ** 2, 1e-20)
    err = np.abs(mask[:, ::8, :] - g['mask_sub'])[big[:, ::8, :]].max()
    record_parity('separate_10s_y_spec_normalised_vs_reference_golden', np.abs(y[:, ::16, :] - g['y_sub']).max() / absmax, MASK_TOL)
    assert err < MASK_TOL
    assert np.abs(y + v - X).max() / absmax < 1e-6
    cs = checksum(y)
    assert abs(cs[2] - g['y_sum'][2]) / g['y_sum'][2] < 1e-3
    # waves through the device inverse STFT
    from lib import spec_utils
    wy = spec_utils.spectrogram_to_wave(y, 1024)
    assert np.abs(wy[:, ::16] - g['wave_inst_sub']).max() < 1e-3


def test_mask_10s_direct_and_tta_vs_golden(default_model, wave10, golden_default):
    import inference
    from lib import _native
    from oracle import stft_oracle
    g = golden_default
    X = stft_oracle.wave_to_spectrogram(wave10, 1024, 2048)
    sp = inference.Separator(default_model, _dev(), 3, 256, False)   # batch 3: 4 windows -> ragged last batch
    d_spec = torch.from_numpy(X).cuda()
    m = sp._mask_device(d_spec, False).cpu().numpy()
    record_parity('mask_10s_vs_reference_golden', np.abs(m[:, ::8, :] - g['mask_sub']).max(), MASK_TOL)
    assert np.abs(m[:, ::8, :] - g['mask_sub']).max() < MASK_TOL
    assert np.array_equal(m[:, 1024, :], m[:, 1023, :])           # replicate-padded Nyquist row (lib/nets.py:111-115)
    mt = sp._mask_device(d_spec, True).cpu().numpy()
    record_parity('mask_10s_tta_vs_reference_golden', np.abs(mt[:, ::8, :] - g['mask_tta_sub']).max(), MASK_TOL)
    assert np.abs(mt[:, ::8, :] - g['mask_tta_sub']).max() < MASK_TOL
    # the TTA normaliser is |lexicographic complex max| (SURVEY 0.8)
    ctx = sp._ctx()
    out = torch.zeros(1, device='cuda')
    ctx.check(ctx.lib.vr_normaliser(ctx.handle, _native.ptr(d_spec), X.shape[2], 1, _native.ptr(out),
                                    _native.stream_ptr()), 'vr_normaliser')
    assert abs(out.item() - abs(complex(g['tta_norm']))) < 1e-4 * abs(complex(g['tta_norm']))


def test_private_separate_matches_oracle(default_model, wave10):
    import inference
    _, Xp = _first_window(wave10)
    sp = inference.Separator(default_model, _dev(), 2, 256, False)
    m = sp._separate(Xp.astype(np.complex64), 128)
    from lib import synth
    from oracle import separator_oracle
    sd = synth.to_torch_state_dict(synth.make_state_dict())
    ref = separator_oracle._separate(sd, Xp.astype(np.complex64), 128, 2048, 256, 64, 2)
    assert m.shape == ref.shape
    assert np.abs(m - ref).max() < MASK_TOL


def test_separate_wave_fused_matches_staged(default_model, wave10, golden_default):
    import inference
    g = golden_default
    sp = inference.Separator(default_model, _dev(), 4, 256, False)
    inst, voc = sp.separate_wave(wave10)
    assert inst.shape == (2, 440320) and voc.shape == inst.shape
    record_parity('wave_10s_instruments_vs_reference_golden', np.abs(inst[:, ::16] - g['wave_inst_sub']).max(), 1e-3)
    record_parity('wave_10s_vocals_vs_reference_golden', np.abs(voc[:, ::16] - g['wave_voc_sub']).max(), 1e-3)
    assert np.abs(inst[:, ::16] - g['wave_inst_sub']).max() < 1e-3
    assert np.abs(voc[:, ::16] - g['wave_voc_sub']).max() < 1e-3
    d_inst, d_voc = sp.separate_wave(torch.from_numpy(wave10).cuda())
    assert np.abs(d_inst.cpu().numpy() - inst).max() < 1e-6
    # stems add up to the (round-tripped) mixture
    assert np.abs(inst + voc - wave10[:, :inst.shape[1]]).max() < 1e-4


def test_small_config_vs_reference_golden(golden_small):
    import inference
    from lib import nets, synth
    from oracle import stft_oracle
    m = nets.CascadedNet(512, 256, 16, 32)
    m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict(512, 16, 32)))
    m.to(_dev())
    X = stft_oracle.wave_to_spectrogram(synth.sine_mix(3.0), 256, 512)
    sp = inference.Separator(m, _dev(), 2, 192, False)
    mask = sp._mask_device(torch.from_numpy(X).cuda(), False).cpu().numpy()
    record_parity('mask_3s_small_config_vs_reference_golden', np.abs(mask[:, ::2, :] - golden_small['mask_sub']).max(), MASK_TOL)
    assert np.abs(mask[:, ::2, :] - golden_small['mask_sub']).max() < MASK_TOL


def test_load_state_dict_is_strict():
    from lib import nets, synth
    m = nets.CascadedNet(2048, 1024, 32, 128)
    sd = synth.to_torch_state_dict(synth.make_state_dict())
    bad = dict(sd)
    bad.pop('out.weight')
    with pytest.raises(RuntimeError):
        m.load_state_dict(bad)
    bad = dict(sd)
    bad['extra.weight'] = torch.zeros(1)
    with pytest.raises(RuntimeError):
        m.load_state_dict(bad)
    # the native library is strict on its own as well
    from lib import _native
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1)
    bad = dict(sd)
    bad.pop('aux_out.weight')
    with pytest.raises(_native.NativeError):
        ctx.load_state_dict(bad)


def test_context_without_weights():
    """A context whose weights were never finalized still runs the spectral calls (lib/spec_utils.py uses such
    contexts), and every call that runs the net fails with "weights not finalized"."""
    from lib import _native
    dev = _dev()
    ctx = _native.Context(0, 2048, 1024, 32, 128, 256, 1)
    st = _native.stream_ptr()
    L = 1024 * 20
    T = 1 + L // 1024
    wave = torch.randn((2, L), generator=torch.Generator().manual_seed(7)).to(dev)
    spec = torch.empty((2, 1025, T), dtype=torch.complex64, device=dev)
    back = torch.empty((2, 1024 * (T - 1)), device=dev)
    ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(wave), L, _native.ptr(spec), T, None, st), 'vr_stft')
    ctx.check(ctx.lib.vr_istft(ctx.handle, _native.ptr(spec), T, _native.ptr(back), st), 'vr_istft')
    torch.cuda.synchronize()
    assert (back - wave[:, :back.shape[1]]).abs().max().item() < 1e-4
    mag = torch.zeros((1, 2, 1025, 256), device=dev)
    mask = torch.empty((1, 2, 1025, 256), device=dev)
    assert ctx.lib.vr_forward(ctx.handle, _native.ptr(mag), 1, _native.ptr(mask), st) == -1
    assert ctx.lib.vr_last_error(ctx.handle) == b'weights not finalized'
    inst, voc = torch.empty_like(back), torch.empty_like(back)
    assert ctx.lib.vr_separate_wave(ctx.handle, _native.ptr(wave), L, 0, _native.ptr(inst), _native.ptr(voc), st) == -1
    assert ctx.lib.vr_last_error(ctx.handle) == b'weights not finalized'


@pytest.mark.parametrize('n_frames', [3, 128, 129, 256])
def test_edge_lengths_vs_oracle(default_model, n_frames):
    """Ragged / tiny / exactly-aligned tracks: make_padding corner cases (lib/dataset.py:198-205)."""
    import inference
    from lib import synth
    from oracle import separator_oracle, stft_oracle
    L = 1024 * (n_frames - 1) + 100
    wave = synth.sine_mix(L / 44100.0, seed=n_frames)[:, :L]
    X = stft_oracle.wave_to_spectrogram(wave, 1024, 2048)
    assert X.shape[2] == n_frames
    sd = synth.to_torch_state_dict(synth.make_state_dict())
    ref = separator_oracle.separate_mask(sd, X)
    sp = inference.Separator(default_model, _dev(), 4, 256, False)
    got = sp._mask_device(torch.from_numpy(X).cuda(), False).cpu().numpy()
    assert got.shape == ref.shape == (2, 1025, n_frames)
    record_parity('mask_edge_%d_frames_vs_oracle' % n_frames, np.abs(got - ref).max(), MASK_TOL)
    assert np.abs(got - ref).max() < MASK_TOL
    inst, voc = sp.separate_wave(wave)
    assert inst.shape == (2, 1024 * (n_frames - 1))
    assert np.abs(inst + voc - wave[:, :inst.shape[1]]).max() < 1e-4


@pytest.mark.parametrize('n_fft,hop,cropsize', [(1024, 256, 256), (4096, 1024, 256), (2048, 512, 144),
                                                (2048, 512, 320)])
def test_other_geometries_vs_oracle(n_fft, hop, cropsize):
    """Band heights 256 and 1024, and the cropsizes whose maps tile for no tensor-core kernel (144, the smallest legal
    one, keeps a 16-frame roi): the mask of a three-window track against the oracle, and separate_wave at a hop other
    than n_fft / 2, whose stems must add up to the input.  The oracle's mask one frame late must miss the mask gate by
    a wide factor, so the windows' placement is what the gate sees."""
    import inference
    from lib import nets, synth
    from oracle import separator_oracle, stft_oracle
    sd = synth.make_state_dict(n_fft, 32, 128)
    model = nets.CascadedNet(n_fft, hop, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(sd))
    model.to(_dev())
    roi = cropsize - 2 * 64
    n_frames = 2 * roi + 5
    L = hop * (n_frames - 1) + 100
    wave = synth.sine_mix(L / 44100.0 + 0.01, seed=n_fft + cropsize)[:, :L]
    X = stft_oracle.wave_to_spectrogram(wave, hop, n_fft)
    assert X.shape == (2, n_fft // 2 + 1, n_frames)
    ref = separator_oracle.separate_mask(synth.to_torch_state_dict(sd), X, n_fft=n_fft, cropsize=cropsize)
    sp = inference.Separator(model, _dev(), 2, cropsize, False)
    got = sp._mask_device(torch.from_numpy(X).cuda(), False).cpu().numpy()
    assert got.shape == ref.shape
    err = float(np.abs(got - ref).max())
    record_parity('mask_nfft%d_crop%d_vs_oracle' % (n_fft, cropsize), err, MASK_TOL)
    assert err < MASK_TOL
    assert np.abs(ref[..., 1:] - ref[..., :-1]).max() > 10 * MASK_TOL
    inst, voc = sp.separate_wave(wave)
    assert inst.shape == voc.shape == (2, hop * (n_frames - 1))
    recon = float(np.abs(inst + voc - wave[:, :inst.shape[1]]).max())
    record_parity('stems_sum_nfft%d_hop%d_crop%d_vs_input' % (n_fft, hop, cropsize), recon, 1e-4)
    assert recon < 1e-4


def test_full_size_track_properties(default_model):
    """BASELINE configs[2] size (4-minute track, 81 windows): size-independent properties of the path."""
    import inference
    from lib import synth
    wave = synth.sine_mix(240.0)
    sp = inference.Separator(default_model, _dev(), 16, 256, False)
    d_wave = torch.from_numpy(wave).cuda()
    inst, voc = sp.separate_wave(d_wave)
    assert inst.shape == (2, 1024 * (wave.shape[1] // 1024))
    # linearity of the inverse STFT: stems add up to the round-tripped mixture
    assert (inst + voc - d_wave[:, :inst.shape[1]]).abs().max().item() < 2e-4
    # window batching must not matter: batch 16 vs batch 5 (ragged last batch) agree to fp32 round-off
    sp5 = inference.Separator(default_model, _dev(), 5, 256, False)
    inst5, _ = sp5.separate_wave(d_wave)
    assert (inst - inst5).abs().max().item() < 1e-5
    # ... and neither must one batch holding the whole track (81 windows x 1024 rows exceeds 65535 grid rows)
    sp81 = inference.Separator(default_model, _dev(), 81, 256, False)
    inst81, _ = sp81.separate_wave(d_wave)
    assert (inst - inst81).abs().max().item() < 1e-5
    del sp81, sp5
    # the first 10 s see the same windows as the 10 s golden case except for the global normaliser, which is
    # identical here (same sine mix amplitude): compare the first two windows' worth of samples with the oracle
    assert torch.isfinite(inst).all() and torch.isfinite(voc).all()
    assert inst.abs().max().item() <= 1.5 * float(np.abs(wave).max())


def test_postprocess_device_matches_host_merge_artifacts(default_model):
    """--postprocess: device frame-min + weight apply == the host merge_artifacts (which tests/test_host_logic.py
    pins against the reference's lib/spec_utils.py:60-93)."""
    import inference
    from lib import _native, spec_utils
    rng = np.random.default_rng(5)
    T = 700
    m = rng.uniform(0.0, 0.04, size=(2, 1025, T)).astype(np.float32)
    for s, e in ((0, 90), (200, 330), (340, 500), (640, 700)):
        m[:, :, s:e] = rng.uniform(0.06, 1.0, size=(2, 1025, e - s))
    ref = spec_utils.merge_artifacts(m.copy())
    sp = inference.Separator(default_model, _dev(), 4, 256, True)
    ctx = sp._ctx()
    d_mask = torch.from_numpy(m).cuda()
    fmin = torch.empty(T, dtype=torch.float32, device='cuda')
    ctx.check(ctx.lib.vr_mask_frame_min(ctx.handle, _native.ptr(d_mask), T, _native.ptr(fmin), _native.stream_ptr()),
              'vr_mask_frame_min')
    assert np.array_equal(fmin.cpu().numpy(), m.min(axis=(0, 1)))
    w = torch.from_numpy(spec_utils.artifact_weights(fmin.cpu().numpy())).cuda()
    assert float(w.max()) == 1.0 and float(w.min()) == 0.0
    ctx.check(ctx.lib.vr_mask_apply_weight(ctx.handle, _native.ptr(d_mask), T, _native.ptr(w), _native.stream_ptr()),
              'vr_mask_apply_weight')
    assert np.abs(d_mask.cpu().numpy() - ref).max() < 1e-6
    # and the flag is wired through the Separator (no long above-threshold run in this track: identical result)
    from lib import synth
    wave = synth.sine_mix(4.0)
    a = sp.separate_wave(wave)[0]
    b = inference.Separator(default_model, _dev(), 4, 256, False).separate_wave(wave)[0]
    assert np.abs(a - b).max() < 1e-6


def test_zero_group_skipping_is_exact(default_model, wave10):
    """vr_debug_set key 6 (VR_KSKIP, on by default): the row kernel does not issue MMAs / interpolation for 8-channel
    input groups whose weights are all zero (lstm and pad groups of the concat layouts) - the skipped products are
    exact zeros, so switching it off may not change the mask by a single bit."""
    import inference
    from lib import _native
    from oracle import stft_oracle
    X = stft_oracle.wave_to_spectrogram(wave10, 1024, 2048)
    sp = inference.Separator(default_model, _dev(), 4, 256, False)
    d_spec = torch.from_numpy(X).cuda()
    lib = _native.load_library()
    base = sp._mask_device(d_spec, False).clone()
    lib.vr_debug_set(6, 0)
    try:
        for _ in range(3):   # repeated: a missing dependency would show up as run-to-run differences
            switched = sp._mask_device(d_spec, False).clone()
            assert torch.equal(base, switched)
    finally:
        lib.vr_debug_set(6, 1)


def test_silent_track_does_not_poison_the_context(default_model, wave10, golden_default):
    """A silent track has max|X| = 0: the normaliser guard packs zeros (finite mask) and, more importantly, nothing
    non-finite may survive in the shared activation buffers - the next track on the same Separator must be unaffected."""
    import inference
    sp = inference.Separator(default_model, _dev(), 4, 256, False)
    before, _ = sp.separate_wave(wave10)
    silent = np.zeros((2, 44100 * 3), dtype=np.float32)
    inst, voc = sp.separate_wave(silent)
    assert np.isfinite(inst).all() and np.isfinite(voc).all()
    assert np.abs(inst).max() == 0.0 and np.abs(voc).max() == 0.0
    bad = silent.copy()
    bad[0, 1000] = np.nan
    bad[1, 5000] = np.inf
    sp.separate_wave(bad)                       # whatever this returns, it must not leak into later calls
    after, _ = sp.separate_wave(wave10)
    assert np.isfinite(after).all()
    assert np.array_equal(before, after)


def test_pseudo_instruments_vs_oracle(default_model):
    """pseudo.py:56-71 (second caller of Separator.separate_tta): STFT of both tracks, separate_tta(X - y), y + a_spec,
    device-resident in PseudoLabeler, against the CPU oracle of the same steps."""
    import pseudo
    from lib import synth
    from oracle import separator_oracle, stft_oracle
    X = synth.sine_mix(5.0)
    y = (0.6 * X + 0.1 * synth.sine_mix(5.0, seed=3)).astype(np.float32)
    got = pseudo.PseudoLabeler(default_model, _dev(), 4, 256, False).pseudo_instruments(X, y)
    Xs = stft_oracle.wave_to_spectrogram(X, 1024, 2048)
    ys = stft_oracle.wave_to_spectrogram(y, 1024, 2048)
    sd = synth.to_torch_state_dict(synth.make_state_dict())
    a_spec, _ = separator_oracle.separate(sd, Xs - ys, tta=True)
    ref = ys + a_spec
    assert got.shape == ref.shape and got.dtype == np.complex64
    err = np.abs(got - ref).max() / np.abs(Xs - ys).max()
    record_parity('pseudo_instruments_5s_normalised_vs_oracle', err, MASK_TOL)
    assert err < MASK_TOL
