"""The streamed end-to-end separation against the staged path, on tracks of several window batches (run on an H100).

Separator.separate_wave of a host wave (inference.py's CLI whenever there is no --postprocess and no
--wiener_iterations) calls vr_separate_wave_host, which writes the stems span by span: after each window batch of the
last pass it runs the masked inverse STFT of the output hops whose mask frames are all final, and copies them to the
host while the next batch runs.  The staged path (Separator._separate_wave_staged) computes the whole mask first, then
one masked inverse STFT.  Every output sample is the overlap-add, in frame order, of the same frames computed by the
same kernels in both (istft_ola_kernel sums frames t0..t1 of its sample whatever span it is launched for, and each
frame's transform does not depend on its neighbours), so the two must agree bit for bit.

A span flushed before the frames it reads are final reads what the mask workspace still holds: the previous track's
mask, or only the first pass of --tta.  So every streamed call here follows the separation of a different track on the
same Separator, the track is separated twice with different tracks before it, and every case has at least three window
batches.  The stems are also anchored in float64 to oracle/stft_oracle.py fed the GPU's own spectrogram and mask, at
the inverse-STFT gate of test_gpu_spectral_geometry.py, and the stems an early flush produces are shown to miss that
gate by a wide factor.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import PKG, record_parity
from test_gpu_spectral_geometry import ISTFT_GATE, NONVACUOUS, _check_inverse, _frame_scale, _istft_ratio, _ola_weight

pytestmark = pytest.mark.gpu

SR = 44100
# 777 frames: with cropsize 256 (roi 128) 7 windows, and 8 in the second pass of --tta; with cropsize 144 (roi 16) 49
# and 50.  So batch 3 always ends on a ragged batch, and batch 1 runs every window as a batch of its own.
FRAMES = 777
GEOMETRIES = [(2048, 1024), (2048, 512), (2048, 256), (2048, 769), (1024, 256), (4096, 1024), (2048, 2048)]
CROPSIZES = (256, 144)
BATCHES = (1, 3)


def _dev():
    assert torch.cuda.is_available(), 'gpu tests need a CUDA device'
    return torch.device('cuda:0')


def _cases():
    for n_fft, hop in GEOMETRIES:
        for cropsize in CROPSIZES:
            for batch in BATCHES:
                for tta in (False, True):
                    yield pytest.param(n_fft, hop, cropsize, batch, tta,
                                       id='nfft%d-hop%d-crop%d-batch%d-%s' % (n_fft, hop, cropsize, batch,
                                                                              'tta' if tta else 'plain'))


@pytest.fixture(scope='module')
def separator():
    """separator(n_fft, hop, cropsize, batch): a Separator over the seeded synthetic checkpoint of that n_fft; the
    model of the last (n_fft, hop) asked for is kept, so that its contexts are built once per geometry."""
    import inference
    from lib import nets, synth
    held = {}

    def make(n_fft, hop, cropsize, batch):
        if (n_fft, hop) not in held:
            held.clear()
            m = nets.CascadedNet(n_fft, hop, 32, 128)
            m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict(n_fft, 32, 128)))
            m.to(_dev())
            held[(n_fft, hop)] = m
        return inference.Separator(held[(n_fft, hop)], _dev(), batch, cropsize, False)

    yield make
    held.clear()


def _tracks(hop):
    """the track under test (FRAMES frames, a ragged last hop) and two tracks of the same length whose masks differ
    from its mask everywhere: white noise, and a loud square wave"""
    from lib import synth
    L = hop * (FRAMES - 1) + hop // 2
    track = synth.sine_mix(L / SR + 0.01, seed=hop)[:, :L]
    noise = 0.5 * np.random.default_rng(hop + 1).standard_normal((2, L)).astype(np.float32)
    t = np.arange(L, dtype=np.float64) / SR
    square = 0.9 * np.sign(np.sin(2 * np.pi * 97.0 * t[None, :] + np.array([[0.0], [1.0]]))).astype(np.float32)
    return track, (noise, square)


def _last_pass_windows(T, roi, tta):
    """windows of the pass whose batches flush spans (Engine::separate: T // roi + 1, one more for --tta's second)"""
    return T // roi + 1 + (1 if tta else 0)


def _spec_and_mask(sp, wave, tta):
    """the GPU's spectrogram (vr_stft) and final mask of a host wave, as _separate_wave_staged computes them"""
    from lib import _native
    ctx = sp._ctx()
    with torch.cuda.device(_dev()):
        w = torch.from_numpy(np.ascontiguousarray(wave)).to(_dev())
        T = 1 + w.shape[1] // sp.model.hop_length
        d_spec = torch.empty((2, sp.model.n_fft // 2 + 1, T), dtype=torch.complex64, device=_dev())
        ctx.check(ctx.lib.vr_stft(ctx.handle, _native.ptr(w), w.shape[1], _native.ptr(d_spec), T, None,
                                  _native.stream_ptr()), 'vr_stft')
        d_mask = sp._mask_device(d_spec, tta)
        return d_spec.cpu().numpy(), d_mask.cpu().numpy()


def _anchor(X, m, hop):
    """float64 stems of the oracle's inverse STFT of m X and (1 - m) X"""
    from oracle import stft_oracle
    X64 = X.astype(np.complex128)
    return stft_oracle.spectrogram_to_wave(m * X64, hop), stft_oracle.spectrogram_to_wave((1.0 - m) * X64, hop)


def _anchor_ratio(stems, ref, weight, dead, scale):
    for name, got, want in zip(('instruments', 'vocals'), stems, ref):
        _check_inverse(name, got, want, dead)
    return max(_istft_ratio(got, want, weight, scale) for got, want in zip(stems, ref))


def _differing(a, b):
    return int((a != b).sum())


@pytest.mark.parametrize('n_fft,hop,cropsize,batch,tta', list(_cases()))
def test_streamed_equals_staged(separator, n_fft, hop, cropsize, batch, tta):
    """Streamed stems (after another track, twice) == staged stems, bit for bit, and within the float64 gate; with
    images (batch 3, cropsize 256) the streamed images == vr_spec_image of the staged spectrogram and mask."""
    sp = separator(n_fft, hop, cropsize, batch)
    track, poisons = _tracks(hop)
    T = 1 + track.shape[1] // hop
    assert T == FRAMES
    windows = _last_pass_windows(T, cropsize - 2 * sp.offset, tta)
    assert -(-windows // batch) >= 3 and (batch == 1 or windows % batch), (windows, batch)
    images = batch == 3 and cropsize == 256

    staged = sp._separate_wave_staged(track, tta, images)
    X, m = _spec_and_mask(sp, track, tta)
    weight, dead = _ola_weight(n_fft, hop, T)
    ref = _anchor(X, m, hop)
    scale = _frame_scale(X)

    sp.separate_wave(poisons[0], tta=tta)
    first = sp.separate_wave(track, tta=tta)
    sp.separate_wave(poisons[1], tta=tta)
    second = sp.separate_wave(track, tta=tta, images=images)
    assert len(second) == (4 if images else 2)

    ratio = _anchor_ratio(first, ref, weight, dead, scale)
    tag = 'streamed_nfft%d_hop%d_crop%d_b%d_tta%d' % (n_fft, hop, cropsize, batch, tta)
    record_parity(tag + '_vs_float64', ratio, ISTFT_GATE)
    failed = []
    if not ratio <= ISTFT_GATE:
        failed.append('streamed stems vs float64: %.4g > gate %.4g' % (ratio, ISTFT_GATE))
    for i, name in enumerate(('instruments', 'vocals')):
        if not np.array_equal(first[i], staged[i]):
            failed.append('%s: %d samples differ from the staged stem' % (name, _differing(first[i], staged[i])))
        if not np.array_equal(first[i], second[i]):
            failed.append('%s: %d samples differ between two streamed calls after different tracks'
                          % (name, _differing(first[i], second[i])))
    if images:
        for i, name in ((2, 'instruments image'), (3, 'vocals image')):
            assert second[i].shape == staged[i].shape == (n_fft // 2 + 1, T, 3)
            if not np.array_equal(second[i], staged[i]):
                failed.append('%s: %d values differ from the staged image' % (name, _differing(second[i], staged[i])))
    assert not failed, '\n'.join(failed)


def _flush_spans(T, roi, batch, windows, lookahead):
    """(k0, k1, f) of every span a streamed call without --tta flushes: output hops [k0, k1) inverse-transformed once
    mask frames [0, f) are final, with hop k taken as finished once k + lookahead < f (Engine::separate_wave_host)"""
    finals = [min(T, (g0 + min(batch, windows - g0)) * roi) for g0 in range(0, windows, batch)]
    spans, k_done = [], 0
    for f in [f for f in finals if f > 0] + [T]:
        k1 = T - 1 if f >= T else f - lookahead
        if k1 > k_done:
            spans.append((k_done, k1, f))
            k_done = k1
    return spans


@pytest.mark.parametrize('cropsize,batch', [(256, 1), (256, 3), (144, 1), (144, 3)])
def test_early_flush_misses_the_float64_gate(separator, cropsize, batch):
    """At n_fft 2048, hop 512 an output hop reads two mask frames past its own index.  A flush that takes hop k as
    finished once frame k + 1 is (the rule that only holds for hop = n_fft / 2) reads, at the end of each span, frames
    the next batch has not written yet: there the mask workspace still holds the previous track's mask.  Those stems,
    built here in float64 from the staged mask with those frames taken from the noise track's mask, must miss the gate
    of test_streamed_equals_staged by NONVACUOUS times, and the streamed stems must pass it."""
    n_fft, hop = 2048, 512
    sp = separator(n_fft, hop, cropsize, batch)
    track, poisons = _tracks(hop)
    T = 1 + track.shape[1] // hop
    roi = cropsize - 2 * sp.offset
    X, m = _spec_and_mask(sp, track, False)
    _, m_stale = _spec_and_mask(sp, poisons[0], False)
    weight, dead = _ola_weight(n_fft, hop, T)
    ref = _anchor(X, m, hop)
    scale = _frame_scale(X)

    spans = _flush_spans(T, roi, batch, _last_pass_windows(T, roi, False), 1)
    assert len(spans) >= 3
    early = tuple(np.empty_like(r) for r in ref)
    frame = np.arange(T)
    for k0, k1, f in spans:
        stems = _anchor(X, np.where(frame < f, m, m_stale), hop)
        for out, s in zip(early, stems):
            out[:, hop * k0:hop * k1] = s[:, hop * k0:hop * k1]
    wrong = max(_istft_ratio(got, want, weight, scale) for got, want in zip(early, ref))

    sp.separate_wave(poisons[0])
    ratio = _anchor_ratio(sp.separate_wave(track), ref, weight, dead, scale)
    record_parity('streamed_nfft2048_hop512_crop%d_b%d_early_flush_variant' % (cropsize, batch), wrong)
    assert ratio <= ISTFT_GATE, 'streamed stems vs float64: %.4g > gate %.4g' % (ratio, ISTFT_GATE)
    assert wrong >= NONVACUOUS * ISTFT_GATE, 'early-flush variant only %.4g (needs >= %.4g)' % (
        wrong, NONVACUOUS * ISTFT_GATE)


def test_cli_hop512_writes_the_staged_stems(tmp_path):
    """inference.py -H 512 on a track of three window batches (the CLI's batch 4, cropsize 256: 10 windows) writes the
    WAVs the staged stems make through audio_io.write, byte for byte."""
    import inference
    from lib import audio_io, nets, synth
    hop, T = 512, 1200
    L = hop * (T - 1) + 100
    src = str(tmp_path / 'mix.wav')
    audio_io.write(src, synth.sine_mix(L / SR + 0.01, seed=7)[:, :L].T, SR)
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
    out = tmp_path / 'cli'
    r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt, '-i', src,
                        '-o', str(out), '-H', str(hop)], capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 0, r.stderr

    args = inference.build_parser().parse_args(['-P', ckpt, '-i', src, '-H', str(hop)])
    model = nets.CascadedNet(args.n_fft, args.hop_length, 32, 128)
    model.load_state_dict(torch.load(ckpt, map_location='cpu'))
    model.to(_dev())
    sp = inference.Separator(model, _dev(), args.batchsize, args.cropsize, args.postprocess)
    X, _ = audio_io.load(src, sr=SR, mono=False, dtype=np.float32, device=_dev())
    assert 1 + X.shape[1] // hop == T
    windows = _last_pass_windows(T, args.cropsize - 2 * sp.offset, False)
    assert -(-windows // args.batchsize) >= 3 and windows % args.batchsize, (windows, args.batchsize)
    inst, voc = sp._separate_wave_staged(X, False, False)
    ref = tmp_path / 'staged'
    ref.mkdir()
    audio_io.write(str(ref / 'mix_Instruments.wav'), inst.T, SR)
    audio_io.write(str(ref / 'mix_Vocals.wav'), voc.T, SR)
    for name in ('mix_Instruments.wav', 'mix_Vocals.wav'):
        assert (out / name).read_bytes() == (ref / name).read_bytes(), name
