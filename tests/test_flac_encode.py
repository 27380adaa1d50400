"""FLAC output: STREAMINFO and stream assembly on the host (CPU), and the GPU encoder (csrc/flac_encode.cu through
lib.flac.encode, lib.audio_io.write and inference.py --output_format flac) decoded by the oracle and by the GPU decoder
(gpu)."""
import os
import subprocess
import sys
import wave

import numpy as np
import pytest

from conftest import PKG, ROOT

sys.path.insert(0, ROOT)
from oracle import flac_oracle as fo  # noqa: E402


def quantise(x):
    """The integers audio_io.write's WAV writer stores: clip(round(x * 32767)) on float32 data."""
    x = np.asarray(x, np.float32)
    return np.clip(np.round(x * np.float32(32767.0)), -32768, 32767).astype(np.int64)


def _inputs():
    """name -> float32 (channels, n), seeded."""
    from lib import synth
    rng = np.random.default_rng(11)
    n = 3 * 4096 + 37
    t = np.arange(n)
    square = np.where((t // 50) % 2 == 0, 1.0, -1.0).astype(np.float32)
    imp = np.zeros((2, n), np.float32)
    imp[0, ::997] = 0.9
    imp[1, 500::1499] = -0.7
    noise_ms = np.clip(rng.normal(0.0, 0.4, n), -1, 1).astype(np.float32)
    out = {
        'sine_mix': synth.sine_mix(2.0),
        'silence': np.zeros((2, n), np.float32),
        'dc': np.full((2, n), 0.25, np.float32),
        'noise': rng.uniform(-1.0, 1.0, (2, n)).astype(np.float32),
        'noise_antiphase': np.stack([noise_ms, -noise_ms]),
        'square_antiphase': np.stack([square, -square]),
        'impulses': imp,
        'mono': (0.5 * np.sin(2 * np.pi * 0.01 * t) + 0.01 * rng.standard_normal(n)).astype(np.float32)[None],
    }
    for length in (1, 11, 4096, 4097, 4096 * 2 + 37):
        out['len%d' % length] = synth.sine_mix(1.0)[:, :length].copy()
    return out


def walk(data):
    """Frame-by-frame walk of a stream from the end of its metadata: per frame its byte offset, number, channel code,
    header codes and every subframe's coding; checks CRC-8 (by parsing) and CRC-16."""
    d = bytes(data)
    p, si = fo.read_streaminfo(d)
    frames = []
    while p < len(d):
        h = fo.parse_frame_header(d, p)
        assert h is not None, 'no frame header at byte %d' % p
        br = fo.BitReader(d, 8 * (p + h['header_len']))
        extra = {8: [0, 1], 9: [1, 0], 10: [0, 1]}.get(h['ch_code'], [0] * si['channels'])
        subs = []
        for c in range(si['channels']):
            bps = 16 + extra[c]
            assert br.read(1) == 0
            t = br.read(6)
            assert br.read(1) == 0                            # no wasted bits
            sub = dict(type=t)
            if t == 0:
                br.read(bps)
            elif t == 1:
                br.pos += h['bs'] * bps
            else:
                order = t - 8 if t < 32 else t - 31
                sub['order'] = order
                br.pos += order * bps
                if t >= 32:
                    sub['precision'] = br.read(4) + 1
                    sub['shift'] = br.read_signed(5)
                    br.pos += order * sub['precision']
                sub['method'] = br.read(2)
                sub['porder'] = br.read(4)
                pbits, esc = (5, 31) if sub['method'] else (4, 15)
                params = []
                for q in range(1 << sub['porder']):
                    m = (h['bs'] >> sub['porder']) - (order if q == 0 else 0)
                    k = br.read(pbits)
                    params.append(k)
                    if k == esc:
                        raw = br.read(5)
                        br.pos += m * raw
                    else:
                        for _ in range(m):
                            br.unary()
                            br.pos += k
                sub['params'] = params
            subs.append(sub)
        br.align()
        e = br.pos // 8
        assert fo.crc16(d[p:e]) == int.from_bytes(d[e:e + 2], 'big')
        frames.append(dict(h, subs=subs, end=e + 2))
        p = e + 2
    return frames


# ---------------------------------------------------------------------------------------------------------------- CPU


@pytest.mark.parametrize('channels, n', [(1, 1), (2, 11), (2, 4096), (1, 4097), (2, 4096 * 3 + 37)])
def test_streaminfo_matches_the_oracle(channels, n):
    from lib import flac
    rng = np.random.default_rng(n)
    x = rng.integers(-32768, 32768, (channels, n))
    frames = [dict(bs=min(flac.BLOCK, n - i), bs_code=7, rate_code=9, bps_code=4, mode=fo.CH_INDEPENDENT,
                   subs=[dict(type='fixed', order=1, porder=0)] * channels) for i in range(0, n, flac.BLOCK)]
    for f in frames:
        if f['bs'] < 2:
            f['subs'] = [dict(type='verbatim')] * channels
    fb, _ = fo.encode_frames(x, 16, 44100, frames, False)
    ref = fo.metadata(x, 16, 44100, frames, fb, extra_blocks=False)
    got = flac.stream_header(channels, n, 44100, [len(b) for b in fb], fo.md5_of(x, 16))
    assert got == ref
    y, rate, bps = fo.decode(got + b''.join(fb))                 # the assembled stream decodes
    assert (rate, bps) == (44100, 16) and np.array_equal(y, x)


def test_rate_codes_stay_in_the_subset():
    from lib import flac
    assert flac.rate_code(44100) == (9, 0) and flac.rate_code(48000) == (10, 0)
    assert flac.rate_code(11000) == (12, 11)
    assert flac.rate_code(11025) == (13, 11025)
    assert flac.rate_code(100000) == (12, 100)
    assert flac.rate_code(200010) == (14, 20001)
    with pytest.raises(ValueError, match='cannot be coded'):
        flac.rate_code(100001)


def test_flac_write_without_gpu_or_soundfile_raises_and_leaves_no_file(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip('a CUDA device encodes FLAC')
    try:
        import soundfile  # noqa: F401
        pytest.skip('soundfile encodes FLAC')
    except ImportError:
        pass
    from lib import audio_io
    path = tmp_path / 'x.flac'
    with pytest.raises(RuntimeError, match='writing FLAC needs a CUDA device'):
        audio_io.write(str(path), np.zeros((100, 2), np.float32), 44100)
    assert not path.exists()


# ---------------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope='module')
def encoded():
    from lib import flac
    import torch
    out = {}
    for name, x in _inputs().items():
        d = torch.from_numpy(x).cuda()
        fr = flac.encode_frames(d, 44100)
        data = flac.encode(d, 44100)
        out[name] = (x, data, fr)
    return out


@pytest.mark.gpu
def test_gpu_round_trip_is_exact(encoded):
    from lib import flac
    for name, (x, data, fr) in encoded.items():
        ints = quantise(x)
        y, rate, bps = fo.decode(data)
        assert (rate, bps) == (44100, 16), name
        assert np.array_equal(y, ints), name
        assert fo.read_streaminfo(data)[1]['md5'] == fo.md5_of(ints, 16), name
        assert np.array_equal(fr.pcm.cpu().numpy().T.astype(np.int64), ints), name
        g, rate, bps = flac.decode(data)
        assert np.array_equal(g.cpu().numpy(), ints.astype(np.float32) / np.float32(32768)), name


@pytest.mark.gpu
def test_gpu_streams_are_in_the_subset_and_frames_end_where_the_scan_said(encoded):
    from lib import flac
    seen = dict(rice5=set(), side=set())
    for name, (x, data, fr) in encoded.items():
        frames = walk(data)
        head = len(flac.stream_header(fr.channels, fr.total, 44100, fr.sizes, bytes(16)))
        offsets = head + np.concatenate([[0], np.cumsum(fr.sizes)[:-1]])
        assert [f['offset'] for f in frames] == offsets.tolist(), name
        assert frames[-1]['end'] == len(data), name
        assert [f['number'] for f in frames] == list(range(len(frames))), name
        for f in frames:
            assert f['bs_code'] == (12 if f['bs'] == 4096 else (6 if f['bs'] <= 256 else 7))
            assert f['rate_code'] == 9 and f['bps_code'] == 4
            for s in f['subs']:
                if s['type'] >= 32:
                    assert s['order'] <= 12 and s['precision'] <= 15 and 0 <= s['shift'] <= 15
                if 'porder' in s:
                    assert s['porder'] <= 8
                    assert (f['bs'] >> s['porder']) > s['order']
                    if s['method'] == 1:
                        seen['rice5'].add(name)
            if f['ch_code'] >= 8:
                seen['side'].add(name)
        assert sum(len(f['subs']) for f in frames) == len(frames) * x.shape[0]
    assert seen['rice5'] & {'noise', 'noise_antiphase', 'square_antiphase'}, seen
    assert {'noise_antiphase', 'square_antiphase'} <= seen['side'], seen


@pytest.mark.gpu
def test_gpu_encode_is_deterministic(encoded):
    import torch
    from lib import flac
    for name in ('sine_mix', 'noise', 'square_antiphase', 'len8229'):
        x, data, _ = encoded[name]
        assert flac.encode(torch.from_numpy(x).cuda(), 44100) == data, name
        assert flac.encode(x, 44100) == data, name            # a host array encodes the same


@pytest.mark.gpu
def test_gpu_non_finite_samples():
    from lib import flac
    x = np.zeros((2, 300), np.float32)
    x[0, 10], x[0, 20], x[0, 30] = np.nan, np.inf, -np.inf
    x[1, 5], x[1, 6] = 2.0, -2.0
    y, _, _ = fo.decode(flac.encode(x, 44100))
    assert (y[0, 10], y[0, 20], y[0, 30], y[1, 5], y[1, 6]) == (0, 32767, -32768, 32767, -32768)
    assert np.count_nonzero(y) == 4


@pytest.mark.gpu
def test_gpu_compression_floor_four_minutes():
    import torch
    from lib import flac, synth
    mix = synth.sine_mix(240.0)
    inst, voc = _separator().separate_wave(torch.from_numpy(mix).cuda())
    for name, x in (('sine_mix', torch.from_numpy(mix).cuda()), ('instruments', inst), ('vocals', voc)):
        data = flac.encode(x, 44100)
        ints = quantise(x.cpu().numpy())
        ref, _ = fo.encode_long(ints)
        wav = 44 + ints.size * 2
        print('FLAC %s: %d bytes, oracle encode_long %d bytes, %.4f of the 16-bit WAV (oracle %.4f)'
              % (name, len(data), len(ref), len(data) / wav, len(ref) / wav))
        assert len(data) <= len(ref), name
        g, _, _ = flac.decode(data)
        assert np.array_equal(g.cpu().numpy(), ints.astype(np.float32) / np.float32(32768)), name


@pytest.mark.gpu
def test_gpu_audio_io_write_flac(tmp_path):
    from lib import audio_io
    x = _inputs()['sine_mix']
    audio_io.write(str(tmp_path / 'a.flac'), x.T, 44100)
    data = (tmp_path / 'a.flac').read_bytes()
    assert data[:4] == b'fLaC'
    assert np.array_equal(fo.decode(data)[0], quantise(x))


def _wav_ints(path):
    with wave.open(str(path), 'rb') as f:
        return np.frombuffer(f.readframes(f.getnframes()), '<i2').reshape(-1, f.getnchannels()).T.astype(np.int64)


@pytest.mark.gpu
def test_gpu_inference_cli_flac_output(tmp_path):
    import torch
    from lib import synth
    wav_in = tmp_path / 'mix.wav'
    x = quantise(synth.sine_mix(6.0))
    with wave.open(str(wav_in), 'wb') as f:
        f.setnchannels(2)
        f.setsampwidth(2)
        f.setframerate(44100)
        f.writeframes(np.ascontiguousarray(x.T).astype('<i2').tobytes())
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)

    def run(out, *extra):
        r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt, '-i', str(wav_in),
                            '-o', str(tmp_path / out)] + list(extra), capture_output=True, text=True, cwd=PKG)
        assert r.returncode == 0, r.stderr
        return {f: (tmp_path / out / f).read_bytes() for f in sorted(os.listdir(tmp_path / out))}

    flac_files = run('flac', '--output_format', 'flac')
    wav_files = run('wav')
    assert sorted(flac_files) == ['mix_Instruments.flac', 'mix_Vocals.flac']
    assert sorted(wav_files) == ['mix_Instruments.wav', 'mix_Vocals.wav']
    from lib import audio_io
    X, _ = audio_io.load(str(wav_in), sr=44100)   # the CLI's stems: the same checkpoint on the same wave
    stems = _separator().separate_wave(torch.from_numpy(X).cuda())
    for stem, name in zip(stems, ('Instruments', 'Vocals')):
        got = fo.decode(flac_files['mix_%s.flac' % name])[0]
        assert np.array_equal(got, quantise(stem.cpu().numpy())), name
        wav_ints = _wav_ints(tmp_path / 'wav' / ('mix_%s.wav' % name))
        diff = int(np.abs(got - wav_ints).max())
        print('CLI %s: FLAC vs WAV stem, max difference %d LSB' % (name, diff))
        assert diff == 0, name
    try:
        import cv2  # noqa: F401
    except ImportError:
        return
    img_flac = run('flac_it', '--output_format', 'flac', '-I', '-t')
    img_wav = run('wav_it', '-I', '-t')
    for name in ('mix_Instruments.jpg', 'mix_Vocals.jpg'):
        assert img_flac[name] == img_wav[name], name
    for name in ('Instruments', 'Vocals'):
        a = fo.decode(img_flac['mix_%s.flac' % name])[0]
        b = np.frombuffer(img_wav['mix_%s.wav' % name][44:], '<i2').reshape(-1, 2).T
        assert np.array_equal(a, b), name


def _separator():
    import torch
    import inference
    from lib import nets, synth
    dev = torch.device('cuda:0')
    model = nets.CascadedNet(2048, 1024, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    model.to(dev)
    return inference.Separator(model, dev, 4, 256, False)


@pytest.mark.gpu
def test_gpu_stream_reads_through_libflac(tmp_path):
    try:
        import soundfile as sf
    except ImportError:
        pytest.skip('soundfile is not installed: reading by libFLAC is unpinned here')
    from lib import flac
    for name, x in _inputs().items():
        path = str(tmp_path / (name + '.flac'))
        flac.encode(x, 44100, path)
        y, rate = sf.read(path, dtype='int16', always_2d=True)
        assert rate == 44100 and np.array_equal(y.T.astype(np.int64), quantise(x)), name
