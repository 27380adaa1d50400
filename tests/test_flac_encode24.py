"""24-bit output (--output_bits 24): the host side of lib.flac / lib.audio_io / the CLI flag (CPU), and the GPU encoder
and PCM packer at 24 bits (csrc/flac_encode.cu) decoded by the oracle and by the GPU decoder, the range corners 16-bit
data never reached, and the 16-bit streams pinned to the bytes they had before the sample width became a parameter (gpu)."""
import hashlib
import os
import subprocess
import sys
import wave

import numpy as np
import pytest

from conftest import PKG, ROOT

sys.path.insert(0, ROOT)
from oracle import flac_oracle as fo  # noqa: E402

HEADER = 42   # fLaC + one STREAMINFO block


def q24(x):
    """The 24-bit integers of every writer: clip(rint(x * 8388607)) with the product in fp32, NaN -> 0."""
    v = np.rint(np.asarray(x, np.float32) * np.float32(8388607))
    return np.clip(np.where(np.isnan(v), np.float32(0), v), -8388608, 8388607).astype(np.int64)


def q16(x):
    v = np.rint(np.asarray(x, np.float32) * np.float32(32767))
    return np.clip(np.where(np.isnan(v), np.float32(0), v), -32768, 32767).astype(np.int64)


def _host_inputs():
    """name -> float32 (channels, n), seeded; the inputs that need no GPU to make."""
    from lib import synth
    rng = np.random.default_rng(24)
    n = 3 * 4096 + 37
    t = np.arange(n)
    return {
        'sine_mix': synth.sine_mix(10.0),
        'noise': rng.uniform(-1.0, 1.0, (2, n)).astype(np.float32),
        'silence': np.zeros((2, n), np.float32),
        'dc': np.full((2, n), 0.25, np.float32),
        'mono': (0.5 * np.sin(2 * np.pi * 0.01 * t) + 0.01 * rng.standard_normal(n)).astype(np.float32)[None],
        'len8229': synth.sine_mix(1.0)[:, :4096 * 2 + 37].copy(),
        'len11': synth.sine_mix(1.0)[:, :11].copy(),
    }


def _separator():
    import torch
    import inference
    from lib import nets, synth
    dev = torch.device('cuda:0')
    model = nets.CascadedNet(2048, 1024, 32, 128)
    model.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict()))
    model.to(dev)
    return inference.Separator(model, dev, 4, 256, False)


def _inputs():
    """The host inputs and the two stems of the 10 s mix from the seeded checkpoint."""
    import torch
    out = _host_inputs()
    inst, voc = _separator().separate_wave(torch.from_numpy(out['sine_mix']).cuda())
    out['instruments'], out['vocals'] = inst.cpu().numpy(), voc.cpu().numpy()
    return out


def _corners():
    """Inputs whose 24-bit integers reach what 16-bit data never did."""
    n = 4096 + 500
    t = np.arange(n)
    alt = np.where(t % 2 == 0, 1.0, -1.0).astype(np.float32)
    flip = np.where((t // 64) % 2 == 0, 1.0, -1.0).astype(np.float32)
    wild = np.zeros((2, 300), np.float32)
    wild[0, 10], wild[0, 20], wild[0, 30] = np.nan, np.inf, -np.inf
    wild[1, 5], wild[1, 6], wild[1, 7] = 2.0, -2.0, 1.0000001
    rng = np.random.default_rng(5)
    sixteen = (rng.integers(-32768, 32768, (2, n)) * 256 / 8388607.0).astype(np.float32)
    return {
        'side_extremes': np.stack([alt, -alt]),              # S = L - R = +-16777214, alternating per sample
        'side_extremes_clipped': np.stack([2 * flip, -2 * flip]),   # clipped to -8388608: S = +-16777215, all 25 bits
        'nyquist_square': np.stack([alt, alt]),
        'nyquist_square_antiphase': np.stack([2 * alt, -2 * alt]),
        'non_finite': wild,
        'low_byte_zero': sixteen,
    }


def _ckpt(tmp_path):
    import torch
    from lib import synth
    path = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), path)
    return path


def _flac24_input(tmp_path):
    """ten_seconds.flac: the 10 s mix as a 24-bit FLAC written by the oracle encoder."""
    from lib import synth
    data, _ = fo.encode_long(q24(synth.sine_mix(10.0)), bps=24)
    path = tmp_path / 'ten_seconds.flac'
    path.write_bytes(data)
    return str(path)


def _cli(tmp_path, ckpt, src, out, *extra):
    r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt, '-i', src,
                        '-o', str(tmp_path / out)] + list(extra), capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 0, r.stderr
    return {f: (tmp_path / out / f).read_bytes() for f in sorted(os.listdir(tmp_path / out))}


def _wav24_ints(path):
    with wave.open(str(path), 'rb') as f:
        assert f.getsampwidth() == 3
        raw = np.frombuffer(f.readframes(f.getnframes()), np.uint8).reshape(-1, 3).astype(np.int32)
        nch = f.getnchannels()
    v = (raw[:, 0] | (raw[:, 1] << 8) | (raw[:, 2] << 16)) << 8 >> 8
    return v.reshape(-1, nch).T.astype(np.int64)


# SHA-256 of flac.encode(x, 44100) of every _inputs() entry, and of the two stems `inference.py -i ten_seconds.flac
# --output_format flac` writes, recorded on an H100 before the encoder kernels took the sample width as a parameter
DIGESTS16 = {
    'sine_mix': '42ed12f9060332564959b561375a46a1ba097a9239b0b1cf1c5f8babef7332c0',
    'noise': 'bc20709200aff0863dcf99b777ff95424a2bb321611254f15fb11499c8bc100e',
    'silence': 'e28c79a57b9ee052127e5aeda25df3f15d39a03237b417ce7778ea899a39fcd1',
    'dc': '21e84870023e415c185027d1efc690ad63a7c53b8976610e14ec75674451a592',
    'mono': '14537025a6f8b340e0f03f033d6224a6312f520347198b7451cb07058498e4ee',
    'len8229': '8c40f95aeb56c4dc7a909e76d921dea7b26fbd12fa74e015e12bc6d575bcab42',
    'len11': 'b7c5fc03aed2639f8004fa2aedcf67c5e95f004706f0b9d78a639980ef02a5e7',
    'instruments': 'ae19818549e5c74b4b3414762988defc11f08b3404ded6aeea52ce1b397a8e00',
    'vocals': 'e7276f3aa78eeb056a4c3e4c3c8c619277bd653e3da81a97fa995bf2a9860ef9',
}
CLI_DIGESTS16 = {
    'Instruments': 'c5b8e6e518844a31c35adad0ae0182964128c29136e7aa6554bd8242a8cf0cfa',
    'Vocals': '0b79f8a9b9c862e25ac64486216bbc20be949244db7fd8f817af894744aad518',
}


# ---------------------------------------------------------------------------------------------------------------- CPU


@pytest.mark.parametrize('channels, n', [(1, 1), (2, 11), (2, 4096), (1, 4097), (2, 4096 * 3 + 37)])
def test_streaminfo_24_matches_the_oracle(channels, n):
    from lib import flac
    rng = np.random.default_rng(n)
    x = rng.integers(-8388608, 8388608, (channels, n))
    frames = [dict(bs=min(flac.BLOCK, n - i), bs_code=7, rate_code=9, bps_code=6, mode=fo.CH_INDEPENDENT,
                   subs=[dict(type='fixed', order=1, porder=0)] * channels) for i in range(0, n, flac.BLOCK)]
    for f in frames:
        if f['bs'] < 2:
            f['subs'] = [dict(type='verbatim')] * channels
    fb, _ = fo.encode_frames(x, 24, 44100, frames, False)
    ref = fo.metadata(x, 24, 44100, frames, fb, extra_blocks=False)
    got = flac.stream_header(channels, n, 44100, [len(b) for b in fb], fo.md5_of(x, 24), bits=24)
    assert got == ref and len(got) == HEADER
    y, rate, bps = fo.decode(got + b''.join(fb))
    assert (rate, bps) == (44100, 24) and np.array_equal(y, x)
    sixteen = flac.stream_header(channels, n, 44100, [len(b) for b in fb], fo.md5_of(x, 24))   # the default stays 16
    assert fo.read_streaminfo(sixteen)[1]['bps'] == 16


@pytest.mark.parametrize('name', ['x.wav', 'x.flac'])
def test_write_rejects_other_widths_before_creating_the_file(tmp_path, name):
    from lib import audio_io
    path = tmp_path / name
    for bits in (20, 8, 32, 0):
        with pytest.raises(ValueError, match='16 or 24'):
            audio_io.write(str(path), np.zeros((100, 2), np.float32), 44100, bits=bits)
    assert not path.exists()


def test_cli_output_bits_flag():
    import inference
    parser = inference.build_parser()
    assert parser.parse_args(['-i', 'a.wav']).output_bits == 16
    assert parser.parse_args(['-i', 'a.wav', '--output_bits', '16']).output_bits == 16
    assert parser.parse_args(['-i', 'a.wav', '--output_bits', '24', '--output_format', 'flac']).output_bits == 24
    for bad in ('20', '32', 'float'):
        with pytest.raises(SystemExit):
            parser.parse_args(['-i', 'a.wav', '--output_bits', bad])
    out = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '--help'], capture_output=True, text=True,
                         cwd=PKG).stdout
    assert '--output_bits' in out and '--output_format' in out


def test_wav24_write_without_gpu_or_soundfile(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip('a CUDA device packs the samples')
    try:
        import soundfile  # noqa: F401
        pytest.skip('soundfile writes PCM_24')
    except ImportError:
        pass
    from lib import audio_io
    rng = np.random.default_rng(3)
    x = rng.uniform(-1.2, 1.2, (2, 5000)).astype(np.float32)
    x[0, 7], x[1, 8], x[1, 9] = np.nan, np.inf, -np.inf
    audio_io.write(str(tmp_path / 'x.wav'), x.T, 44100, bits=24)
    with wave.open(str(tmp_path / 'x.wav'), 'rb') as f:
        assert (f.getnchannels(), f.getsampwidth(), f.getframerate(), f.getnframes()) == (2, 3, 44100, 5000)
    assert np.array_equal(_wav24_ints(tmp_path / 'x.wav'), q24(x))
    audio_io.write(str(tmp_path / 'm.wav'), x[0], 44100, bits=24)   # (L,) is mono, as for soundfile.write
    assert np.array_equal(_wav24_ints(tmp_path / 'm.wav'), q24(x[:1]))
    y, rate = audio_io.load(str(tmp_path / 'x.wav'), sr=None)       # and the package's own reader takes it back
    assert rate == 44100 and np.array_equal(y, q24(x).astype(np.float32) / np.float32(8388608))


# ---------------------------------------------------------------------------------------------------------------- GPU


@pytest.fixture(scope='module')
def inputs():
    return _inputs()


@pytest.fixture(scope='module')
def encoded(inputs):
    import torch
    from lib import flac
    out = {}
    for name, x in inputs.items():
        d = torch.from_numpy(x).cuda()
        out[name] = (x, flac.encode(d, 44100, bits=24), flac.encode_frames(d, 44100, bits=24))
    return out


def _check_stream(name, x, data, fr=None):
    """The whole of check 4 for one stream: both decoders, the MD5, every frame header."""
    from lib import flac
    ints = q24(x)
    y, rate, bps = fo.decode(data)
    assert (rate, bps) == (44100, 24), name
    assert np.array_equal(y, ints), name
    assert fo.read_streaminfo(data)[1]['md5'] == fo.md5_of(ints, 24), name
    g, rate, bps = flac.decode(data)
    assert (rate, bps) == (44100, 24), name
    assert np.array_equal(g.cpu().numpy(), ints.astype(np.float32) / np.float32(8388608)), name
    p, k = HEADER, 0
    sizes = []
    while p < len(data):
        h = fo.parse_frame_header(data, p)
        assert h is not None and h['number'] == k, (name, k)
        assert h['bps_code'] == 6 and h['rate_code'] == 9 and not h['variable'], (name, k)
        last = (k + 1) * 4096 >= x.shape[1]
        assert h['bs'] == (x.shape[1] - k * 4096 if last else 4096), (name, k)
        assert (h['bs_code'] == 12) == (h['bs'] == 4096), (name, k)
        size = int(fr.sizes[k]) if fr is not None else None
        if size is None:                                   # without the plan: the next header is where this frame ends
            q = p + h['header_len']
            while q < len(data) and fo.parse_frame_header(data, q) is None:
                q += 1
            size = q - p
        sizes.append(size)
        p += size
        k += 1
    assert p == len(data) and k == (x.shape[1] + 4095) // 4096, name
    if fr is not None:
        assert fr.bits == 24 and sizes == fr.sizes.tolist(), name
        assert np.array_equal(fr.pcm.cpu().numpy().T.astype(np.int64), ints), name


@pytest.mark.gpu
def test_gpu_24_bit_round_trip_is_exact(encoded):
    for name, (x, data, fr) in encoded.items():
        assert data[HEADER:] == fr.body, name                # encode_frames found no non-zero status either
        _check_stream(name, x, data, fr)


@pytest.mark.gpu
def test_gpu_24_bit_range_corners():
    from lib import flac
    for name, x in _corners().items():
        _check_stream(name, x, flac.encode(x, 44100, bits=24), flac.encode_frames(x, 44100, bits=24))
    ints = q24(_corners()['side_extremes_clipped'])
    side = ints[0] - ints[1]
    assert side.max() == 16777215 and side.min() == -16777215          # both ends of 25 bits went through a frame
    w = q24(_corners()['non_finite'])
    assert (w[0, 10], w[0, 20], w[0, 30], w[1, 5], w[1, 6], w[1, 7]) == (0, 8388607, -8388608, 8388607, -8388608,
                                                                         8388607)
    assert not (q24(_corners()['low_byte_zero']) & 0xFF).any()


def _first_residual_fields(data, sizes):
    """Per frame, of its first subframe: (subframe type, residual method, first partition's parameter, raw bits of an
    escaped partition or None); FIXED / LPC subframes only."""
    d = bytes(data)
    p = HEADER
    out = []
    for size in sizes:
        h = fo.parse_frame_header(d, p)
        br = fo.BitReader(d[p:p + size], 8 * h['header_len'])
        assert br.read(1) == 0
        t = br.read(6)
        assert br.read(1) == 0
        if t >= 8:
            order = t - 8 if t < 32 else t - 31
            br.pos += order * (24 + (h['ch_code'] == 9))
            if t >= 32:
                prec = br.read(4) + 1
                br.pos += 5 + order * prec
            method = br.read(2)
            br.read(4)
            k = br.read(5 if method else 4)
            out.append((t, method, k, br.read(5) if k == (31 if method else 15) else None))
        else:
            out.append((t, None, None, None))
        p += size
    return out


@pytest.mark.gpu
def test_gpu_24_bit_residuals_use_wide_rice_parameters_and_escapes(encoded):
    """What 16-bit data hardly reached: Rice parameters above 14, which only the 5-bit method has (Gaussian noise at
    -26 dB: residuals near 2^19 with tails), escaped partitions with 20+ raw bits (uniform noise: raw bits beat any
    Rice code), and full-scale uniform noise, which nothing codes below VERBATIM."""
    from lib import flac
    rng = np.random.default_rng(7)
    n = 3 * 4096 + 37
    gauss = np.clip(rng.normal(0.0, 0.05, (2, n)), -1, 1).astype(np.float32)
    uniform = rng.uniform(-0.25, 0.25, (2, n)).astype(np.float32)
    seen = {}
    for name, x in (('gauss', gauss), ('uniform', uniform)):
        fr = flac.encode_frames(x, 44100, bits=24)
        _check_stream(name, x, flac.encode(x, 44100, bits=24), fr)
        seen[name] = _first_residual_fields(bytes(HEADER) + fr.body, fr.sizes.tolist())
    assert any(m == 1 and 15 <= k <= 30 for _, m, k, _ in seen['gauss']), seen['gauss']
    assert any(raw is not None and raw >= 20 for *_, raw in seen['uniform']), seen['uniform']
    x, data, fr = encoded['noise']
    assert all(t == 1 for t, *_ in _first_residual_fields(data, fr.sizes.tolist()))
    assert len(data) <= HEADER + 16 * len(fr.sizes) + q24(x).size * 3 + 8, 'noise costs no more than VERBATIM'


@pytest.mark.gpu
def test_gpu_24_bit_encode_is_deterministic(encoded):
    import torch
    from lib import flac
    for name in ('sine_mix', 'noise', 'len8229', 'vocals'):
        x, data, _ = encoded[name]
        assert flac.encode(torch.from_numpy(x).cuda(), 44100, bits=24) == data, name
        assert flac.encode(x, 44100, bits=24) == data, name               # a host array encodes the same
        assert flac.encode(x, 44100, None, True, 24) == data, name        # and bits is the fifth positional argument


@pytest.mark.gpu
def test_gpu_24_bit_streams_compress(encoded):
    for name in ('sine_mix', 'instruments', 'vocals'):
        x, data, _ = encoded[name]
        ints = q24(x)
        ref, _ = fo.encode_long(ints, bps=24)
        pcm = ints.size * 3
        print('FLAC24 %s: %d bytes, oracle encode_long %d bytes, %.4f of 24-bit PCM (oracle %.4f)'
              % (name, len(data), len(ref), len(data) / pcm, len(ref) / pcm))
        assert len(data) < pcm, name
        assert len(data) <= len(ref), name


@pytest.mark.gpu
def test_gpu_pcm_pack_and_wav24(tmp_path, inputs):
    import torch
    from lib import audio_io, flac
    for name in ('sine_mix', 'noise', 'mono', 'len11'):
        x = inputs[name]
        for dev_input in (False, True):
            data = torch.from_numpy(x).cuda().T if dev_input else x.T
            path = tmp_path / ('%s%d.wav' % (name, dev_input))
            audio_io.write(str(path), data, 44100, bits=24)
            with wave.open(str(path), 'rb') as f:
                assert (f.getnchannels(), f.getframerate(), f.getnframes()) == (x.shape[0], 44100, x.shape[1])
            got = _wav24_ints(path)
            assert np.array_equal(got, q24(x)), name
        g, _, bps = flac.decode(flac.encode(x, 44100, bits=24))            # WAV and FLAC hold the same integers
        assert bps == 24 and np.array_equal(got.astype(np.float32) / np.float32(8388608), g.cpu().numpy()), name
        b16 = flac.pcm_bytes(x, 16)
        assert bytes(b16) == np.ascontiguousarray(q16(x).T).astype('<i2').tobytes(), name
        b24 = flac.pcm_bytes(torch.from_numpy(x).cuda(), 24)
        assert hashlib.md5(bytes(b24)).digest() == fo.md5_of(q24(x), 24), name
    wild = _corners()['non_finite']
    audio_io.write(str(tmp_path / 'wild.wav'), wild.T, 44100, bits=24)
    assert np.array_equal(_wav24_ints(tmp_path / 'wild.wav'), q24(wild))
    audio_io.write(str(tmp_path / 'a.flac'), inputs['len8229'].T, 44100, bits=24)
    y, _, bps = fo.decode((tmp_path / 'a.flac').read_bytes())
    assert bps == 24 and np.array_equal(y, q24(inputs['len8229']))
    with pytest.raises(ValueError, match='16 or 24'):
        flac.encode(inputs['len11'], 44100, bits=20)
    with pytest.raises(ValueError, match='16 or 24'):
        flac.pcm_bytes(inputs['len11'], 32)


@pytest.mark.gpu
def test_gpu_16_bit_streams_did_not_move(inputs):
    import torch
    from lib import flac
    assert sorted(DIGESTS16) == sorted(inputs)
    for name, x in inputs.items():
        data = flac.encode(torch.from_numpy(x).cuda(), 44100)
        assert hashlib.sha256(data).hexdigest() == DIGESTS16[name], name
        assert flac.encode(x, 44100, None, True, 16) == data, name
        fr = flac.encode_frames(x, 44100)
        assert fr.bits == 16 and fr.pcm.dtype == torch.int16 and tuple(fr.pcm.shape) == x.shape[::-1], name


@pytest.mark.gpu
def test_gpu_inference_cli_output_bits(tmp_path):
    import torch
    from lib import audio_io
    ckpt, src = _ckpt(tmp_path), _flac24_input(tmp_path)
    flac24 = _cli(tmp_path, ckpt, src, 'flac24', '--output_format', 'flac', '--output_bits', '24')
    flac16 = _cli(tmp_path, ckpt, src, 'flac16', '--output_format', 'flac')
    wav24 = _cli(tmp_path, ckpt, src, 'wav24', '--output_bits', '24')
    assert sorted(flac24) == sorted(flac16) == ['ten_seconds_Instruments.flac', 'ten_seconds_Vocals.flac']
    assert sorted(wav24) == ['ten_seconds_Instruments.wav', 'ten_seconds_Vocals.wav']
    X, _ = audio_io.load(src, sr=44100)
    stems = _separator().separate_wave(torch.from_numpy(X).cuda())
    for stem, name in zip(stems, ('Instruments', 'Vocals')):
        _check_stream(name, stem.cpu().numpy(), flac24['ten_seconds_%s.flac' % name])
        assert np.array_equal(_wav24_ints(tmp_path / 'wav24' / ('ten_seconds_%s.wav' % name)), q24(stem.cpu().numpy())), name
        assert hashlib.sha256(flac16['ten_seconds_%s.flac' % name]).hexdigest() == CLI_DIGESTS16[name], name
