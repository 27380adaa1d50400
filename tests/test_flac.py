"""FLAC input: the oracle encoder / decoder (oracle/flac_oracle.py), the host side of lib/flac.py, the 24-bit WAV reader
(CPU), and the GPU decoder (csrc/flac.cu) against the oracle, through lib.flac, lib.audio_io and inference.py (gpu)."""
import os
import subprocess
import sys
import wave

import numpy as np
import pytest

from conftest import PKG, ROOT

sys.path.insert(0, ROOT)
from oracle import flac_oracle as fo  # noqa: E402


@pytest.fixture(scope='module')
def matrix():
    return fo.matrix_streams()


def _write_wav(path, x, bps, rate):
    """x: int (channels, n) -> PCM WAV of bps // 8 bytes per sample."""
    nb = bps // 8
    inter = np.ascontiguousarray(np.asarray(x, np.int64).T).reshape(-1).astype('<i4')
    with wave.open(str(path), 'wb') as f:
        f.setnchannels(x.shape[0])
        f.setsampwidth(nb)
        f.setframerate(rate)
        f.writeframes(inter.view(np.uint8).reshape(-1, 4)[:, :nb].tobytes())


def _tones(channels, n, bps, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    amp = (1 << (bps - 1)) * 0.4
    x = [amp * np.sin(2 * np.pi * (0.01 + 0.003 * c) * t) + rng.integers(-50, 51, n) for c in range(channels)]
    return np.clip(np.round(x), -(1 << (bps - 1)), (1 << (bps - 1)) - 1).astype(np.int64)


def _planted_stream():
    """8-bit mono, VERBATIM frames: frame 1's samples spell out frame 3's header (a sync pattern with a valid CRC-8 and
    another frame's number) and frame 2's samples a header claiming block size 192 of frame 0."""
    x = _tones(1, 192 * 6, 8, seed=3)
    x = np.clip(x, -100, 100)

    def frames():
        return [dict(bs=192, bs_code=1, rate_code=4, bps_code=1, subs=[dict(type='verbatim')]) for _ in range(6)]
    first, info = fo.encode(x, 8, 8000, frames(), id3='plain')
    planted = []
    for k, src in ((1, 3), (2, 0)):
        o = info['frame_offsets'][src]
        hdr = first[o:o + fo.parse_frame_header(first, o)['header_len']]
        at = k * 192 + 40
        x[0, at:at + len(hdr)] = [b - 256 if b >= 128 else b for b in hdr]
        planted.append((k, len(hdr)))
    data, info = fo.encode(x, 8, 8000, frames(), id3='plain')
    planted_offs = [info['frame_offsets'][k] + fo.parse_frame_header(data, info['frame_offsets'][k])['header_len'] + 1
                    + 40 for k, _ in planted]
    return data, x, info, planted_offs


# ---------------------------------------------------------------------------------------------------------------- CPU


def test_crc_catalogue_check_values():
    assert fo.crc8(b'123456789') == 0xF4          # CRC-8, poly 0x07
    assert fo.crc16(b'123456789') == 0xFEE8       # CRC-16/UMTS, poly 0x8005
    assert fo.crc16_many([b'123456789', b'12345678', b'']) == [0xFEE8, fo.crc16(b'12345678'), 0]


def test_matrix_covers_the_format(matrix):
    st = fo.merged_stats(matrix)
    kinds = st['kinds']
    assert {('constant', 0), ('verbatim', 0)} <= kinds
    assert {('fixed', o) for o in range(5)} <= kinds and {('lpc', o) for o in range(1, 33)} <= kinds
    assert st['precisions'] == set(range(1, 16)) and st['shifts'] == set(range(16))
    assert st['wasted'] >= {1, 2, 3}
    assert st['rice4'] and st['rice5'] and st['escape'] and st['escape_raw0']
    assert st['porders'] == set(range(16))
    assert st['modes'] >= {'independent', 8, 9, 10} | {'independent%d' % c for c in (1, 3, 4, 5, 6, 7, 8)}
    assert st['bs_codes'] == set(range(1, 16)) and st['rate_codes'] == set(range(15))
    assert st['bps_codes'] == {0, 1, 2, 4, 5, 6}
    assert {bps for _, _, bps, _, _ in matrix} == {8, 12, 16, 20, 24}
    variable = {bool(data[info['frame_offsets'][0] + 1] & 1) for data, *_, info in matrix}
    assert variable == {False, True}
    assert {data[:3] == b'ID3' for data, *_ in matrix} == {False, True}


def test_matrix_round_trips_through_the_oracle(matrix):
    for data, x, bps, rate, info in matrix:
        y, r, b = fo.decode(data)
        assert (r, b) == (rate, bps)
        assert np.array_equal(x, y)
        _, si = fo.read_streaminfo(data)
        assert si['md5'] == fo.md5_of(y, bps)


def test_host_metadata_matches_the_oracle(matrix):
    from lib import flac
    for data, x, bps, rate, info in matrix:
        start, si = flac.parse_metadata(data)
        assert start == info['audio_start']
        assert (si['rate'], si['channels'], si['bps'], si['total']) == (rate, x.shape[0], bps, x.shape[1])


def test_chain_finds_the_true_frames(matrix):
    from lib import flac
    for data, x, bps, rate, info in matrix:
        start, si = flac.parse_metadata(data)
        frames, total = flac.build_chain(fo.scan_candidates(data)[::-1], start, len(data), si)
        assert frames[:, 0].tolist() == info['frame_offsets'] and total == x.shape[1]


def test_chain_passes_over_planted_headers():
    from lib import flac
    data, x, info, planted = _planted_stream()
    cands = fo.scan_candidates(data)
    assert set(planted) <= set(cands[:, 0].tolist())             # the planted headers are candidates
    start, si = flac.parse_metadata(data)
    frames, total = flac.build_chain(cands, start, len(data), si)
    assert frames[:, 0].tolist() == info['frame_offsets'] and total == x.shape[1]
    y, _, _ = fo.decode(data)
    assert np.array_equal(y, x)


def _with_header_byte(data, info, k, byte, value):
    """The stream with byte `byte` of frame k's header set to `value` and the header's CRC-8 recomputed."""
    d = bytearray(data)
    o = info['frame_offsets'][k]
    hl = fo.parse_frame_header(data, o)['header_len']
    d[o + byte] = value
    d[o + hl - 1] = fo.crc8(d[o:o + hl - 1])
    return bytes(d)


@pytest.mark.parametrize('what, byte, fn', [
    ('block-size code 0000', 2, lambda b: b & 0x0F),
    ('sample-rate code 1111', 2, lambda b: b | 0x0F),
    ('channel assignment 11', 3, lambda b: (b & 0x0F) | 0xB0),
    ('sample-size code 011', 3, lambda b: (b & 0xF1) | 0x06),
    ('32-bit sample size', 3, lambda b: b | 0x0E),
    ('reserved bit', 3, lambda b: b | 0x01),
])
def test_host_rejects_reserved_codes(matrix, what, byte, fn):
    from lib import flac
    data, x, bps, rate, info = matrix[1]
    k = 1                                                     # sample-rate code 9: no coded rate bytes to lose
    bad = _with_header_byte(data, info, k, byte, fn(data[info['frame_offsets'][k] + byte]))
    start, si = flac.parse_metadata(bad)
    with pytest.raises(ValueError, match=r'<bytes>: frame %d \(byte %d\)' % (k, info['frame_offsets'][k])):
        flac.build_chain(fo.scan_candidates(bad), start, len(bad), si, '<bytes>')


def test_host_rejects_32_bit_and_non_flac(tmp_path):
    from lib import flac
    x = _tones(1, 64, 16)
    data, _ = fo.encode(x, 16, 44100, [dict(bs=64, bs_code=6, rate_code=9, bps_code=4,
                                            subs=[dict(type='verbatim')])])
    start, si = flac.parse_metadata(data)
    assert si['bps'] == 16
    p = data.index(b'fLaC') + 4 + 4 + 10                     # STREAMINFO's packed rate / channels / bps / total
    packed = int.from_bytes(data[p:p + 8], 'big')
    packed = (packed & ~(31 << 36)) | (31 << 36)              # 32 bits per sample
    bad = data[:p] + packed.to_bytes(8, 'big') + data[p + 8:]
    with pytest.raises(ValueError, match='32-bit'):
        flac.parse_metadata(bad)
    with pytest.raises(ValueError, match='32-bit'):
        flac.decode(bad)
    with pytest.raises(ValueError, match='not a FLAC stream'):
        flac.decode(b'RIFF\x24\0\0\0WAVEfmt ' + bytes(40))
    path = tmp_path / 'song.flac'
    path.write_bytes(b'ID3\x04\0\0\0\0\0\x02ab' + b'\xff\xfb\x90\x00' * 8)   # an MP3 behind an ID3 tag
    assert not flac.sniff(str(path))
    with pytest.raises(ValueError, match='song.flac: not a FLAC stream'):
        flac.decode(str(path))
    path.write_bytes(data)
    assert flac.sniff(str(path))


def test_24_bit_wav_loads_exactly(tmp_path):
    from lib import audio_io
    x = _tones(2, 5000, 24)
    x[0, :4] = [-(1 << 23), (1 << 23) - 1, -1, 1]
    path = tmp_path / 'stem24.wav'
    _write_wav(path, x, 24, 44100)
    y, sr = audio_io.load(str(path), sr=44100, mono=False)
    assert sr == 44100 and y.dtype == np.float32
    assert np.array_equal(y, x.astype(np.float32) / np.float32(1 << 23))


def test_flac_without_gpu_or_soundfile_says_why(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip('a CUDA device decodes FLAC')
    try:
        import soundfile  # noqa: F401
        pytest.skip('soundfile decodes FLAC')
    except ImportError:
        pass
    from lib import audio_io
    data, *_ = fo.matrix_streams()[0]
    path = tmp_path / 'a.flac'
    path.write_bytes(data)
    with pytest.raises(RuntimeError, match='FLAC file: decoding it needs a CUDA device'):
        audio_io.load(str(path), sr=None)


# ---------------------------------------------------------------------------------------------------------------- GPU


def _exact(y, x, bps):
    import torch
    assert isinstance(y, torch.Tensor) and y.is_cuda and y.dtype == torch.float32
    y = y.cpu().numpy()
    assert y.shape == x.shape
    assert np.array_equal(y, x.astype(np.float32) / np.float32(2.0 ** (bps - 1)))
    return np.round(y.astype(np.float64) * 2.0 ** (bps - 1)).astype(np.int64)


@pytest.mark.gpu
def test_gpu_decodes_every_matrix_stream(matrix):
    from lib import flac
    for data, x, bps, rate, info in matrix:
        y, r, b = flac.decode(data)
        assert (r, b) == (rate, bps)
        ints = _exact(y, x, bps)
        assert np.array_equal(ints, fo.decode(data)[0])
        assert fo.md5_of(ints, bps) == fo.read_streaminfo(data)[1]['md5']


@pytest.mark.gpu
def test_gpu_decodes_planted_headers_and_id3v1_trailer():
    from lib import flac
    data, x, info, _ = _planted_stream()
    _exact(flac.decode(data)[0], x, 8)
    _exact(flac.decode(data + b'TAG' + bytes(125))[0], x, 8)


@pytest.mark.gpu
def test_gpu_decodes_four_minute_track():
    from lib import flac, synth
    x = np.clip(np.round(synth.sine_mix(240.0).astype(np.float64) * 32768), -32768, 32767).astype(np.int64)
    data, info = fo.encode_long(x)
    y, rate, bps = flac.decode(data)
    assert (rate, bps) == (44100, 16)
    ints = _exact(y, x, 16)
    assert fo.md5_of(ints, 16) == fo.read_streaminfo(data)[1]['md5']
    assert ('lpc', 8) in info['stats']['kinds']               # FIXED orders 0-4 were tried per frame as well


@pytest.mark.gpu
def test_gpu_malformed_streams_raise_and_leave_the_decoder_usable(matrix):
    from lib import flac
    data, x, bps, rate, info = matrix[1]                      # stereo 16-bit, 8 frames
    offs = info['frame_offsets']
    k = 5
    with pytest.raises(ValueError, match=r'frame %d \(byte %d\)' % (k, offs[k])):
        flac.decode(data[:offs[k] + (offs[k + 1] - offs[k]) // 2])          # truncated inside frame k
    flipped = bytearray(data)
    flipped[(offs[3] + offs[4]) // 2] ^= 0x10                                # a residual bit of frame 3
    with pytest.raises(ValueError, match=r'frame 3 \(byte %d\)' % offs[3]):
        flac.decode(bytes(flipped))
    broken = bytearray(data)
    broken[offs[4] + 2] ^= 0x01                                              # frame 4's header fails its CRC-8
    with pytest.raises(ValueError, match=r'frame [34] \(byte'):
        flac.decode(bytes(broken))
    _exact(flac.decode(data)[0], x, bps)                                     # same process, a good stream


@pytest.mark.gpu
@pytest.mark.parametrize('bps', [16, 24])
@pytest.mark.parametrize('rate', [44100, 48000])
def test_gpu_audio_io_flac_equals_wav(tmp_path, bps, rate):
    from lib import audio_io
    x = _tones(2, int(rate * 1.5), bps, seed=bps + rate)
    data, _ = fo.encode_long(x, bps=bps, rate=rate)
    (tmp_path / 'a.flac').write_bytes(data)
    _write_wav(tmp_path / 'a.wav', x, bps, rate)
    yf, srf = audio_io.load(str(tmp_path / 'a.flac'), sr=44100, mono=False)
    yw, srw = audio_io.load(str(tmp_path / 'a.wav'), sr=44100, mono=False)
    assert srf == srw == 44100 and yf.dtype == yw.dtype == np.float32 and yf.shape == yw.shape
    assert np.array_equal(yf, yw)
    if rate == 44100:
        assert np.array_equal(yf, x.astype(np.float32) / np.float32(2.0 ** (bps - 1)))
    mf, _ = audio_io.load(str(tmp_path / 'a.flac'), sr=44100, mono=True)
    mw, _ = audio_io.load(str(tmp_path / 'a.wav'), sr=44100, mono=True)
    assert np.array_equal(mf, mw)


@pytest.mark.gpu
def test_gpu_inference_cli_flac_equals_wav(tmp_path):
    import torch
    from lib import synth
    x = _tones(2, 44100 * 3, 16, seed=7)
    data, _ = fo.encode_long(x)
    (tmp_path / 'in_flac').mkdir()
    (tmp_path / 'in_wav').mkdir()
    (tmp_path / 'in_flac' / 'mix.flac').write_bytes(data)
    _write_wav(tmp_path / 'in_wav' / 'mix.wav', x, 16, 44100)
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
    outs = []
    for src in ('in_flac/mix.flac', 'in_wav/mix.wav'):
        out = tmp_path / ('out_' + src[3:7])
        r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt,
                            '-i', str(tmp_path / src), '-o', str(out)], capture_output=True, text=True, cwd=PKG)
        assert r.returncode == 0, r.stderr
        outs.append({f: (out / f).read_bytes() for f in sorted(os.listdir(out))})
    assert sorted(outs[0]) == ['mix_Instruments.wav', 'mix_Vocals.wav']
    assert outs[0] == outs[1]


@pytest.mark.gpu
def test_gpu_matches_libflac_through_soundfile(tmp_path):
    try:
        import soundfile as sf
    except ImportError:
        pytest.skip('soundfile is not installed: parity with libFLAC is unpinned here')
    from lib import flac
    for bps, subtype in ((16, 'PCM_16'), (24, 'PCM_24')):
        x = _tones(2, 30000, bps, seed=bps)
        path = str(tmp_path / ('lib%d.flac' % bps))
        sf.write(path, x.T.astype(np.float64) / 2.0 ** (bps - 1), 44100, format='FLAC', subtype=subtype)
        ref, _ = sf.read(path, dtype='float32', always_2d=True)
        y, rate, b = flac.decode(path)
        assert (rate, b) == (44100, bps)
        assert np.array_equal(y.cpu().numpy(), np.ascontiguousarray(ref.T))
