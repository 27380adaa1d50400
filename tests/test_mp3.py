"""MP3 input: the oracle (oracle/mp3_oracle.py) against FFmpeg's mp3float, its encoder's round trip and its coverage,
the host side of lib/mp3.py (CPU), and the GPU decoder (csrc/mp3.cu) against the oracle, through lib.mp3,
lib.audio_io, inference.py and spec_utils.cache_or_load (gpu)."""
import os
import re
import subprocess
import sys
import wave

import numpy as np
import pytest

from conftest import PKG, ROOT

sys.path.insert(0, ROOT)
from oracle import ffmpeg_mp3 as ff  # noqa: E402
from oracle import mp3_oracle as mo  # noqa: E402
from oracle import mp3_tables as mt  # noqa: E402

# ISO/IEC 11172-4 "full accuracy", full scale +-1
MAX_BOUND = 2.0 ** -14
RMS_BOUND = 2.0 ** -15 / np.sqrt(12.0)


@pytest.fixture(scope='module')
def matrix():
    return mo.matrix()


def _snr(ref, y):
    return 10 * np.log10(np.sum(ref ** 2) / np.sum((y - ref) ** 2))


def _host_cands(data, start, end):
    """What vr_mp3_scan returns, computed with numpy."""
    d = np.frombuffer(data, np.uint8)
    i = np.flatnonzero((d[:-1] == 0xFF) & ((d[1:] & 0xE0) == 0xE0))
    i = i[(i >= start) & (i + 4 <= end)]
    words = [int.from_bytes(data[k:k + 4], 'big') for k in i]
    return np.stack([i, np.asarray(words, np.int64)], axis=1) if len(i) else np.zeros((0, 2), np.int64)


def _chain(data, name='<bytes>'):
    from lib import flac, mp3
    start = flac._id3_size(data)
    end = mp3.audio_end(data, start)
    return mp3.build_chain(_host_cands(data, start, end), start, end, name)


# ------------------------------------------------------------------------------------------------------------ oracle


def test_tables_are_complete_prefix_codes_and_match_the_kernel_copy():
    o = 0
    for size in mt.HUFF_SIZES:
        lens = mt.HUFF_LENGTHS[o:o + size * size]
        assert sum(2.0 ** -ln for ln in lens) == 1.0
        symbols = sorted(x << 4 | y for x in range(size) for y in range(size))
        assert sorted(mt.HUFF_SYMBOLS[o:o + size * size]) == symbols
        o += size * size
    assert o == len(mt.HUFF_LENGTHS) == len(mt.HUFF_SYMBOLS)
    assert sum(2.0 ** -ln for ln in mt.QUAD_A_LENGTHS) == 1.0
    src = open(os.path.join(PKG, 'csrc', 'mp3.cu')).read()

    def arr(name):
        body = re.search(name + r'\[\d+\] = \{([^}]*)\}', src).group(1)
        return [int(v) for v in body.replace('\n', ' ').split(',') if v.strip()]
    assert arr('kHuffSymbols') == list(mt.HUFF_SYMBOLS)
    assert arr('kHuffLengths') == list(mt.HUFF_LENGTHS)
    assert arr('kSynthWindow') == list(mt.SYNTH_WINDOW)


def test_matrix_covers_the_format(matrix):
    st = mo.new_stats()
    info = {}
    for name, data in matrix:
        info[name] = mo.decode(data, stats=st)[2]
    assert st['rates'] == {0, 1, 2}                                         # 44.1, 48, 32 kHz
    assert st['modes'] >= {(0, 0), (2, 0), (3, 0), (1, 0), (1, 1), (1, 2), (1, 3)}   # stereo, dual, mono, joint MS/IS
    assert st['blocks'] == {(0, 0), (1, 0), (2, 0), (2, 1), (3, 0)}         # block types 0-3, mixed blocks
    # at every rate (so every rate's short-band widths are used), and intensity stereo at every rate
    assert st['rate_blocks'] == {(r,) + b for r in range(3) for b in st['blocks']}
    assert st['rate_is'] == {0, 1, 2}
    assert st['table_select'] >= set(range(32)) - {4, 14}                   # 4 and 14 do not exist in the standard
    assert st['count1table'] == {0, 1}
    assert st['scfsi'] and st['preflag'] == {0, 1} and st['scalefac_scale'] == {0, 1}
    assert max(st['subblock_gain']) > 0
    assert st['bitrates'] == set(range(1, 15))
    assert st['padding'] == {0, 1} and st['crc'] == {False, True}
    assert st['main_data_begin'] == 511                                     # deep reservoir use
    assert st['spanning'] > 0                                               # granules whose data spans frames
    assert st['quad_dropped'] > 0                                           # count1 quadruples crossing the end
    assert info['tags_info_lame']['lame'] and info['xing_vbr_crc_48k']['xing']
    data = dict(matrix)['tags_info_lame']
    assert data[:3] == b'ID3' and data[-128:-125] == b'TAG' and b'APETAGEX' in data[-300:]


def test_filterbank_and_round_trip_snr():
    """The encoder's analysis inverts the decoder's synthesis: polyphase alone, then through quantisation."""
    x = mo.sine_mix(44100, 44100, 1, seed=3)[0]
    y = mo.synthesise(mo.analyse(x))
    pqmf = _snr(x[:-1000], y[481:481 + len(x) - 1000])
    assert pqmf > 80                                                        # measured 86.0 dB
    x = mo.sine_mix(44100 // 2, 44100, 2, seed=4)
    snr = {}
    for kbps in (128, 320):
        y, rate, info = mo.decode(mo.encode(x, 44100, kbps, mode='stereo', xing='Info'))
        assert rate == 44100 and y.shape == x.shape                         # the LAME trim removes the lag exactly
        snr[kbps] = _snr(x, y)
    assert snr[128] > 25 and snr[320] > 45                                  # measured about 33 and 58 dB
    one = 0.3 * np.sin(2 * np.pi * 1000 * np.arange(44100 // 2) / 44100)
    y, _, _ = mo.decode(mo.encode(one[None], 44100, 320, mode='mono', xing='Info'))
    assert _snr(one, y[0]) > 70                                             # finest quantisation: near the filterbank


def test_oracle_matches_ffmpeg_mp3float(matrix):
    ok, why = ff.available()
    if not ok:
        pytest.skip('libavcodec unavailable (%s): parity of the oracle with FFmpeg is unpinned' % why)
    for name, data in matrix:
        if name == 'tables_48k_stereo_crc':
            continue   # holds quadruples crossing the granule end: FFmpeg keeps them (see test below)
        frames, C = mo.frames_of(data)
        offs, hdrs, _ = mo.find_frames(data)
        skip = 1 if mo.xing_info(data, offs[0], hdrs[0]) is not None else 0
        z = ff.decode(frames[skip:], C)
        y, _ = mo.decode_frames(data, offs[skip:], hdrs[skip:])
        assert z.shape == y.shape, name
        e = z.astype(np.float64) - y
        assert np.abs(e).max() < MAX_BOUND and np.sqrt(np.mean(e ** 2)) < RMS_BOUND, name


def test_ffmpeg_keeps_the_quadruples_that_cross_the_granule_end(matrix):
    """The one rule where this decoder and FFmpeg's mp3float part: a count1 quadruple whose bits cross the end of
    part2_3_length is dropped here and kept by mp3float.  Both stay within the full-accuracy bound on this stream."""
    ok, why = ff.available()
    if not ok:
        pytest.skip('libavcodec unavailable (%s): parity of the oracle with FFmpeg is unpinned' % why)
    data = dict(matrix)['tables_48k_stereo_crc']
    frames, C = mo.frames_of(data)
    offs, hdrs, _ = mo.find_frames(data)
    z = ff.decode(frames, C).astype(np.float64)
    y, _ = mo.decode_frames(data, offs, hdrs)
    assert np.abs(z - y).max() < MAX_BOUND and np.sqrt(np.mean((z - y) ** 2)) < RMS_BOUND


def test_host_chain_skips_false_syncs_in_tags(matrix):
    data = dict(matrix)['tags_info_lame']
    offs, hdrs, _ = mo.find_frames(data)
    frames, dropped = _chain(data)
    assert frames[:, 0].tolist() == offs and dropped == 0
    # a false sync inside the ID3v2 tag and inside the trailing tags
    assert b'\xff\xfb\x90\x44' in data[:40] and b'\xff\xfb\x90' in data[-128:]
    cut = data[:offs[-1] + 100]                                              # a last frame cut short
    frames2, dropped2 = _chain(cut)
    assert frames2[:, 0].tolist() == offs[:-1] and dropped2 == 1


def test_gapless_trim_arithmetic():
    from lib import mp3
    assert mp3.trim_range(11520, None) == (0, 11520)
    assert mp3.trim_range(11520, dict(delay=576, padding=1000, lame=True)) == (1105, 11520 - 471)
    assert mp3.trim_range(11520, dict(delay=576, padding=300, lame=True)) == (1105, 11520)
    assert mp3.trim_range(11520, dict(delay=0, padding=0, lame=False)) == (0, 11520)
    x = mo.sine_mix(5000, 44100, 1)
    data = mo.encode(x, 44100, 128, xing='Info')
    y, _, info = mo.decode(data)
    assert y.shape[1] == 5000 and info['delay'] + 529 == mo.LAG
    assert mp3.xing_info(data, *_chain(data)[0][0].tolist()) == dict(delay=info['delay'], padding=info['padding'],
                                                                     lame=True)


def test_sniff(tmp_path, matrix):
    from lib import mp3
    from oracle import flac_oracle as fo
    flac_data = fo.matrix_streams()[0][0]
    mp3_data = dict(matrix)['reservoir_44k_stereo']
    id3 = b'ID3\x03\x00\x00\x00\x00\x00\x0a' + bytes(10)
    cases = {'a.wav': None, 'a.flac': flac_data, 'b.flac': id3 + flac_data, 'a.mp3': mp3_data,
             'b.mp3': id3 + mp3_data, 'noise.bin': np.random.default_rng(0).integers(0, 256, 20000, np.uint8).tobytes()}
    with wave.open(str(tmp_path / 'a.wav'), 'wb') as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(44100)
        f.writeframes(bytes(1000))
    for k, v in cases.items():
        if v is not None:
            (tmp_path / k).write_bytes(v)
    got = {k: mp3.sniff(str(tmp_path / k)) for k in cases}
    assert got == {'a.wav': False, 'a.flac': False, 'b.flac': False, 'a.mp3': True, 'b.mp3': True, 'noise.bin': False}


def _set_header(data, off, **fields):
    h = int.from_bytes(data[off:off + 4], 'big')
    pos = dict(version=19, layer=17, br=12, sr=10, emph=0, mode=6)
    width = dict(version=2, layer=2, br=4, sr=2, emph=2, mode=2)
    for k, v in fields.items():
        h = (h & ~(((1 << width[k]) - 1) << pos[k])) | (v << pos[k])
    return data[:off] + h.to_bytes(4, 'big') + data[off + 4:]


@pytest.mark.parametrize('fields,msg', [(dict(version=2), 'MPEG-2'), (dict(version=0), 'MPEG-2'),
                                        (dict(layer=2), 'Layer II'), (dict(layer=3), 'Layer I'),
                                        (dict(br=0), 'free-format'), (dict(br=15), 'reserved bitrate'),
                                        (dict(sr=3), 'reserved sampling'), (dict(emph=2), 'reserved emphasis'),
                                        (dict(version=1), 'reserved MPEG version')])
def test_out_of_scope_headers_raise(matrix, fields, msg):
    data = dict(matrix)['reservoir_44k_stereo']
    offs, _, _ = mo.find_frames(data)
    k = 4
    bad = _set_header(data, offs[k], **fields)
    with pytest.raises(ValueError, match=r'frame %d \(byte %d\).*%s' % (k, offs[k], msg)):
        _chain(bad, 'x.mp3')
    every = data
    for o in offs:                                                          # every frame out of scope
        every = _set_header(every, o, **fields)
    with pytest.raises(ValueError, match=r'frame 0 \(byte %d\).*%s' % (offs[0], msg)):
        _chain(every, 'x.mp3')


def test_junk_and_changes_raise(matrix):
    data = dict(matrix)['reservoir_44k_stereo']
    offs, _, _ = mo.find_frames(data)
    junk = data[:offs[3]] + b'\x00\x01\x02' + data[offs[3]:]
    with pytest.raises(ValueError, match=r'frame 3 \(byte %d\).*chain breaks' % offs[3]):
        _chain(junk)
    with pytest.raises(ValueError, match=r'frame 5 \(byte %d\).*rate or channel mode changes' % offs[5]):
        _chain(_set_header(data, offs[5], mode=1))
    with pytest.raises(ValueError, match=r'frame 5 \(byte %d\).*rate or channel mode changes' % offs[5]):
        _chain(_set_header(data, offs[5], sr=1))


def test_mp3_without_gpu_or_soundfile_says_why(tmp_path, matrix):
    import torch
    if torch.cuda.is_available():
        pytest.skip('a CUDA device decodes MP3')
    try:
        import soundfile  # noqa: F401
        pytest.skip('soundfile decodes MP3')
    except ImportError:
        pass
    from lib import audio_io
    path = tmp_path / 'a.mp3'
    path.write_bytes(dict(matrix)['reservoir_44k_stereo'])
    with pytest.raises(RuntimeError, match='MP3 file: decoding it needs a CUDA device'):
        audio_io.load(str(path), sr=None)


# ---------------------------------------------------------------------------------------------------------------- GPU


def _within_bound(y, ref):
    import torch
    assert isinstance(y, torch.Tensor) and y.is_cuda and y.dtype == torch.float32
    y = y.cpu().numpy().astype(np.float64)
    assert y.shape == ref.shape
    e = y - ref
    mx, rms = float(np.abs(e).max()), float(np.sqrt(np.mean(e ** 2)))
    assert mx < MAX_BOUND and rms < RMS_BOUND, (mx, rms)
    return mx, rms


@pytest.mark.gpu
def test_gpu_decodes_every_matrix_stream(matrix):
    from lib import mp3
    for name, data in matrix:
        y, rate, info = mp3.decode(data)
        ref, rate_o, info_o = mo.decode(data)
        assert rate == rate_o, name
        _within_bound(y, ref)
        for k in ('frames', 'delay', 'padding', 'zeroed', 'xing', 'lame', 'dropped'):
            assert info[k] == info_o[k], (name, k)


def _tiled(kbps, seconds=240.0, tile_s=10.0):
    """A long CBR stream made of one encoded tile repeated; every tile after the first decodes to the same samples."""
    from lib import synth
    x = synth.sine_mix(tile_s).astype(np.float64)
    data = mo.encode(x, 44100, kbps, mode='joint', seed=kbps)
    offs, hdrs, _ = mo.find_frames(data)
    reps = int(np.ceil(seconds / tile_s))
    return data * reps, len(offs), data * 2


@pytest.mark.gpu
@pytest.mark.parametrize('kbps', [128, 320])
def test_gpu_decodes_four_minute_track(kbps):
    from lib import mp3
    long_data, per_tile, two = _tiled(kbps)
    y, rate, info = mp3.decode(long_data)
    ref, _, _ = mo.decode(two)
    n = per_tile * mo.FRAME
    assert rate == 44100 and info['frames'] == per_tile * 24 and y.shape[1] == 24 * n
    _within_bound(y[:, :2 * n], ref)
    for t in range(2, 24):
        _within_bound(y[:, t * n:(t + 1) * n], ref[:, n:])


def _set_side_info_bits(data, off, first_bit, width, value):
    """data with ``width`` bits of the side info of the CRC-less frame at ``off``, from bit ``first_bit``, set to
    ``value``."""
    base = 8 * (off + 4) + first_bit
    v = int.from_bytes(data, 'big')
    n = 8 * len(data)
    shift = n - base - width
    v = (v & ~(((1 << width) - 1) << shift)) | (value << shift)
    return v.to_bytes(len(data), 'big')


# bit offsets in a stereo side info: main_data_begin 0, private 9, scfsi 12; granule 0 channel 0 from bit 20:
# part2_3_length +0, big_values +12, global_gain +21, scalefac_compress +29, window switching +33, block type +34;
# each granule-channel takes 59 bits
P23, BIG, WS = 0, 12, 33


@pytest.mark.gpu
def test_gpu_malformed_streams_raise_and_leave_the_decoder_usable(matrix):
    """Each status code of csrc/mp3.cu, from a side-info edit of one frame: a ValueError naming the frame, its byte and
    the reason, and the next call decodes a good stream."""
    from lib import mp3
    data = dict(matrix)['reservoir_44k_stereo']
    offs, hdrs, _ = mo.find_frames(data)
    assert not hdrs[0]['crc'] and hdrs[0]['mode'] != 3
    sis = [mo.parse_side_info(data, o, h) for o, h in zip(offs, hdrs)]
    k = next(f for f in range(1, len(offs)) if sis[f]['gr'][0][0]['big_values'] >= 8 and
             sis[f]['gr'][0][0]['table_select'][0] not in (0, 4, 14))
    g00 = 20

    def expect(bad, code):
        with pytest.raises(ValueError, match=r'frame %d \(byte %d\): %s' % (k, offs[k], re.escape(mp3.ERRORS[code]))):
            mp3.decode(bad)

    bad = data                                          # every granule's part2_3_length at 4095: past the main data
    for q in range(4):
        bad = _set_side_info_bits(bad, offs[k], g00 + 59 * q + P23, 12, 4095)
    expect(bad, 4)
    expect(_set_side_info_bits(data, offs[k], g00 + P23, 12, 1), 5)     # 1 bit for 8+ pairs: past the granule end
    expect(_set_side_info_bits(data, offs[k], g00 + BIG, 9, 511), 3)    # big_values above 288
    ws = _set_side_info_bits(data, offs[k], g00 + WS, 3, 0b100)         # window switching with block type 0
    expect(ws, 2)
    y, _, _ = mp3.decode(data)                          # same process, a good stream
    _within_bound(y, mo.decode(data)[0])


@pytest.mark.gpu
def test_gpu_scfsi_after_a_short_granule(matrix):
    """scfsi in a granule 1 after a short or mixed granule 0 (no valid encoder writes it): the shared bands take granule
    0's long scale factors, a mixed block's bands 0-7, else 0, on the GPU as in the oracle."""
    from lib import mp3
    data = mo.scfsi_after_short_stream()
    offs, hdrs, _ = mo.find_frames(data)
    kinds = set()
    for o, h in zip(offs, hdrs):
        si = mo.parse_side_info(data, o, h)
        for ch in range(2):
            g0 = si['gr'][0][ch]
            if si['scfsi'][ch] and g0['window_switching'] and g0['block_type'] == 2:
                kinds.add(g0['mixed'])
    assert kinds == {0, 1}
    y, _, _ = mp3.decode(data)
    _within_bound(y, mo.decode(data)[0])


@pytest.mark.gpu
def test_gpu_cut_stream_counts_zeroed_frames(matrix):
    from lib import mp3
    data = dict(matrix)['reservoir_44k_stereo']
    offs, hdrs, _ = mo.find_frames(data)
    k = next(i for i in range(1, len(offs)) if mo.parse_side_info(data, offs[i], hdrs[i])['main_data_begin'] > 0)
    cut = data[offs[k]:]
    y, _, info = mp3.decode(cut)
    ref, _, info_o = mo.decode(cut)
    assert info['zeroed'] == info_o['zeroed'] >= 1
    _within_bound(y, ref)


def _write_mp3(path, x, rate, kbps=192):
    path.write_bytes(mo.encode(x, rate, kbps, mode='mono' if x.shape[0] == 1 else 'joint', xing='Info'))


@pytest.mark.gpu
@pytest.mark.parametrize('rate,channels', [(44100, 2), (48000, 2), (44100, 1)])
def test_gpu_audio_io_mp3_equals_decode(tmp_path, rate, channels):
    from lib import audio_io, mp3
    x = mo.sine_mix(int(rate * 1.5), rate, channels, seed=rate + channels)
    _write_mp3(tmp_path / 'a.mp3', x, rate)
    y, sr = audio_io.load(str(tmp_path / 'a.mp3'), sr=44100, mono=False)
    d, r, _ = mp3.decode(str(tmp_path / 'a.mp3'))
    d = d.cpu().numpy()
    if channels == 1:
        d = d.mean(axis=0)
    if r != 44100:
        d = audio_io.resample(d, r, 44100)
    assert sr == 44100 and y.dtype == np.float32 and np.array_equal(y, d)


@pytest.mark.gpu
def test_gpu_inference_cli_mp3_equals_python_path(tmp_path):
    import torch
    sys.path.insert(0, PKG)
    import inference
    from lib import audio_io, mp3, nets, spec_utils, synth
    x = mo.sine_mix(44100 * 3, 44100, 2, seed=11)
    (tmp_path / 'in').mkdir()
    _write_mp3(tmp_path / 'in' / 'mix.mp3', x, 44100)
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
    out = tmp_path / 'out_cli'
    r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt,
                        '-i', str(tmp_path / 'in' / 'mix.mp3'), '-o', str(out)],
                       capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 0, r.stderr
    args = inference.build_parser().parse_args(['-P', ckpt, '-i', 'unused'])
    device = torch.device('cuda:0')
    model = nets.CascadedNet(args.n_fft, args.hop_length, 32, 128)
    model.load_state_dict(torch.load(ckpt, map_location='cpu'))
    model.to(device)
    spec_utils.set_device(0)
    X = mp3.decode(str(tmp_path / 'in' / 'mix.mp3'))[0].cpu().numpy()
    sp = inference.Separator(model=model, device=device, batchsize=args.batchsize, cropsize=args.cropsize,
                             postprocess=args.postprocess, wiener_iterations=args.wiener_iterations)
    inst, voc = sp.separate_wave(X)[:2]
    ref = tmp_path / 'out_py'
    ref.mkdir()
    audio_io.write(str(ref / 'mix_Instruments.wav'), inst.T, 44100)
    audio_io.write(str(ref / 'mix_Vocals.wav'), voc.T, 44100)
    for f in ('mix_Instruments.wav', 'mix_Vocals.wav'):
        assert (out / f).read_bytes() == (ref / f).read_bytes()


@pytest.mark.gpu
def test_gpu_cache_or_load_on_mp3_pairs(tmp_path):
    from lib import audio_io, spec_utils
    mix = mo.sine_mix(44100 * 2, 44100, 2, seed=21)
    inst = 0.5 * mix
    _write_mp3(tmp_path / 'mix.mp3', mix, 44100)
    _write_mp3(tmp_path / 'inst.mp3', inst, 44100)
    X, y, pm, pi = spec_utils.cache_or_load(str(tmp_path / 'mix.mp3'), str(tmp_path / 'inst.mp3'), 44100, 1024, 2048)
    assert os.path.exists(pm) and os.path.exists(pi)
    a, _ = audio_io.load(str(tmp_path / 'mix.mp3'), sr=44100)
    assert X.shape[0] == 2 and X.shape[1] == 1025 and X.shape[2] == 1 + a.shape[1] // 1024
    X2, y2, _, _ = spec_utils.cache_or_load(str(tmp_path / 'mix.mp3'), str(tmp_path / 'inst.mp3'), 44100, 1024, 2048)
    assert np.array_equal(X, X2) and np.array_equal(y, y2)
