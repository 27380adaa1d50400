"""M4A / MP4 (AAC-LC) input: the oracle (oracle/aac_oracle.py) against FFmpeg's aac decoder, its coverage and round
trip, the container side of lib/aac.py (CPU), and the GPU decoder (csrc/aac.cu) against the oracle, through lib.aac,
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
from oracle import aac_oracle as ao  # noqa: E402
from oracle import aac_tables as at  # noqa: E402
from oracle import ffmpeg_aac as ff  # noqa: E402

# the gate of DESIGN.md §13 / §14, full scale +-1
MAX_BOUND = 2.0 ** -14
RMS_BOUND = 2.0 ** -15 / np.sqrt(12.0)
# oracle against FFmpeg's float decoder on streams without PNS (measured up to 9.1e-6, with outputs up to 1.5)
FFMPEG_BOUND = 2.0e-5


@pytest.fixture(scope='module')
def matrix():
    return ao.matrix()


def _packets(data):
    from lib import aac
    t = aac.parse(data)
    return [bytes(data[o:o + s]) for o, s in zip(t['offsets'], t['sizes'])], t


# ------------------------------------------------------------------------------------------------------------ oracle


def test_tables_are_complete_prefix_codes_and_match_the_kernel_copy():
    sizes = (121, 81, 81, 81, 81, 81, 81, 64, 64, 169, 169, 289)
    for b, n in enumerate(sizes):
        a, e = at.HUFF_START[b], at.HUFF_START[b + 1]
        assert e - a == n
        assert sum(2.0 ** -ln for ln in at.HUFF_LENGTHS[a:e]) == 1.0
        assert sorted(at.HUFF_SYMBOLS[a:e]) == list(range(n))
    for tab, n_long in ((at.SWB_LONG, (41, 41, 47, 49, 49, 51, 47, 47, 43, 43, 43, 40)),
                        (at.SWB_SHORT, (12, 12, 12, 14, 14, 14, 15, 15, 15, 15, 15, 15))):
        assert tuple(len(t) - 1 for t in tab) == n_long
        assert all(t[0] == 0 and t[-1] == (1024 if tab is at.SWB_LONG else 128) and np.all(np.diff(t) > 0) for t in tab)
    for w in at.WINDOW_LONG + at.WINDOW_SHORT:   # Princen-Bradley: each half-window pair is power complementary
        assert np.allclose(w ** 2 + w[::-1] ** 2, 1.0, atol=1e-12)
    src = open(os.path.join(PKG, 'csrc', 'aac.cu')).read()

    def arr(name, conv=int):
        body = re.search(name + r'(?:\[\d+\])+ = \{(.*?)\};', src, re.S).group(1)
        return [conv(v.strip().rstrip('f')) for v in body.replace('{', ' ').replace('}', ' ').replace('\n', ' ').split(',')
                if v.strip()]
    assert arr('kAacHuffLengths') == list(at.HUFF_LENGTHS)
    assert arr('kAacHuffSymbols') == list(at.HUFF_SYMBOLS)
    assert arr('kAacHuffStart') == list(at.HUFF_START)
    assert arr('kTnsMaxBandsLong') == list(at.TNS_MAX_BANDS_LONG)
    assert arr('kTnsMaxBandsShort') == list(at.TNS_MAX_BANDS_SHORT)
    for name, ref in (('kSwbLong', at.SWB_LONG), ('kSwbShort', at.SWB_SHORT)):
        body = re.search(name + r'\[12\]\[\d+\] = \{(.*?)\};', src, re.S).group(1)
        rows = [[int(v) for v in r.split(',')] for r in re.findall(r'\{([^{}]*)\}', body)]
        assert rows == [list(t) for t in ref], name
    for name, ref in (('kTnsCoef3', at.TNS_COEF_3), ('kTnsCoef4', at.TNS_COEF_4),
                      ('kWinLong', np.concatenate(at.WINDOW_LONG)), ('kWinShort', np.concatenate(at.WINDOW_SHORT))):
        assert np.allclose(arr(name, float), ref, rtol=0, atol=1e-8), name


def test_matrix_covers_the_contract(matrix):
    st = ao.new_stats()
    for name, data in matrix:
        ao.decode(data, stats=st)
    assert st['rates'] == set(range(12)) and st['channels'] == {1, 2}
    assert st['codebooks'] == set(range(12)) | {13, 14, 15}                 # all spectral codebooks, PNS, intensity
    assert st['ws'] == {0, 1, 2, 3}
    assert st['ws_pairs'] >= {(0, 0), (0, 1), (1, 2), (2, 2), (2, 3), (3, 0), (3, 1)}   # every allowed transition
    assert st['shapes'] == {(0, 0), (0, 1), (1, 0), (1, 1)}                 # KBD after sine and sine after KBD
    assert len(st['groupings'] - {1}) >= 5                                  # grouped short windows
    assert st['pulse'] > 0 and st['esc_long'] > 0
    assert {(w, r, c) for w in ('long', 'short') for r in (3, 4) for c in (0, 1)} <= st['tns']
    assert st['ms'] == {0, 1, 2} and st['common_window'] == {0, 1}
    assert st['is_cb'] == {14, 15} and st['is_inverted'] > 0
    assert st['pns'] > 0 and st['pns_ms'] > 0                               # PNS, also in an M/S band
    assert st['fil'] > 0 and st['dse'] > 0


def test_filterbank_and_round_trip_snr():
    """The encoder's analysis inverts the decoder's synthesis (every window sequence and shape), then through
    quantisation: the decoded signal is the input delayed by one frame."""
    x = ao.sine_mix(8 * 1024, 44100, 1, seed=3)[0] * 32768
    seq = [(0, 0), (1, 1), (2, 0), (2, 1), (3, 1), (0, 0), (0, 1), (0, 0), (0, 0)]
    s = np.concatenate([np.zeros(1024), x, np.zeros(2048)])
    out = np.zeros(len(s) + 2048)
    prev = 0
    for k, (ws, shape) in enumerate(seq):
        z = ao.synthesis(ao.analysis(s[k * 1024:k * 1024 + 2048], ws, shape, prev), ws, shape, prev)
        out[k * 1024:k * 1024 + 2048] += z
        prev = shape
    assert np.abs(out[1024:1024 + len(x)] - x).max() < 1e-7 * 32768
    x = ao.sine_mix(44100 // 2, 44100, 2, seed=4)
    for kbps, floor in ((128, 15), (256, 22)):
        packets, _ = ao.encode(x, 44100, kbps)
        y, _ = ao.decode_packets(packets, 4, 2)
        e = y[:, 1024:1024 + x.shape[1]] - x
        assert 10 * np.log10(np.sum(x ** 2) / np.sum(e ** 2)) > floor       # measured about 20 and 28 dB


def test_oracle_matches_ffmpeg_aac(matrix):
    ok, why = ff.available()
    if not ok:
        pytest.skip('libavcodec unavailable (%s): parity of the oracle with FFmpeg is unpinned' % why)
    for name, data in matrix:
        if ao.is_pns(name):
            continue
        packets, t = _packets(data)
        z = ff.decode(packets, t['rate_index'], t['channels'])
        y, _ = ao.decode_packets(packets, t['rate_index'], t['channels'])
        assert z.shape == y.shape, name
        assert np.abs(z.astype(np.float64) - y).max() < FFMPEG_BOUND, name


def test_oracle_matches_ffmpeg_aac_on_pns_streams_in_the_mdct_domain(matrix):
    """PNS noise differs by construction (FFmpeg's LCG, the oracle's hash).  The oracle's forward MDCT of both outputs,
    with each frame's windows, recovers each frame's spectrum: non-noise bins agree, and so does each noise band's
    energy, window by window."""
    ok, why = ff.available()
    if not ok:
        pytest.skip('libavcodec unavailable (%s): parity of the oracle with FFmpeg is unpinned' % why)
    checked = 0
    for name, data in matrix:
        if not ao.is_pns(name):
            continue
        packets, t = _packets(data)
        z = ff.decode(packets, t['rate_index'], t['channels']).astype(np.float64)
        y, frames = ao.decode_packets(packets, t['rate_index'], t['channels'])
        Sy, Sz = ao.frame_spectra(y, frames), ao.frame_spectra(z, frames)
        for k in range(len(Sy)):
            for c, f in enumerate(frames[k]['ics']):
                assert np.allclose(Sy[k][c], frames[k]['spec'][c], atol=1e-6 * 32768 * 1e-3)   # recovery is exact
                noise = np.zeros(1024, bool)
                w0 = 0
                for g, n in enumerate(f['group_len']):
                    for w in range(w0, w0 + n):
                        for b in range(f['max_sfb']):
                            if f['cb'][g, b] != 13:
                                continue
                            a, e = 128 * w + f['swb'][b], 128 * w + f['swb'][b + 1]
                            noise[a:e] = True
                            ey, ez = np.sum(Sy[k][c][a:e] ** 2), np.sum(Sz[k][c][a:e] ** 2)
                            assert abs(ey - ez) <= 1e-4 * ey + 1e-3, (name, k, c, b)
                            checked += 1
                    w0 += n
                d = np.abs(Sy[k][c][~noise] - Sz[k][c][~noise]) * ao.OUT_SCALE
                assert d.max() < 1e-4, (name, k, c)
    assert checked > 50


def test_container_layouts_yield_the_same_packets_and_trim():
    from lib import aac
    x = ao.sine_mix(9 * 1024 + 100, 44100, 2, seed=5)
    packets, a = ao.encode(x, 44100, 128, seed=5)
    n = x.shape[1]
    for layout in ('plain', 'moov_last', 'co64', 'chunks', 'fragmented'):
        for video in (False, True):
            for edit, movie_ts in ((None, 1000), ((1024, n), 1000), ((2112, n - 1500), 600), ((1024, n), 44100)):
                data, truth = ao.mp4(packets, a, 44100, 2, layout=layout, edit=edit, video=video, movie_ts=movie_ts)
                t = aac.parse(data)
                assert t['offsets'].tolist() == truth['offsets'] and t['sizes'].tolist() == truth['sizes']
                assert [bytes(data[o:o + s]) for o, s in zip(t['offsets'], t['sizes'])] == packets
                assert t['rate'] == 44100 and t['channels'] == 2 and t['fragmented'] == (layout == 'fragmented')
                lo, hi = aac.trim_range(len(packets) * 1024, t)
                if edit is None:
                    assert (lo, hi) == (0, len(packets) * 1024)
                else:
                    assert (lo, hi - lo) == (truth['priming'], truth['kept'])
    assert aac.trim_range(10240, dict(edit=True, media_time=1024, segment=None)) == (1024, 10240)


@pytest.mark.parametrize('box,layout,msg', [(b'mvhd', 'plain', 'no mvhd box in moov'),
                                              (b'mdia', 'plain', 'no mdia box in trak'),
                                              (b'stsd', 'moov_last', 'no stsd box in stbl'),
                                              (b'tfhd', 'fragmented', 'no tfhd box in traf')])
def test_missing_boxes_raise_value_error(box, layout, msg):
    from lib import aac
    x = ao.sine_mix(3 * 1024, 44100, 2, seed=12)
    packets, a = ao.encode(x, 44100, 128, seed=12)
    data, _ = ao.mp4(packets, a, 44100, 2, layout=layout)
    with pytest.raises(ValueError, match='x.m4a: %s' % msg):
        aac.parse(data.replace(box, b'junk'), 'x.m4a')


def test_only_the_audio_packets_are_gathered_for_the_device():
    """A video track and bytes between chunks stay on the host: the device gets the packets back to back."""
    from lib import aac
    x = ao.sine_mix(9 * 1024, 44100, 2, seed=13)
    packets, a = ao.encode(x, 44100, 128, seed=13)
    data, truth = ao.mp4(packets, a, 44100, 2, layout='chunks', video=True)
    t = aac.parse(data)
    packed, table = aac.gather(data, t['offsets'], t['sizes'])
    assert packed.tobytes() == b''.join(packets) and len(packed) < len(data)
    assert table[:, 1].tolist() == [len(p) for p in packets]
    assert table[:, 0].tolist() == np.concatenate([[0], np.cumsum([len(p) for p in packets])[:-1]]).tolist()


def test_constant_sample_size_stream(matrix):
    data = dict(matrix)['cbr_48k_stereo_fragmented']
    packets, t = _packets(data)
    assert len(set(len(p) for p in packets)) == 1
    from lib import aac
    raw, truth = ao.mp4(packets, ao.asc(3, 2), 48000, 2)
    t = aac.parse(raw)
    assert t['sizes'].tolist() == [420] * len(packets)
    assert b'stsz\x00\x00\x00\x00\x00\x00\x01\xa4' in raw          # one sample_size for every sample


def test_sniff(tmp_path, matrix):
    from lib import aac
    from oracle import flac_oracle as fo
    from oracle import mp3_oracle as mo
    m4a = dict(matrix)['tools_44k_stereo_fragmented']
    cases = {'a.wav': None, 'a.flac': fo.matrix_streams()[0][0], 'a.mp3': dict(mo.matrix())['reservoir_44k_stereo'],
             'a.m4a': m4a, 'cut.m4a': m4a[:6], 'noise.bin': np.random.default_rng(0).integers(0, 256, 2000,
                                                                                              np.uint8).tobytes()}
    with wave.open(str(tmp_path / 'a.wav'), 'wb') as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(44100)
        f.writeframes(bytes(1000))
    for k, v in cases.items():
        if v is not None:
            (tmp_path / k).write_bytes(v)
    moov_last = ao.mp4([b'\x00' * 8], ao.asc(4, 2), 44100, 2, layout='moov_last')[0]
    (tmp_path / 'b.m4a').write_bytes(moov_last[int.from_bytes(moov_last[:4], 'big'):])   # no ftyp: a free box first
    got = {k: aac.sniff(str(tmp_path / k)) for k in list(cases) + ['b.m4a']}
    assert got == {'a.wav': False, 'a.flac': False, 'a.mp3': False, 'a.m4a': True, 'cut.m4a': False,
                   'noise.bin': False, 'b.m4a': True}


def _edit_asc(data, new_asc):
    """The file with its AudioSpecificConfig replaced by one of the same length."""
    from lib import aac
    old = aac.parse(data)['asc']
    assert len(old) == len(new_asc) and data.count(b'\x05\x02' + old) == 1
    return data.replace(b'\x05\x02' + old, b'\x05\x02' + new_asc)


@pytest.mark.parametrize('case,msg', [
    ('he_aac', r'audio object type 5 \(HE-AAC \(SBR\)\)'), ('he_aac_v2', r'audio object type 29 \(HE-AACv2'),
    ('main', r'audio object type 1 \(AAC Main\)'), ('ssr', r'audio object type 3 \(AAC SSR\)'),
    ('ltp', r'audio object type 4 \(AAC LTP\)'), ('sbr_sync', r'SBR sync extension'),
    ('frame960', r'960-sample frames'), ('pce', r'channel configuration 0'), ('surround', r'channel configuration 6'),
    ('stts', r'stts delta 960'), ('enca', r'encrypted \(enca\)'), ('alac', r'ALAC'), ('edits', r'2 edits'),
    ('mp3_in_mp4', r'objectTypeIndication 0x6b')])
def test_out_of_scope_files_raise(case, msg):
    from lib import aac
    x = ao.sine_mix(3 * 1024, 44100, 2, seed=6)
    packets, a = ao.encode(x, 44100, 128, seed=6)
    kw = {}
    if case in ('he_aac', 'he_aac_v2', 'main', 'ssr', 'ltp'):
        a = ao.asc(4, 2, aot=dict(he_aac=5, he_aac_v2=29, main=1, ssr=3, ltp=4)[case])
    elif case == 'sbr_sync':
        a = ao.asc(4, 2, sbr_ext=1)
    elif case == 'frame960':
        a = ao.asc(4, 2, frame960=True)
    elif case == 'pce':
        a = ao.asc(4, 0)
    elif case == 'surround':
        a = ao.asc(4, 6)
    elif case == 'stts':
        kw['stts_delta'] = 960
    elif case in ('enca', 'alac'):
        kw['fmt'] = case.encode()
    elif case == 'edits':
        kw['edit'] = [(1024, 1024), (2048, 1024)]
    elif case == 'mp3_in_mp4':
        kw['oti'] = 0x6B
    data, _ = ao.mp4(packets, a, 44100, 2, **kw)
    with pytest.raises(ValueError, match=msg):
        aac.parse(data, 'x.m4a')
    if case == 'sbr_sync':   # the same extension with sbrPresentFlag 0 is plain AAC-LC
        assert aac.parse(ao.mp4(packets, ao.asc(4, 2, sbr_ext=0), 44100, 2)[0])['channels'] == 2


def _bit_edit(packet, bit, width, value):
    v = int.from_bytes(packet, 'big')
    n = 8 * len(packet)
    shift = n - bit - width
    v = (v & ~(((1 << width) - 1) << shift)) | (value << shift)
    return v.to_bytes(len(packet), 'big')


def _sce_stream():
    x = ao.sine_mix(4 * 1024, 44100, 1, seed=8)
    packets, a = ao.encode(x, 44100, 96, seed=8)
    return ao.mp4(packets, a, 44100, 1)[0]


# SCE bit layout: element id 0, tag 3, global_gain 7, ics_reserved_bit 15, window_sequence 16, window_shape 18,
# max_sfb 19 (6 bits), predictor_data_present 25, then the section data from bit 26
PACKET_CASES = [
    ('sbr_fil', 'an SBR extension payload in a FIL element', 12),
    ('cce', 'a CCE element', 11), ('lfe', 'an LFE element', 11), ('pce', 'a PCE element', 11),
    ('main_prediction', 'predictor_data_present is set', 9), ('reserved_bit', 'ics_reserved_bit is set', 14),
    ('max_sfb', 'max_sfb', 4), ('section', 'a section runs past max_sfb', 2), ('codebook12', 'reserved section codebook 12', 3),
    ('cut', 'the bits run past the end of the packet', 1)]


def _bad_packet(packet, case):
    if case == 'sbr_fil':     # a FIL element carrying EXT_SBR_DATA ahead of the SCE
        bw = ao.BitWriter()
        bw.write(ao.FIL, 3)
        bw.write(1, 4)
        bw.write(13, 4)
        bw.write(0, 4)
        nbits = bw.n + 8 * len(packet)
        v = (bw.v << (8 * len(packet))) | int.from_bytes(packet, 'big')
        return (v << ((-nbits) % 8)).to_bytes((nbits + 7) // 8, 'big')
    if case in ('cce', 'lfe', 'pce'):
        return _bit_edit(packet, 0, 3, dict(cce=ao.CCE, lfe=ao.LFE, pce=ao.PCE)[case])
    if case == 'main_prediction':
        return _bit_edit(packet, 25, 1, 1)
    if case == 'reserved_bit':
        return _bit_edit(packet, 15, 1, 1)
    if case == 'max_sfb':
        return _bit_edit(packet, 19, 6, 63)
    if case == 'section':      # the first section's length: 31 + (max_sfb) bands
        return _bit_edit(packet, 30, 10, (31 << 5) | 31)
    if case == 'codebook12':
        return _bit_edit(packet, 26, 4, 12)
    if case == 'cut':
        return packet[:len(packet) // 3]


def _cpe_stream():
    x = ao.sine_mix(4 * 1024, 44100, 2, seed=9)
    packets, a = ao.encode(x, 44100, 160, seed=9)
    return ao.mp4(packets, a, 44100, 2)[0]


def _ics_head(bw, gg, ws=0, max_sfb=0):
    """global_gain and an ics_info (sine window, no grouping, no prediction) of an individual channel stream."""
    bw.write(gg, 8)
    bw.write(0, 1)
    bw.write(ws, 2)
    bw.write(0, 1)
    if ws == ao.EIGHT_SHORT:
        bw.write(max_sfb, 4)
        bw.write(0, 7)
    else:
        bw.write(max_sfb, 6)
        bw.write(0, 1)


def _built_packet(case):
    """A packet written bit by bit (44.1 kHz) that holds one status case, or one extreme but valid value."""
    bw = ao.BitWriter()
    if case == 'no_channel':
        bw.write(ao.END, 3)
        return bw.bytes()
    if case in ('ms_reserved', 'is_extreme'):
        bw.write(ao.CPE, 3)
        bw.write(0, 4)
        bw.write(1, 1)                                   # common_window
        bw.write(0, 1)
        bw.write(0, 2)
        bw.write(0, 1)
        bw.write(0 if case == 'ms_reserved' else 3, 6)   # max_sfb
        bw.write(0, 1)
        bw.write(3 if case == 'ms_reserved' else 0, 2)   # ms_mask_present
        if case == 'is_extreme':
            bw.write(100, 8)                             # left: codebook 1 over bands 0-2, one +-1 per quadruple
            bw.write(1, 4)
            bw.write(3, 5)
            for _ in range(3):
                bw.huff(0, 60)
            bw.write(0, 3)
            for _ in range(3):
                bw.huff(1, 27 * 2 + 9 + 3 + 1)
            bw.write(100, 8)                             # right: intensity, positions -60, -120, -180
            bw.write(14, 4)
            bw.write(3, 5)
            for _ in range(3):
                bw.huff(0, 0)
            bw.write(0, 3)
        bw.write(ao.END, 3)
        return bw.bytes()
    bw.write(ao.SCE, 3)
    bw.write(0, 4)
    if case == 'gain_control':
        _ics_head(bw, 100)
        bw.write(0, 2)
        bw.write(1, 1)
    elif case == 'tns_order':
        _ics_head(bw, 100)
        bw.write(0, 1)
        bw.write(1, 1)                                   # tns_data_present
        bw.write(1, 2)
        bw.write(0, 1)
        bw.write(10, 6)
        bw.write(13, 5)                                  # order 13 > 12
    elif case == 'pulse_short':
        _ics_head(bw, 100, ws=ao.EIGHT_SHORT)
        bw.write(1, 1)                                   # pulse_data_present
    elif case == 'escape':
        _ics_head(bw, 100, max_sfb=1)
        bw.write(11, 4)
        bw.write(1, 5)
        bw.huff(0, 60)
        bw.write(0, 3)
        bw.huff(11, 16 * 17)                             # (16, 0): an escaped value
        bw.write(0, 1)
        bw.write(0x3FF << 1, 11)                         # ten escape-prefix ones: longer than 13 bits
    elif case == 'scale_factor':
        _ics_head(bw, 255, max_sfb=1)
        bw.write(1, 4)
        bw.write(1, 5)
        bw.huff(0, 61)                                   # 255 + 1
        bw.write(0, 3)
        bw.huff(1, 40)
    elif case == 'noise_extreme':
        _ics_head(bw, 255, max_sfb=1)
        bw.write(13, 4)
        bw.write(1, 5)
        bw.write(511, 9)                                 # noise energy 255 - 90 + 255 = 420
        bw.write(0, 3)
    bw.write(ao.END, 3)
    bw.write(0, 16)
    return bw.bytes()


BUILT_CASES = [('no_channel', 'no channel element before END', 13, 1), ('ms_reserved', 'reserved ms_mask_present 3', 8, 2),
               ('gain_control', 'gain_control_data_present is set', 10, 1), ('tns_order', 'TNS order', 7, 1),
               ('pulse_short', 'pulse data in an EIGHT_SHORT frame', 6, 1),
               ('escape', 'an escape sequence is longer than 13 bits', 5, 1),
               ('scale_factor', 'a scale factor leaves [0, 255]', 15, 1)]


def _bad_file(case, channels):
    """(file with packet 2 replaced by the case's packet, the good file)."""
    data = _sce_stream() if channels == 1 else _cpe_stream()
    packets, t = _packets(data)
    cases = dict((c, m) for c, m, _ in PACKET_CASES)
    bad = _bad_packet(packets[2], case) if case in cases else _built_packet(case)
    return ao.mp4(packets[:2] + [bad] + packets[3:], ao.asc(4, channels), 44100, channels)[0], data


ALL_CASES = [(c, m, k, 1) for c, m, k in PACKET_CASES] + BUILT_CASES


def test_status_table_is_covered():
    from lib import aac
    assert {k for _, _, k, _ in ALL_CASES} == set(aac.ERRORS)


@pytest.mark.parametrize('case,msg,code,channels', ALL_CASES)
def test_out_of_scope_and_malformed_packets_raise_in_the_oracle(case, msg, code, channels):
    from lib import aac
    raw, _ = _bad_file(case, channels)
    packets, t = _packets(raw)
    assert msg in aac.ERRORS[code] or code == 11
    with pytest.raises(ValueError, match=r'packet 2 \(byte %d\): .*%s' % (t['offsets'][2], re.escape(msg))):
        ao.decode_packets(packets, t['rate_index'], channels, t['offsets'])


@pytest.mark.parametrize('case,channels', [('noise_extreme', 1), ('is_extreme', 2)])
def test_extreme_noise_energy_and_intensity_position_are_clipped(case, channels):
    """A noise energy of 420 and intensity positions down to -180 are valid syntax; clipped to FFmpeg's ranges they
    scale their bands by finite amounts."""
    raw, _ = _bad_file(case, channels)
    packets, t = _packets(raw)
    y, frames = ao.decode_packets(packets, t['rate_index'], channels)
    assert np.all(np.isfinite(y)) and np.abs(y[:, 2 * 1024:4 * 1024]).max() > 1e3
    cb = frames[2]['ics'][-1]['cb'][0]
    assert (cb[0] == 13) if case == 'noise_extreme' else (list(cb[:3]) == [14, 14, 14])


def test_m4a_without_gpu_says_why(tmp_path, matrix):
    import torch
    if torch.cuda.is_available():
        pytest.skip('a CUDA device decodes M4A')
    from lib import audio_io
    path = tmp_path / 'a.m4a'
    path.write_bytes(dict(matrix)['tools_44k_stereo_fragmented'])
    with pytest.raises(RuntimeError, match='MP4 / M4A file: decoding it needs a CUDA device'):
        audio_io.load(str(path), sr=None)


# ---------------------------------------------------------------------------------------------------------------- GPU


def _within_bound(y, ref):
    import torch
    assert isinstance(y, torch.Tensor) and y.is_cuda and y.dtype == torch.float32
    y = y.cpu().numpy().astype(np.float64)
    assert y.shape == ref.shape, (y.shape, ref.shape)
    e = y - ref
    mx, rms = float(np.abs(e).max()), float(np.sqrt(np.mean(e ** 2)))
    assert mx < MAX_BOUND and rms < RMS_BOUND, (mx, rms)
    return mx, rms


@pytest.mark.gpu
def test_gpu_decodes_every_matrix_stream(matrix):
    from lib import aac
    for name, data in matrix:
        y, rate, info = aac.decode(data)
        ref, rate_o, info_o = ao.decode(data)
        assert rate == rate_o, name
        assert info == info_o, name
        _within_bound(y, ref)


def _tiled(kbps, seconds=240.0, tile_s=10.0):
    """A long stream made of one encoded tile repeated: every tile after the first decodes to the same samples."""
    from lib import synth
    x = synth.sine_mix(tile_s).astype(np.float64)
    packets, a = ao.encode(x, 44100, kbps, seed=kbps)
    reps = int(np.ceil(seconds / tile_s))
    return packets, a, reps


@pytest.mark.gpu
@pytest.mark.parametrize('kbps', [128, 256])
def test_gpu_decodes_four_minute_track(kbps):
    from lib import aac
    packets, a, reps = _tiled(kbps)
    data, _ = ao.mp4(packets * reps, a, 44100, 2)
    y, rate, info = aac.decode(data)
    ref, _ = ao.decode_packets(packets * 2, 4, 2)
    n = len(packets) * 1024
    assert rate == 44100 and info['frames'] == len(packets) * reps and y.shape[1] == reps * n
    _within_bound(y[:, :2 * n], ref)
    for t in range(2, reps):
        _within_bound(y[:, t * n:(t + 1) * n], ref[:, n:])


@pytest.mark.gpu
def test_gpu_malformed_packets_raise_and_leave_the_decoder_usable():
    """Each status of csrc/aac.cu from a byte edit of one packet: a ValueError naming the packet, its byte and the
    reason; the next call decodes a good file."""
    from lib import aac
    for case, msg, code, channels in ALL_CASES:
        raw, data = _bad_file(case, channels)
        off = aac.parse(raw)['offsets'][2]
        with pytest.raises(ValueError, match=r'packet 2 \(byte %d\): %s' % (off, re.escape(aac.ERRORS[code]))):
            aac.decode(raw)
        y, _, _ = aac.decode(data)
        _within_bound(y, ao.decode(data)[0])


@pytest.mark.gpu
@pytest.mark.parametrize('case,channels', [('noise_extreme', 1), ('is_extreme', 2)])
def test_gpu_extreme_noise_energy_and_intensity_position_stay_finite(case, channels):
    from lib import aac
    raw, _ = _bad_file(case, channels)
    y, _, _ = aac.decode(raw)
    ref, _, _ = ao.decode(raw)
    y = y.cpu().numpy().astype(np.float64)
    assert np.all(np.isfinite(y)) and y.shape == ref.shape
    assert np.abs(y - ref).max() < 1e-5 * np.abs(ref).max()


@pytest.mark.gpu
@pytest.mark.parametrize('packets', [32, 64])
def test_gpu_mono_stream_of_a_multiple_of_32_packets(packets):
    """A mono file whose descriptor array ends on a 256-byte boundary, with energy in the lowest bins of packet 0."""
    from lib import aac
    n = (packets - 1) * 1024
    t = np.arange(n) / 44100.0
    x = 0.4 * np.sin(2 * np.pi * 75.0 * t)[None] + 0.5 * ao.sine_mix(n, 44100, 1, seed=packets)
    pk, a = ao.encode(x, 44100, 128, seed=packets)
    assert len(pk) == packets
    data = ao.mp4(pk, a, 44100, 1)[0]
    ref, _, _ = ao.decode(data)
    assert np.abs(ref[0, :2048]).max() > 0.05
    y, _, _ = aac.decode(data)
    _within_bound(y, ref)


def _write_m4a(path, x, rate, kbps=192):
    packets, a = ao.encode(x, rate, kbps * x.shape[0] // 2, seed=rate)
    path.write_bytes(ao.mp4(packets, a, rate, x.shape[0], edit=(1024, x.shape[1]))[0])


@pytest.mark.gpu
@pytest.mark.parametrize('rate,channels', [(44100, 2), (48000, 2), (44100, 1)])
def test_gpu_audio_io_m4a_equals_decode(tmp_path, rate, channels):
    from lib import aac, audio_io
    x = ao.sine_mix(int(rate * 1.5), rate, channels, seed=rate + channels)
    _write_m4a(tmp_path / 'a.m4a', x, rate)
    y, sr = audio_io.load(str(tmp_path / 'a.m4a'), sr=44100, mono=False)
    d, r, _ = aac.decode(str(tmp_path / 'a.m4a'))
    d = d.cpu().numpy()
    if channels == 1:
        d = d.mean(axis=0)
    if r != 44100:
        d = audio_io.resample(d, r, 44100)
    assert sr == 44100 and y.dtype == np.float32 and np.array_equal(y, d)


@pytest.mark.gpu
def test_gpu_inference_cli_m4a_equals_python_path(tmp_path):
    import torch
    sys.path.insert(0, PKG)
    import inference
    from lib import aac, audio_io, nets, spec_utils, synth
    x = ao.sine_mix(44100 * 3, 44100, 2, seed=11)
    (tmp_path / 'in').mkdir()
    _write_m4a(tmp_path / 'in' / 'song.m4a', x, 44100)
    ckpt = str(tmp_path / 'synthetic.pth')
    torch.save(synth.to_torch_state_dict(synth.make_state_dict()), ckpt)
    out = tmp_path / 'out_cli'
    r = subprocess.run([sys.executable, os.path.join(PKG, 'inference.py'), '-g', '0', '-P', ckpt,
                        '-i', str(tmp_path / 'in' / 'song.m4a'), '-o', str(out)],
                       capture_output=True, text=True, cwd=PKG)
    assert r.returncode == 0, r.stderr
    args = inference.build_parser().parse_args(['-P', ckpt, '-i', 'unused'])
    device = torch.device('cuda:0')
    model = nets.CascadedNet(args.n_fft, args.hop_length, 32, 128)
    model.load_state_dict(torch.load(ckpt, map_location='cpu'))
    model.to(device)
    spec_utils.set_device(0)
    X = aac.decode(str(tmp_path / 'in' / 'song.m4a'))[0].cpu().numpy()
    sp = inference.Separator(model=model, device=device, batchsize=args.batchsize, cropsize=args.cropsize,
                             postprocess=args.postprocess, wiener_iterations=args.wiener_iterations)
    inst, voc = sp.separate_wave(X)[:2]
    ref = tmp_path / 'out_py'
    ref.mkdir()
    audio_io.write(str(ref / 'song_Instruments.wav'), inst.T, 44100)
    audio_io.write(str(ref / 'song_Vocals.wav'), voc.T, 44100)
    for f in ('song_Instruments.wav', 'song_Vocals.wav'):
        assert (out / f).read_bytes() == (ref / f).read_bytes()


@pytest.mark.gpu
def test_gpu_cache_or_load_on_m4a_pairs(tmp_path):
    from lib import audio_io, spec_utils
    mix = ao.sine_mix(44100 * 2, 44100, 2, seed=21)
    inst = 0.5 * mix
    _write_m4a(tmp_path / 'mix.m4a', mix, 44100)
    _write_m4a(tmp_path / 'inst.m4a', inst, 44100)
    X, y, pm, pi = spec_utils.cache_or_load(str(tmp_path / 'mix.m4a'), str(tmp_path / 'inst.m4a'), 44100, 1024, 2048)
    assert os.path.exists(pm) and os.path.exists(pi)
    a, _ = audio_io.load(str(tmp_path / 'mix.m4a'), sr=44100)
    assert X.shape[0] == 2 and X.shape[1] == 1025 and X.shape[2] == 1 + a.shape[1] // 1024
    X2, y2, _, _ = spec_utils.cache_or_load(str(tmp_path / 'mix.m4a'), str(tmp_path / 'inst.m4a'), 44100, 1024, 2048)
    assert np.array_equal(X, X2) and np.array_equal(y, y2)
